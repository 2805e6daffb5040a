"""Images of any size (``interpolate_pos_encoding``) without a GPU: the CPU oracle against the live-transformers golden
vectors, the Python size validation, and the argument checks of the new C entry points (no device is touched)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import hires_oracle as HO
from oracle import clip_oracle as O
from plip_b200 import _lib
from plip_b200 import engine as E
from plip_b200.synthetic import pixel_values_hw

torch.set_grad_enabled(False)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hires_golden.npz")


@pytest.fixture(scope="module")
def hires_golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


@pytest.mark.parametrize("h,w", [s for s in HO.HIRES_SIZES if s != (1024, 1024)])
def test_oracle_matches_transformers_golden(hires_golden, state_dict, h, w):
    k = HO.size_key(h, w)
    px = pixel_values_hw(2, h, w)
    hid = []
    out = HO.vision_transformer(state_dict, px, hidden=hid, interpolate_pos_encoding=True)
    feats = O.linear(out, state_dict["visual_projection.weight"])
    ref = torch.from_numpy(hires_golden[f"image_features_{k}"])
    assert (1 - O.cosine(feats, ref)).max().item() < 1e-10
    assert (feats - ref).abs().max().item() < 2e-5
    for l in (0, 1, 12):
        got = torch.cat([hid[l][:1, :5], hid[l][:1, -5:]], dim=1)
        assert (got - torch.from_numpy(hires_golden[f"vision_hidden_{l}_{k}"])).abs().max().item() < 2e-5, l


def test_oracle_flag_off_and_7x7_grid(state_dict):
    px = pixel_values_hw(1, 224, 224)
    base = O.get_image_features(state_dict, px)
    assert torch.equal(HO.get_image_features(state_dict, px, interpolate_pos_encoding=True), base)
    with pytest.raises(ValueError, match=r"Input image size \(256\*256\) doesn't match model \(224\*224\)"):
        HO.get_image_features(state_dict, pixel_values_hw(1, 256, 256))
    pos = state_dict["vision_model.embeddings.position_embedding.weight"]
    assert torch.equal(HO.interpolate_pos(pos, 7, 7), pos)  # bicubic 7 -> 7 has the weights (0, 1, 0, 0)


def test_pixel_format_with_interpolate_pos_encoding():
    for shape in [(2, 3, 448, 448), (1, 3, 32, 32), (1, 3, 266, 250), (1, 3, 1055, 1024), (1, 3, 224, 224)]:
        assert E._pixel_format(torch.zeros(shape), True) == E.PIX_F32_NCHW
        assert E._pixel_hw(torch.zeros(shape), E.PIX_F32_NCHW) == shape[2:]
    assert E._pixel_format(torch.zeros(1, 3, 320, 480, dtype=torch.bfloat16), True) == E.PIX_BF16_NCHW
    u8 = np.zeros((1, 300, 500, 3), np.uint8)
    assert E._pixel_format(u8, True) == E.PIX_U8_NHWC and E._pixel_hw(u8, E.PIX_U8_NHWC) == (300, 500)
    assert E.vision_seq_len(448, 448) == 197 and E.vision_seq_len(266, 250) == 57 and E.vision_seq_len(224, 255) == 50
    for shape in [(1, 3, 31, 224), (1, 3, 224, 31), (1, 3, 1056, 224), (1, 3, 224, 2048)]:
        with pytest.raises(ValueError, match="out of range for interpolate_pos_encoding"):
            E._pixel_format(torch.zeros(shape), True)
    with pytest.raises(ValueError, match="out of range"):
        E._pixel_format(np.zeros((1, 20, 224, 3), np.uint8), True)
    # the flag off keeps the 224-only contract and its message
    with pytest.raises(ValueError, match=r"Input image size \(448\*448\) doesn't match model \(224\*224\)"):
        E._pixel_format(torch.zeros(1, 3, 448, 448))
    with pytest.raises(TypeError):
        E._pixel_format(torch.zeros(1, 3, 448, 448, dtype=torch.float64), True)


def test_c_entry_points_reject_bad_arguments_without_a_device():
    L = _lib.lib()
    buf = (C.c_char * 64)()
    p = C.cast(buf, C.c_void_p)
    for fn in (lambda h, w: L.plip_encode_images_hw(None, p, 0, 1, h, w, p, 0, None),
               lambda h, w: L.plip_dbg_hidden_states_hw(None, p, 0, 1, h, w, 1, p, None)):
        assert fn(16, 224) != 0 and "out of range" in _lib.last_error()
        assert fn(224, 31) != 0 and "out of range" in _lib.last_error()
        assert fn(1056, 224) != 0 and "out of range" in _lib.last_error()   # 33 patches
        assert fn(448, 448) != 0 and "null engine" in _lib.last_error()
    assert L.plip_encode_images_hw(None, None, 0, 1, 448, 448, p, 0, None) != 0 and "null" in _lib.last_error()
    assert L.plip_encode_images_hw(None, p, 0, 0, 448, 448, p, 0, None) != 0 and "positive" in _lib.last_error()
    assert L.plip_encode_images_hw(None, p, 7, 1, 448, 448, p, 0, None) != 0 and "format" in _lib.last_error()
    assert L.plip_dbg_pos_interp(None, 8, 8, p, None) != 0 and "null" in _lib.last_error()
    assert L.plip_dbg_pos_interp(p, 33, 8, p, None) != 0 and "out of" in _lib.last_error()
    assert L.plip_dbg_pos_interp(p, 8, 0, p, None) != 0 and "out of" in _lib.last_error()
    # the long-sequence attention kernel is vision-only: no causal mask, no key mask, S <= 1025
    assert L.plip_dbg_attention(p, 2, 200, 12, 1, None, p, None) != 0 and "causal" in _lib.last_error()
    assert L.plip_dbg_attention(p, 2, 200, 12, 0, p, p, None) != 0 and "mask" in _lib.last_error()
    assert L.plip_dbg_attention(p, 2, 1026, 12, 0, None, p, None) != 0 and "bad shape" in _lib.last_error()
