"""The bilinear resize of the MuDiPath path without a GPU: the library's filter rows reproduce PIL's BILINEAR resize
exactly, every argument check of ``plip_resize_crop_bilinear_u8``, and the strict ``$PLIP_B200_MTDP`` resolution."""
import ctypes as C

import numpy as np
import PIL.Image
import pytest

from plip_b200 import _lib

SIZES = [(1, 224), (7, 224), (224, 224), (225, 224), (300, 224), (401, 223), (1000, 224), (5000, 224), (224, 1000),
         (13, 1), (641, 387), (387, 641), (2, 3), (65536, 224)]


def _rows(in_size, out_size):
    L = _lib.lib()
    ks = L.plip_dbg_resize_filter_bilinear(in_size, out_size, 0, C.addressof((C.c_int32 * 1)()), 0,
                                           C.byref(C.c_int()), C.byref(C.c_int()))
    assert ks < 0
    ks = -ks
    fs = max(in_size / out_size, 1.0)
    assert ks == int(np.ceil(fs)) * 2 + 1                  # support 1 (bicubic: 2)
    buf = (C.c_int32 * ks)()
    xmin, cnt = C.c_int(), C.c_int()
    rows = []
    for xx in range(out_size):
        assert L.plip_dbg_resize_filter_bilinear(in_size, out_size, xx, C.addressof(buf), ks, C.byref(xmin),
                                                 C.byref(cnt)) == ks
        rows.append((xmin.value, list(buf[:cnt.value])))
    return rows


@pytest.mark.parametrize("in_size,out_size", SIZES)
def test_filter_rows_reproduce_pil_bilinear(in_size, out_size):
    """Pillow skips the pass of an axis whose size does not change, so resizing a few-row image along its width
    applies exactly the horizontal filter rows: fixed point with 22 fraction bits, rounding bias, >> 22, clamp."""
    if in_size * out_size > 3e7:
        out_size = min(out_size, 224)
    rows = _rows(in_size, out_size)
    img = np.random.default_rng(in_size * 7 + out_size).integers(0, 256, (3, in_size, 3), dtype=np.uint8)
    ref = np.asarray(PIL.Image.fromarray(img).resize((out_size, 3), PIL.Image.BILINEAR))
    got = np.empty_like(ref)
    src = img.astype(np.int64)
    for xx, (lo, k) in enumerate(rows):
        acc = (1 << 21) + (src[:, lo:lo + len(k), :] * np.asarray(k, dtype=np.int64)[None, :, None]).sum(1)
        got[:, xx, :] = np.clip(acc >> 22, 0, 255)
    assert np.array_equal(got, ref)


def test_filter_hook_rejects_bad_arguments():
    L = _lib.lib()
    buf = (C.c_int32 * 8)()
    xmin, cnt = C.c_int(), C.c_int()
    assert L.plip_dbg_resize_filter_bilinear(10, 5, 5, C.addressof(buf), 8, C.byref(xmin), C.byref(cnt)) != 0
    assert "plip_dbg_resize_filter_bilinear" in _lib.last_error()
    assert L.plip_dbg_resize_filter_bilinear(0, 5, 0, C.addressof(buf), 8, C.byref(xmin), C.byref(cnt)) != 0


def test_resize_crop_bilinear_argument_errors():
    """Rejected on the host, before any CUDA call; the messages name the entry point and the bad value."""
    L = _lib.lib()
    d = _lib.ResizeDesc(0, 10, 10, 224, 224, 0, 0)
    assert L.plip_resize_crop_bilinear_u8(None, 300, C.byref(d), 1, None, None) != 0
    assert "plip_resize_crop_bilinear_u8: null argument" in _lib.last_error()
    buf = (C.c_char * 512)()
    addr = C.addressof(buf)
    addr += (-addr) % 4
    assert L.plip_resize_crop_bilinear_u8(addr, 300, C.byref(d), 0, addr, None) != 0
    assert "positive" in _lib.last_error()
    for bad, msg in [(_lib.ResizeDesc(0, 10, 10, 224, 224, 0, 0), "exceeds"),
                     (_lib.ResizeDesc(0, 5, 5, 100, 224, 0, 0), "smaller"),
                     (_lib.ResizeDesc(0, 5, 5, 224, 224, 0, 3), "crop origin (0,3)"),
                     (_lib.ResizeDesc(0, 0, 5, 224, 224, 0, 0), "invalid size 0x5")]:
        assert L.plip_resize_crop_bilinear_u8(addr, 256, C.byref(bad), 1, addr, None) != 0
        err = _lib.last_error()
        assert err.startswith("plip_resize_crop_bilinear_u8: image 0") and msg in err, err
    assert L.plip_resize_crop_bilinear_u8(addr + 1, 256, C.byref(_lib.ResizeDesc(0, 5, 5, 224, 224, 0, 0)), 1, addr,
                                          None) != 0
    assert "aligned" in _lib.last_error()


def test_mtdp_variable_that_names_nothing_raises(tmp_path, monkeypatch):
    from plip_b200.densenet import CHECKPOINT_NAME
    from plip_b200.embedders import mudipath_checkpoint
    zoo = tmp_path / "zoo"
    zoo.mkdir()
    (zoo / CHECKPOINT_NAME).write_bytes(b"x")          # a fallback exists, but is not used
    monkeypatch.setenv("TORCH_MODEL_ZOO", str(zoo))
    monkeypatch.setenv("PLIP_B200_MTDP", str(tmp_path / "typo.pth"))
    with pytest.raises(FileNotFoundError, match="typo.pth"):
        mudipath_checkpoint()
    monkeypatch.setenv("PLIP_B200_MTDP", str(tmp_path))  # a directory without the file
    with pytest.raises(FileNotFoundError, match="PLIP_B200_MTDP"):
        mudipath_checkpoint()
    monkeypatch.delenv("PLIP_B200_MTDP")
    assert mudipath_checkpoint() == str(zoo / CHECKPOINT_NAME)
