"""MuDiPath DenseNet-121 without a GPU: the oracle against the torchvision golden, the host preprocessing, the
packer's key mapping and BN folding, every argument check of the new ABI symbols and the factory's file resolution."""
import ctypes as C
import os
from argparse import Namespace

import numpy as np
import PIL.Image
import pytest
import torch

import densenet_oracle as O
from plip_b200 import _lib
from plip_b200.densenet import CHECKPOINT_NAME, clean_state_dict, fold_bn, pack_state_dict
from plip_b200.preprocess import resize_center_crop_bilinear, to_uint8_tiles_bilinear

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "densenet_golden.npz")


@pytest.fixture(scope="module")
def sd():
    return O.make_state_dict(0)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_weights_checksum_and_bn_statistics(sd, golden):
    assert str(golden["weights_sha256"]) == O.checksum(sd)
    v = sd["features.denseblock2.denselayer3.norm1.running_var"]
    assert (v - 1).abs().max() > 0.1          # calibrated: eval BN is far from the identity


def test_oracle_matches_torchvision_golden(sd, golden):
    out = O.forward_u8(sd, torch.from_numpy(golden["tiles"]))
    ref = torch.from_numpy(golden["outputs"])
    # two fp32 evaluations of the same network that differ only in their convolution algorithms: 1.8e-5 apart at
    # most on these features (largest 17), far inside 1e-4 per element
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-4)


def test_emulation_is_close_to_fp32(sd, golden):
    tiles = torch.from_numpy(golden["tiles"])
    gap = O.cosine_gap(O.forward_u8(sd, tiles, emulate=True), torch.from_numpy(golden["outputs"]))
    assert gap.max().item() < 1e-2


def test_host_bilinear_matches_torchvision_tiles(golden):
    srcs = [golden[f"src{i}"] for i in range(3)]
    tiles = to_uint8_tiles_bilinear([PIL.Image.fromarray(s) for s in srcs])
    assert np.array_equal(tiles, golden["tiles"])
    assert resize_center_crop_bilinear(PIL.Image.fromarray(srcs[0])).size == (224, 224)


@pytest.mark.parametrize("w,h", [(225, 224), (224, 1000), (17, 9), (401, 223), (1200, 900), (224, 224)])
def test_host_bilinear_matches_torchvision_transform(w, h):
    transforms = pytest.importorskip("torchvision.transforms")
    img = PIL.Image.fromarray(np.random.default_rng(w * h).integers(0, 256, (h, w, 3), dtype=np.uint8))
    ref = transforms.Compose([transforms.Resize(224), transforms.CenterCrop(224)])(img)
    assert np.array_equal(np.asarray(resize_center_crop_bilinear(img)), np.asarray(ref))


def test_fold_bn_algebra_fp64():
    g = torch.Generator().manual_seed(0)
    w, b, m = torch.rand(64, generator=g) + 0.5, torch.randn(64, generator=g), torch.randn(64, generator=g)
    v = torch.rand(64, generator=g) * 3
    s, t = fold_bn(w, b, m, v)
    assert s.dtype == torch.float32 and t.dtype == torch.float32
    s64 = w.double() / torch.sqrt(v.double() + 1e-5)
    assert torch.equal(s, s64.float())
    assert torch.equal(t, (b.double() - m.double() * s64).float())
    x = torch.randn(8, 64, 5, 5, generator=g, dtype=torch.float64)
    bn = torch.nn.functional.batch_norm(x, m.double(), v.double(), w.double(), b.double(), training=False, eps=1e-5)
    assert torch.allclose(bn, x * s64.view(1, -1, 1, 1) + (b.double() - m.double() * s64).view(1, -1, 1, 1))


def _table():
    L = _lib.lib()
    out = {}
    for i in range(L.plip_densenet_num_tensors()):
        ti = _lib.TensorInfo()
        assert L.plip_densenet_tensor_info(i, C.byref(ti)) == 0
        out[ti.name.decode()] = (ti.offset, ti.numel, ti.dtype, ti.rows, ti.cols)
    return out


def test_blob_layout():
    L = _lib.lib()
    t = _table()
    assert len(t) == 3 + 58 * 6 + 3 * 3 + 2
    convs = [k for k, v in t.items() if v[2] == 1]
    assert len(convs) == 1 + 58 * 2 + 3
    # every torchvision convolution of DenseNet-121 (the stem padded from 147 to 160 inputs)
    assert sum(t[k][1] for k in convs) == sum(np.prod(s) for k, s in O.param_shapes().items()
                                              if k.endswith(".weight") and len(s) == 4) + 64 * 13
    prev = 0
    for off, numel, dtype, rows, cols in sorted(t.values()):
        assert off % 256 == 0 and off >= prev and numel == rows * cols
        prev = off + numel * (2 if dtype == 1 else 4)
    assert prev <= L.plip_densenet_blob_bytes() < prev + 256


def _read(blob, entry, dtype):
    off, numel = entry[0], entry[1]
    nb = numel * (2 if dtype == torch.bfloat16 else 4)
    return blob[off:off + nb].view(dtype)


def test_packer_mapping(sd):
    t = _table()
    blob = pack_state_dict(sd)
    w = _read(blob, t["features.conv0.weight"], torch.bfloat16).view(64, 160)
    assert torch.equal(w[:, :147], sd["features.conv0.weight"].permute(0, 2, 3, 1).reshape(64, 147).bfloat16())
    assert not w[:, 147:].float().any()
    k = "features.denseblock3.denselayer7.conv2.weight"
    assert torch.equal(_read(blob, t[k], torch.bfloat16).view(32, 1152),
                       sd[k].permute(0, 2, 3, 1).reshape(32, 1152).bfloat16())
    k = "features.transition2.conv.weight"
    assert torch.equal(_read(blob, t[k], torch.bfloat16).view(256, 512), sd[k].view(256, 512).bfloat16())
    s, b = O.fold(sd, "features.denseblock4.denselayer16.norm2")
    assert torch.equal(_read(blob, t["features.denseblock4.denselayer16.norm2.scale"], torch.float32), s)
    assert torch.equal(_read(blob, t["features.denseblock4.denselayer16.norm2.shift"], torch.float32), b)


def test_packer_accepts_raw_mudipath_checkpoint(sd):
    raw = {"features." + k: v for k, v in sd.items() if not k.startswith("classifier.")}
    raw["heads.0.weight"] = torch.zeros(9, 1024)
    raw["heads.0.bias"] = torch.zeros(9)
    cleaned = clean_state_dict(raw, prefix="features.", filter=lambda k: not k.startswith("heads."))
    assert "features.conv0.weight" in cleaned and not any(k.startswith("heads.") for k in cleaned)
    assert torch.equal(pack_state_dict(raw), pack_state_dict(sd))


def test_packer_missing_key_names_it(sd):
    bad = dict(sd)
    del bad["features.denseblock2.denselayer5.norm1.running_var"]
    with pytest.raises(KeyError, match="denseblock2.denselayer5.norm1.running_var"):
        pack_state_dict(bad)
    raw = {"features." + k: v for k, v in sd.items() if k != "features.norm5.bias"}
    raw["heads.0.weight"] = torch.zeros(9, 1024)
    with pytest.raises(KeyError, match="features.norm5.bias"):
        pack_state_dict(raw)


def test_abi_argument_errors():
    L = _lib.lib()
    ti = _lib.TensorInfo()
    assert L.plip_densenet_tensor_info(-1, C.byref(ti)) != 0 and "out of range" in _lib.last_error()
    assert L.plip_densenet_tensor_info(0, None) != 0 and "null" in _lib.last_error()
    assert L.plip_densenet_workspace_bytes(0) == 0
    assert L.plip_densenet_workspace_bytes(2) == 2 * L.plip_densenet_workspace_bytes(1) > 5e6
    h = C.c_void_p()
    buf = (C.c_char * 64)()
    assert L.plip_densenet_create(None, 64, 0, 8, C.byref(h)) != 0 and "null" in _lib.last_error()
    assert L.plip_densenet_create(C.cast(buf, C.c_void_p), 64, 0, 8, C.byref(h)) != 0
    assert "blob is 64 bytes" in _lib.last_error()
    nb = L.plip_densenet_blob_bytes()
    big = (C.c_char * nb)()
    for mb in (0, 4097):
        assert L.plip_densenet_create(C.cast(big, C.c_void_p), nb, 0, mb, C.byref(h)) != 0
        assert f"max_micro_batch {mb}" in _lib.last_error()
    assert L.plip_densenet_destroy(None) == 0
    assert L.plip_densenet_max_micro_batch(None) == 0
    assert L.plip_densenet_encode(None, 1, 1, 1, None) != 0 and "null handle" in _lib.last_error()
    assert L.plip_dbg_densenet_op(6, 16, 0, 1, 7, 32, 16, 16, 16, 16, 16, 16, 32, None) != 0
    assert "op = 6" in _lib.last_error()
    assert L.plip_dbg_densenet_op(2, 16, 0, 0, 7, 32, 16, 16, 16, 16, 16, 16, 128, None) != 0
    assert "n = 0" in _lib.last_error()
    assert L.plip_dbg_densenet_op(2, 17, 64, 1, 7, 32, 16, 16, 16, 16, 16, 16, 128, None) != 0
    assert "aligned" in _lib.last_error()
    assert L.plip_dbg_densenet_op(2, 16, 64, 1, 7, 48, 16, 16, 16, 16, 16, 16, 128, None) != 0
    assert "c_in = 48" in _lib.last_error()
    assert L.plip_dbg_densenet_op(4, 16, 256, 1, 7, 256, 16, 16, 16, None, None, 16, 64, None) != 0
    assert "ldo = 64" in _lib.last_error()
    assert L.plip_dbg_densenet_op(2, 16, 64, 1, 7, 64, 16, None, None, 16, 16, 16, 128, None) != 0
    assert "a_scale" in _lib.last_error()


def test_factory_checkpoint_resolution(tmp_path, monkeypatch):
    from plip_b200.embedders import EmbedderFactory, mudipath_checkpoint
    for var in ("PLIP_B200_MTDP", "TORCH_MODEL_ZOO", "TORCH_HOME"):
        monkeypatch.delenv(var, raising=False)
    monkeypatch.setenv("HOME", str(tmp_path / "home"))
    with pytest.raises(FileNotFoundError, match="PLIP_B200_MTDP"):
        mudipath_checkpoint()
    with pytest.raises(FileNotFoundError, match=CHECKPOINT_NAME):
        EmbedderFactory().factory(Namespace(model_name="mudipath", backbone="default"))
    home_file = tmp_path / "home" / ".torch" / "models" / CHECKPOINT_NAME
    home_file.parent.mkdir(parents=True)
    home_file.write_bytes(b"x")
    assert mudipath_checkpoint() == str(home_file)
    zoo = tmp_path / "zoo"
    zoo.mkdir()
    (zoo / CHECKPOINT_NAME).write_bytes(b"x")
    monkeypatch.setenv("TORCH_MODEL_ZOO", str(zoo))
    assert mudipath_checkpoint() == str(zoo / CHECKPOINT_NAME)
    explicit = tmp_path / "elsewhere.pth"
    explicit.write_bytes(b"x")
    monkeypatch.setenv("PLIP_B200_MTDP", str(explicit))
    assert mudipath_checkpoint() == str(explicit)
    monkeypatch.setenv("PLIP_B200_MTDP", str(zoo))       # a directory holding the file
    assert mudipath_checkpoint() == str(zoo / CHECKPOINT_NAME)
