"""The train-time transform on the GPU: ``plip_warp_tiles_u8`` bit-identical to Pillow's flip / AFFINE / PERSPECTIVE
warps, the whole device route equal to the frozen torchvision tiles (and to torchvision itself when it is importable),
the host-resize route equal to the device route, and ``CLIPEmbedder`` with a ``TrainTransform`` equal to the engine's
encoding of what a real ``DataLoader`` over torchvision produces."""
import hashlib
import types

import numpy as np
import PIL.Image
import pytest
import torch
from torch.utils.data import DataLoader, Dataset

from test_train_transform_host import _golden_cases, golden_image, params_of

pytestmark = pytest.mark.gpu

IDENT = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0]


def _affine(angle=0.0, t=(0, 0), scale=1.0, shear=(0.0, 0.0)):
    from plip_b200.preprocess import inverse_affine_matrix
    return inverse_affine_matrix(angle, t, scale, shear)


def _persp(ends):
    from plip_b200.preprocess import PERSPECTIVE_CORNERS, perspective_coeffs
    return perspective_coeffs(PERSPECTIVE_CORNERS, ends)


MAX_IN = [[33, 33], [190, 33], [190, 190], [33, 190]]        # every corner pulled in as far as p = 0.3 allows
MAX_SKEW = [[0, 33], [223, 0], [190, 223], [33, 190]]
# (flip, affine, perspective or None, fill)
WARPS = [
    (0, IDENT, None, 127), (1, IDENT, None, 127),
    (0, _affine(angle=10.0), None, 127), (0, _affine(angle=-10.0), None, 127),
    (0, _affine(t=(22, -22)), None, 127), (1, _affine(t=(-22, 22)), None, 127),
    (0, _affine(scale=0.8), None, 127), (0, _affine(scale=1.2), None, 127),
    (0, _affine(shear=(15.0, 0.0)), None, 127), (0, _affine(shear=(-15.0, 0.0)), None, 127),
    (0, _affine(shear=(0.0, 15.0)), None, 127), (0, _affine(shear=(0.0, -15.0)), None, 127),
    (0, IDENT, IDENT + [0.0, 0.0], 127), (0, IDENT, _persp(MAX_IN), 127), (1, IDENT, _persp(MAX_SKEW), 0),
    (0, _affine(-10.0, (-22, -22), 0.8, (15.0, -15.0)), _persp(MAX_IN), 127),          # fill-heavy
    (1, _affine(10.0, (22, 22), 0.8, (-15.0, 15.0)), _persp(MAX_SKEW), 255),
    (1, _affine(7.3, (3, -9), 1.13, (-4.2, 11.9)), _persp([[5, 20], [200, 3], [219, 201], [12, 222]]), 127),
]


def _warp_params(cases):
    from plip_b200.preprocess import WARP_DESC_DTYPE
    p = np.zeros(len(cases), WARP_DESC_DTYPE)
    for i, (flip, aff, per, fill) in enumerate(cases):
        p["affine"][i], p["flip"][i], p["fill"][i] = aff, flip, fill
        if per is not None:
            p["perspective"][i], p["apply_perspective"][i] = per, 1
    return p


def _pil_warp(tile, flip, aff, per, fill):
    img = PIL.Image.fromarray(tile)
    if flip:
        img = img.transpose(PIL.Image.FLIP_LEFT_RIGHT)
    img = img.transform((224, 224), PIL.Image.AFFINE, tuple(aff), PIL.Image.BILINEAR, fillcolor=(fill,) * 3)
    if per is not None:
        img = img.transform((224, 224), PIL.Image.PERSPECTIVE, tuple(per), PIL.Image.BILINEAR, fillcolor=(fill,) * 3)
    return np.asarray(img)


def test_warp_kernel_bit_identical_to_pil():
    from plip_b200.engine import warp_tiles
    rng = np.random.default_rng(0)
    src = rng.integers(0, 256, (len(WARPS), 224, 224, 3), dtype=np.uint8)
    src[::3] = (src[::3] // 64) * 64                     # some flat areas: exact blends
    params = _warp_params(WARPS)
    dev = torch.from_numpy(src).cuda()
    out = warp_tiles(dev, params).cpu().numpy()
    for i, case in enumerate(WARPS):
        ref = _pil_warp(src[i], *case)
        assert np.array_equal(out[i], ref), (i, int((out[i] != ref).sum()))
    assert (out[-3] == 127).mean() > 0.1                   # the fill-heavy cases are fill-heavy
    inplace = warp_tiles(dev, params, out=dev)
    assert inplace.data_ptr() == dev.data_ptr() and np.array_equal(inplace.cpu().numpy(), out)


def test_warp_kernel_random_draws_over_several_launches():
    """300 tiles (three launches of at most 128) with the transform's own random draws."""
    from plip_b200.engine import warp_tiles
    from plip_b200.preprocess import TrainTransform
    tt = TrainTransform(224)
    torch.manual_seed(5)
    params = tt.draw([(224, 224)] * 300)
    assert 40 < params["warp"]["apply_perspective"].sum() < 150 and 100 < params["warp"]["flip"].sum() < 200
    src = np.random.default_rng(1).integers(0, 256, (300, 224, 224, 3), dtype=np.uint8)
    out = warp_tiles(torch.from_numpy(src).cuda(), params["warp"]).cpu().numpy()
    for i in range(0, 300, 7):
        w = params[i]["warp"]
        ref = _pil_warp(src[i], int(w["flip"]), [float(x) for x in w["affine"]],
                        [float(x) for x in w["perspective"]] if w["apply_perspective"] else None, int(w["fill"]))
        assert np.array_equal(out[i], ref), i


def test_warp_tiles_rejects_before_launch():
    from plip_b200.engine import warp_tiles
    from plip_b200.preprocess import WARP_DESC_DTYPE
    t = torch.full((2, 224, 224, 3), 7, dtype=torch.uint8, device="cuda")
    p = np.zeros(2, WARP_DESC_DTYPE)
    p["affine"] = IDENT
    p["fill"][1] = 300
    with pytest.raises(ValueError, match="tile 1: fill = 300"):
        warp_tiles(t, p, out=t)
    with pytest.raises(ValueError, match="2 tiles"):
        warp_tiles(t, p[:1])
    assert bool((t == 7).all())


def _device_route(cases):
    """Golden cases through TrainTransform.apply, one call per first_resize."""
    from plip_b200.preprocess import TrainTransform
    tiles = [None] * len(cases)
    for fr in sorted({c[0][3] for c in cases}):
        idx = [i for i, c in enumerate(cases) if c[0][3] == fr]
        tt = TrainTransform(fr)
        arrays, params = [], []
        for i in idx:
            (h, w, seed, _, torch_seed), kind = cases[i][:2]
            arrays.append(golden_image(h, w, seed, kind))
            torch.manual_seed(torch_seed)
            params.append(params_of(tt, w, h))
        out = tt.apply(arrays, np.array(params), "cuda").cpu().numpy()
        for k, i in enumerate(idx):
            tiles[i] = out[k]
    return tiles


def test_device_route_equals_golden_and_torchvision():
    from golden.make_train_transform_golden import train_transform
    from plip_b200.preprocess import device_resizable
    cases = _golden_cases()
    assert all(device_resizable(c[0][1], c[0][0], c[0][3]) for c in cases)
    tiles = _device_route(cases)
    for (key, kind, sha, patch, _), t in zip(cases, tiles):
        assert np.array_equal(t[:24, :24], patch), key
        assert hashlib.sha256(np.ascontiguousarray(t).tobytes()).hexdigest() == sha, key
    try:
        import torchvision  # noqa: F401
    except ImportError:
        return
    for ((h, w, seed, fr, torch_seed), kind, *_), t in zip(cases, tiles):
        torch.manual_seed(torch_seed)
        ref = np.asarray(train_transform(fr)(PIL.Image.fromarray(golden_image(h, w, seed, kind))))
        assert np.array_equal(t, ref), (h, w, seed, fr, torch_seed)


def test_host_resize_route_equals_device_route(monkeypatch):
    import plip_b200.preprocess as P
    cases = _golden_cases()
    dev = _device_route(cases)
    monkeypatch.setattr(P, "device_resizable", lambda w, h, size=224: False)
    host = _device_route(cases)
    for a, b, c in zip(dev, host, cases):
        assert np.array_equal(a, b), c[0]


class _TorchvisionTiles(Dataset):
    """The reference's CLIPImageDataset with _train_transform up to ToTensor: uint8 HWC tiles."""

    def __init__(self, paths):
        self.paths = paths

    def __len__(self):
        return len(self.paths)

    def __getitem__(self, i):
        from golden.make_train_transform_golden import train_transform
        img = PIL.Image.open(self.paths[i]).convert("RGB")
        return torch.from_numpy(np.asarray(train_transform(512)(img)).copy())


def _image_files(tmp_path):
    rng = np.random.default_rng(7)
    sizes = [(300, 260), (224, 224), (1200, 900), (181, 410), (512, 700), (640, 480), (97, 130), (900, 1200),
             (2048, 1536), (333, 333), (700, 512)]
    paths = []
    for i, (w, h) in enumerate(sizes):
        p = tmp_path / f"img{i}.png"
        mode = "L" if i == 3 else "RGB"                  # converted to RGB first, as CLIPImageDataset does
        PIL.Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).convert(mode).save(p)
        paths.append(str(p))
    return paths


def test_clip_embedder_equals_dataloader_over_torchvision(engine, tmp_path):
    pytest.importorskip("torchvision")
    from plip_b200.embedders import CLIPEmbedder
    from plip_b200.preprocess import TrainTransform
    paths = _image_files(tmp_path)
    torch.manual_seed(0)
    ref_tiles = torch.cat(list(DataLoader(_TorchvisionTiles(paths), batch_size=4, num_workers=2)))
    after_ref = torch.rand(1).item()
    ref = engine.encode_images(ref_tiles.cuda(), normalize=True).cpu().numpy()
    model = types.SimpleNamespace(engine=engine, encode_image=engine.encode_images)
    emb = CLIPEmbedder(model, TrainTransform(), "plip", "synthetic")
    torch.manual_seed(0)
    got = emb.embed_images(paths, num_workers=2, batch_size=4)
    assert torch.rand(1).item() == after_ref
    assert got.shape == (len(paths), 512) and got.dtype == np.float32
    assert np.array_equal(got, ref)
    torch.manual_seed(0)
    tiles = TrainTransform().tiles(paths, "cuda", num_workers=2, batch_size=4)
    assert torch.equal(tiles.cpu(), ref_tiles)


def test_two_runs_are_identical(tmp_path):
    from plip_b200.preprocess import TrainTransform
    paths = _image_files(tmp_path)
    tt = TrainTransform()
    torch.manual_seed(1)
    a = tt.tiles(paths, "cuda", num_workers=3, batch_size=2)
    torch.manual_seed(1)
    b = tt.tiles(paths, "cuda", num_workers=3, batch_size=2)
    assert torch.equal(a, b)
    torch.manual_seed(2)
    assert not torch.equal(a, tt.tiles(paths, "cuda", num_workers=3, batch_size=2))
