"""The train-time transform without a GPU: the parameter draws equal torchvision's, their layout equals a real
``DataLoader``'s, PIL applied with them reproduces the frozen torchvision tiles, and every argument check of
``plip_warp_tiles_u8`` and ``TrainTransform``."""
import ctypes as C
import hashlib
import math
import os

import numpy as np
import PIL.Image
import pytest
import torch
from torch.utils.data import DataLoader, Dataset

from plip_b200 import _lib
from plip_b200.preprocess import TRAIN_PARAMS_DTYPE, TrainTransform, resize_crop_at, resize_plan

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_transform_golden.npz")

# (width, height, first_resize): upscales, exact fits, the no-draw crop, large and extreme aspect ratios
SIZES = [(100, 100, 512), (224, 300, 512), (512, 700, 512), (1200, 900, 512), (4000, 3000, 512), (3000, 250, 512),
         (260, 3000, 512), (300, 300, 224), (224, 224, 224), (640, 480, 256)]


def params_of(tt, w, h, generator=None):
    out = np.zeros(1, dtype=TRAIN_PARAMS_DTYPE)
    out[0] = tt.draw_one(w, h, generator)
    return out[0]


def pil_apply(a, p):
    """Resize + crop, flip, affine and perspective with PIL calls and the drawn parameters."""
    img = resize_crop_at(PIL.Image.fromarray(a), int(p["new_width"]), int(p["new_height"]), int(p["left"]),
                         int(p["top"]))
    w = p["warp"]
    if w["flip"]:
        img = img.transpose(PIL.Image.FLIP_LEFT_RIGHT)
    fill = (int(w["fill"]),) * 3
    img = img.transform((224, 224), PIL.Image.AFFINE, tuple(float(x) for x in w["affine"]), PIL.Image.BILINEAR,
                        fillcolor=fill)
    if w["apply_perspective"]:
        img = img.transform((224, 224), PIL.Image.PERSPECTIVE, tuple(float(x) for x in w["perspective"]),
                            PIL.Image.BILINEAR, fillcolor=fill)
    return np.asarray(img)


@pytest.mark.parametrize("seed", range(12))
def test_draws_equal_torchvision_get_params(seed):
    """Per image: RandomCrop.get_params on the resized size, the flip draw, RandomAffine.get_params and
    _get_inverse_affine_matrix about (112, 112), the perspective draw, RandomPerspective.get_params and
    _get_perspective_coeffs; the generator ends in the same state."""
    T = pytest.importorskip("torchvision.transforms")
    F = pytest.importorskip("torchvision.transforms.functional")
    w, h, first_resize = SIZES[seed % len(SIZES)]
    tt = TrainTransform(first_resize)
    ra = T.RandomAffine(degrees=10, translate=(0.1, 0.1), scale=(0.8, 1.2), shear=(-15, 15, -15, 15))
    torch.manual_seed(seed)
    got = [params_of(tt, w, h) for _ in range(6)]
    after_got = torch.rand(1).item()
    torch.manual_seed(seed)
    nw, nh, _, _ = resize_plan(w, h, first_resize)
    for p in got:
        i, j, _, _ = T.RandomCrop.get_params(PIL.Image.new("RGB", (nw, nh)), (224, 224))
        assert (int(p["new_width"]), int(p["new_height"]), int(p["top"]), int(p["left"])) == (nw, nh, i, j)
        assert bool(p["warp"]["flip"]) == bool(torch.rand(1) < 0.5)
        angle, (tx, ty), scale, shear = T.RandomAffine.get_params(ra.degrees, ra.translate, ra.scale, ra.shear,
                                                                  [224, 224])
        assert (float(p["angle"]), tuple(p["translate"]), float(p["scale"]), tuple(p["shear"])) == \
            (angle, (tx, ty), scale, tuple(shear))
        m = F._get_inverse_affine_matrix([112.0, 112.0], angle, [tx, ty], scale, list(shear))
        assert list(p["warp"]["affine"]) == m
        persp = bool(torch.rand(1) < 0.3)
        assert bool(p["warp"]["apply_perspective"]) == persp
        if persp:
            sp, ep = T.RandomPerspective.get_params(224, 224, 0.3)
            assert p["endpoints"].tolist() == ep
            assert list(p["warp"]["perspective"]) == F._get_perspective_coeffs(sp, ep)
        else:
            assert not p["warp"]["perspective"].any()
        assert int(p["warp"]["fill"]) == 127
    assert torch.rand(1).item() == after_got


def test_exact_fit_draws_no_crop():
    """torchvision's RandomCrop draws nothing when the resized image is exactly 224 x 224."""
    tt = TrainTransform(224)
    torch.manual_seed(3)
    p = params_of(tt, 300, 300)
    assert (int(p["left"]), int(p["top"]), int(p["new_width"]), int(p["new_height"])) == (0, 0, 224, 224)
    torch.manual_seed(3)
    assert bool(p["warp"]["flip"]) == bool(torch.rand(1) < 0.5)   # the flip is the first draw


class _DrawSet(Dataset):
    """What each DataLoader worker draws per image: the transform's draws from the default generator."""

    def __init__(self, tt, sizes):
        self.tt, self.sizes = tt, sizes

    def __len__(self):
        return len(self.sizes)

    def __getitem__(self, i):
        p = params_of(self.tt, *self.sizes[i])
        return torch.from_numpy(np.frombuffer(p.tobytes(), dtype=np.uint8).copy())


@pytest.mark.parametrize("num_workers", [0, 2, 3])
def test_stream_layout_equals_dataloader(num_workers):
    tt = TrainTransform()
    rng = np.random.default_rng(num_workers)
    sizes = [(int(rng.integers(100, 1500)), int(rng.integers(100, 1500))) for _ in range(23)]
    sizes[5] = (512, 512)
    torch.manual_seed(11)
    ref = [bytes(r.numpy()) for b in DataLoader(_DrawSet(tt, sizes), batch_size=4, num_workers=num_workers)
           for r in b]
    after_ref = torch.rand(1).item()
    torch.manual_seed(11)
    stream = tt.stream(num_workers, batch_size=4)
    got = np.concatenate([stream.draw(sizes[:9]), stream.draw(sizes[9:])])   # chunked like the embedder
    after_got = torch.rand(1).item()
    assert [g.tobytes() for g in got] == ref
    assert after_got == after_ref
    torch.manual_seed(11)
    assert tt.draw(sizes, num_workers, 4).tobytes() == got.tobytes()


def _golden_cases():
    g = np.load(GOLDEN, allow_pickle=False)
    return [(tuple(int(v) for v in c), str(k), str(s), pt, bool(pr))
            for c, k, s, pt, pr in zip(g["cases"], g["kinds"], g["sha256"], g["patches"], g["perspective"])]


def golden_image(h, w, seed, kind):
    from golden.make_train_transform_golden import make_image
    return make_image(h, w, seed, kind)


def test_golden_has_perspective_both_ways():
    fired = [c[4] for c in _golden_cases()]
    assert any(fired) and not all(fired)


@pytest.mark.parametrize("case", range(16))
def test_pil_with_drawn_parameters_reproduces_golden(case):
    (h, w, seed, first_resize, torch_seed), kind, sha, patch, persp = _golden_cases()[case]
    a = golden_image(h, w, seed, kind)
    torch.manual_seed(torch_seed)
    p = params_of(TrainTransform(first_resize), w, h)
    assert bool(p["warp"]["apply_perspective"]) == persp
    tile = pil_apply(a, p)
    assert np.array_equal(tile[:24, :24], patch)
    assert hashlib.sha256(np.ascontiguousarray(tile).tobytes()).hexdigest() == sha


def _aligned(buf, k=16):
    addr = C.addressof(buf)
    return addr + (-addr) % k


def _desc(**kw):
    d = _lib.WarpDesc()
    d.affine[:] = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0]
    d.fill = 127
    for k, v in kw.items():
        if k in ("affine", "perspective"):
            getattr(d, k)[:] = v
        else:
            setattr(d, k, v)
    return d


def test_warp_tiles_argument_errors():
    """Rejected on the host, before any CUDA call; the messages name the entry point and the bad value."""
    L = _lib.lib()
    assert C.sizeof(_lib.WarpDesc) == 128
    buf = (C.c_char * 64)()
    a = _aligned(buf)
    tile = 224 * 224 * 3
    one = (_lib.WarpDesc * 2)(_desc(), _desc())
    assert L.plip_warp_tiles_u8(None, a, one, 1, None) != 0
    assert "plip_warp_tiles_u8: null argument" in _lib.last_error()
    assert L.plip_warp_tiles_u8(a, a, None, 1, None) != 0
    assert "null argument" in _lib.last_error()
    for n in (0, -3):
        assert L.plip_warp_tiles_u8(a, a, one, n, None) != 0
        assert f"n must be positive (got {n})" in _lib.last_error()
    assert L.plip_warp_tiles_u8(a + 4, a + 4, one, 1, None) != 0
    assert "16-byte aligned" in _lib.last_error()
    assert L.plip_warp_tiles_u8(a, a + 16 * 9408 - 16, one, 1, None) != 0    # dst starts inside the source tile
    assert "overlap" in _lib.last_error()
    assert L.plip_warp_tiles_u8(a, a + tile - 16, one, 2, None) != 0
    assert "overlap" in _lib.last_error()
    nan, inf = float("nan"), float("inf")
    bad = [(dict(flip=2), "tile 1: flip = 2"), (dict(apply_perspective=-1), "tile 1: apply_perspective = -1"),
           (dict(fill=256), "tile 1: fill = 256"), (dict(fill=-1), "tile 1: fill = -1"),
           (dict(affine=[1, 0, nan, 0, 1, 0]), "tile 1: affine[2] = nan"),
           (dict(affine=[1, 0, 0, 0, 1, -inf]), "tile 1: affine[5] = -inf"),
           (dict(apply_perspective=1, perspective=[1, 0, 0, 0, 1, 0, inf, 0]), "tile 1: perspective[6] = inf")]
    for kw, msg in bad:
        descs = (_lib.WarpDesc * 2)(_desc(), _desc(**kw))
        assert L.plip_warp_tiles_u8(a, a, descs, 2, None) != 0
        err = _lib.last_error()
        assert err.startswith("plip_warp_tiles_u8: ") and msg in err, err


def test_unused_perspective_coefficients_are_not_checked():
    """A descriptor without the perspective warp passes the host checks whatever its perspective field holds: the call
    then gets as far as the launch, which fails here only for want of a device."""
    if torch.cuda.is_available():
        pytest.skip("the launch would run")
    L = _lib.lib()
    buf = (C.c_char * 64)()
    a = _aligned(buf)
    d = (_lib.WarpDesc * 1)(_desc(perspective=[float("nan")] * 8))
    assert L.plip_warp_tiles_u8(a, a, d, 1, None) != 0
    assert "perspective" not in _lib.last_error()


def test_train_transform_argument_errors():
    with pytest.raises(ValueError, match="n_px must be 224"):
        TrainTransform(512, 336)
    with pytest.raises(ValueError, match="first_resize must be >= n_px"):
        TrainTransform(200)
    tt = TrainTransform()
    assert tt.first_resize == 512 and tt.n_px == 224
    with pytest.raises(ValueError, match="num_workers"):
        tt.stream(-1)
    with pytest.raises(ValueError, match="batch_size"):
        tt.stream(0, 0)
    a = np.zeros((300, 400, 3), np.uint8)
    p = tt.draw([(400, 300)])
    with pytest.raises(ValueError, match="2 images but 1 parameter rows"):
        tt.apply([a, a], p, "cpu")
    with pytest.raises(ValueError, match="image 0 is 300x400, its parameters were drawn for 400x300"):
        tt.apply([np.zeros((400, 300, 3), np.uint8)], p, "cpu")
    with pytest.raises(ValueError, match="uint8"):
        tt.apply([a.astype(np.float32)], p, "cpu")


def test_warp_tiles_python_argument_errors():
    from plip_b200.engine import warp_tiles
    with pytest.raises(ValueError, match="CUDA uint8"):
        warp_tiles(torch.zeros(1, 224, 224, 3, dtype=torch.uint8), np.zeros(1, TRAIN_PARAMS_DTYPE)["warp"])


def test_inverse_affine_identity_and_translation():
    from plip_b200.preprocess import inverse_affine_matrix
    assert inverse_affine_matrix(0.0, (0, 0), 1.0, (0.0, 0.0)) == [1.0, -0.0, 0.0, -0.0, 1.0, 0.0]
    m = inverse_affine_matrix(0.0, (5, -3), 2.0, (0.0, 0.0))
    assert m[2] == pytest.approx(112 - (112 + 5) / 2) and m[5] == pytest.approx(112 - (112 - 3) / 2)
    assert math.isclose(m[0], 0.5) and math.isclose(m[4], 0.5)
