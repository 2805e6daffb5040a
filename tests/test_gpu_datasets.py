"""plip_resize_crop_fill_u8 and plip_mask_value_sets_u8 against PIL and np.unique, and the dataset builders of
plip_b200.datasets against the frozen PanNuke golden and the embedders reading the reference's saved tiles."""
import hashlib
import os
import types

import numpy as np
import PIL.Image
import pytest
import torch

import dataset_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pannuke_golden.npz")


def _pil(a, nw, nh, left, top):
    return np.asarray(PIL.Image.fromarray(a).resize((nw, nh), PIL.Image.BICUBIC).crop((left, top, left + 224, top + 224)))


def _fill(arrays, plans):
    from plip_b200.datasets import RESIZE_DESC_DTYPE, pack_rgb
    from plip_b200.engine import resize_crop_fill
    plan = np.zeros(len(plans), dtype=RESIZE_DESC_DTYPE)
    for k, p in enumerate(plans):
        plan[k]["new_width"], plan[k]["new_height"], plan[k]["left"], plan[k]["top"] = p
    buf, descs = pack_rgb(arrays, plan=plan)
    return resize_crop_fill(buf.cuda(), descs).cpu().numpy()


def test_fill_kernel_equals_pil_sweep():
    from plip_b200.datasets import resize_fits_device, resizeimg_plan
    rng = np.random.default_rng(0)
    sizes = [(50, 70), (70, 50), (207, 300), (300, 207), (301, 200), (200, 301), (1000, 800), (800, 1000),
             (256, 256), (1000, 1000), (224, 224), (225, 224), (1, 1), (1, 2), (5, 300)]
    arrays, plans = [], []
    for w, h in sizes:
        arrays.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        plans.append(resizeimg_plan(w, h))
    assert plans[6] == (280, 224, 388, 288) and plans[2][0] == 223
    while len(arrays) < 600:                       # > 512 descriptors: two launches
        w, h = (int(x) for x in rng.integers(1, 160, 2))
        nw, nh = (int(x) for x in rng.integers(1, 400, 2))
        left, top = (int(x) for x in rng.integers(-300, 450, 2))
        if rng.integers(0, 4) == 0:
            nw, nh, left, top = resizeimg_plan(w, h)
        if not resize_fits_device(w, h, nw, nh):
            continue
        arrays.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        plans.append((nw, nh, left, top))
    arrays.append(rng.integers(0, 256, (30, 40, 3), dtype=np.uint8))
    plans.append((50, 60, 10 ** 9, -10 ** 9))      # far outside
    got = _fill(arrays, plans)
    for k, (a, p) in enumerate(zip(arrays, plans)):
        assert np.array_equal(got[k], _pil(a, *p)), (k, a.shape, p)
    assert not got[6].any()
    assert got[4][:12].max() == 0 and got[4][12:].any()   # 301 x 200: 12 black rows on top
    extremes = _fill(arrays[:2], [(50, 60, 2 ** 31 - 1, 0), (300, 300, -2 ** 31, -2 ** 31)])
    assert not extremes.any()


def test_fill_kernel_rejects_before_launch():
    from plip_b200._lib import lib
    from plip_b200.datasets import RESIZE_DESC_DTYPE
    from plip_b200.engine import resize_crop_fill
    src = torch.zeros(64 * 64 * 3, dtype=torch.uint8, device="cuda")
    out = torch.full((2, 224, 224, 3), 7, dtype=torch.uint8, device="cuda")
    good = (0, 64, 64, 224, 224, 0, 0)
    bad = [((0, 64, 64, 0, 224, 0, 0), "0x224"), ((0, 64, 64, 224, 65537, 0, 0), "65537"),
           ((0, 64, 65, 224, 224, 0, 0), "exceeds"), ((0, 0, 64, 224, 224, 0, 0), "0x64"),
           ((0, 64, 64, 1, 224, 0, 0), "shrinks too much")]
    torch.cuda.synchronize()
    for d, what in bad:
        descs = np.array([good, d], dtype=RESIZE_DESC_DTYPE)
        before = lib().plip_launch_count()
        with pytest.raises(ValueError, match=what):
            resize_crop_fill(src, descs, out=out)
        assert lib().plip_launch_count() == before
    assert bool((out == 7).all())


def _check_sets(masks_u8):
    from plip_b200.engine import mask_value_sets
    got = mask_value_sets(torch.from_numpy(np.ascontiguousarray(masks_u8)).cuda()).cpu().numpy().view(np.uint32)
    assert np.array_equal(got, O.value_sets(masks_u8)), masks_u8.shape


def test_mask_value_sets_equal_np_unique():
    from plip_b200.synthetic import make_pannuke_folds
    for _, masks, _ in make_pannuke_folds(0, sizes=(9, 7)):
        _check_sets(masks.astype(np.uint8))
    rng = np.random.default_rng(3)
    for shape in [(5, 255, 257, 6), (37, 31, 33, 1), (11, 17, 19, 8), (3, 1, 3, 1), (50, 1, 1, 7), (2, 300, 301, 3),
                  (1, 64, 64, 5)]:
        m = rng.integers(0, 256, shape, dtype=np.uint8)
        m[:, : shape[1] // 2] = rng.integers(0, 3, (shape[0], 1, 1, shape[3]), dtype=np.uint8)   # long runs
        _check_sets(m)
    runs = np.repeat(rng.integers(0, 256, (4, 1, 1, 6), dtype=np.uint8), 200, axis=1).repeat(200, axis=2)
    runs[1, 199, 199, 5] = 77      # one odd byte at the very end
    runs[2, 0, 0, 0] = 78          # and at the very start
    _check_sets(runs)


def test_mask_value_sets_rejects_bad_arguments():
    from plip_b200._lib import lib
    from plip_b200.engine import mask_value_sets
    with pytest.raises(ValueError):
        mask_value_sets(torch.zeros((2, 4, 4, 9), dtype=torch.uint8, device="cuda"))
    base = torch.zeros(4 * 4 * 4 * 2 + 1, dtype=torch.uint8, device="cuda")
    out = torch.zeros((2, 2, 8), dtype=torch.int32, device="cuda")
    before = lib().plip_launch_count()
    rc = lib().plip_mask_value_sets_u8(base.data_ptr() + 1, 2, 4, 4, 2, out.data_ptr(), None)
    assert rc != 0 and lib().plip_launch_count() == before


@pytest.fixture(scope="module")
def pannuke():
    from plip_b200.datasets import pannuke_binary, split_pannuke
    from plip_b200.synthetic import make_pannuke_folds
    folds = make_pannuke_folds(0)
    table = pannuke_binary(folds)
    return folds, table, split_pannuke(table, 1, 0.7)


def _sha(t):
    return hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()


def test_pannuke_end_to_end_equals_golden(pannuke):
    _, table, (train, test) = pannuke
    g = np.load(GOLDEN)
    assert list(table["image"]) == list(g["table_image"])
    assert list(table["caption"]) == list(g["table_caption"])
    assert np.array_equal(table["source_index"], g["table_source_index"])
    assert [_sha(t) for t in table["tiles"]] == list(g["table_tile_sha256"])
    for part, got in (("train", train), ("test", test)):
        assert list(got["image"]) == list(g[f"{part}_image"])
        assert np.array_equal(got["label"], g[f"{part}_label"])
        for col in ("label_text", "text_style_0", "text_style_1", "text_style_4"):
            assert list(got[col]) == list(g[f"{part}_{col}"])
        assert [_sha(t) for t in got["tiles"]] == list(g[f"{part}_tile_sha256"])


def _embedder(engine):
    from plip_b200.embedders import CLIPEmbedder
    model = types.SimpleNamespace(engine=engine, encode_image=engine.encode_images)
    return CLIPEmbedder(model, None, "plip", "synthetic")


def test_pannuke_embeddings_equal_embedder_on_saved_tiles(engine, pannuke, tmp_path):
    folds, _, (train, _) = pannuke
    images = np.concatenate([f[0] for f in folds]).astype(np.uint8)
    paths = []
    for name, src in zip(train["image"], train["source_index"]):
        raw = str(tmp_path / ("raw_" + name))
        PIL.Image.fromarray(images[src]).save(raw)
        with PIL.Image.open(raw) as im:
            O.resizeimg(im).save(str(tmp_path / name))
        paths.append(str(tmp_path / name))
    want = _embedder(engine).embed_images(paths)
    got = engine.encode_images(train["tiles"], normalize=True).cpu().numpy()
    assert np.array_equal(got, want)


def test_evaluation_tiles_equal_saved_tiles(engine, tmp_path):
    from plip_b200.datasets import evaluation_tiles
    rng = np.random.default_rng(5)
    sizes = [(224, 224), (250, 230), (301, 200), (1000, 800), (207, 300), (160, 200), (512, 512), (90, 60), (300, 301)]
    paths = []
    for k, (w, h) in enumerate(sizes):
        img = PIL.Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        if k == 5:
            img = img.quantize(colors=9)                     # a palette PNG
        elif k == 7:
            img = img.convert("RGBA")
        path = str(tmp_path / f"src_{k}.png")
        img.save(path)
        paths.append(path)
    assert PIL.Image.open(paths[5]).mode == "P"
    saved = []
    for k, p in enumerate(paths):
        with PIL.Image.open(p) as im:
            O.saved_tile(im, str(tmp_path / f"tile_{k}.png"))
        saved.append(str(tmp_path / f"tile_{k}.png"))
    want = np.stack([np.asarray(PIL.Image.open(p).convert("RGB")) for p in saved])
    for workers in (0, 3):
        got = evaluation_tiles(paths, num_workers=workers)
        assert np.array_equal(got.cpu().numpy(), want)
    assert not want[3].any()
    emb = _embedder(engine).embed_images(saved)
    assert np.array_equal(engine.encode_images(got, normalize=True).cpu().numpy(), emb)
