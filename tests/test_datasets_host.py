"""Host side of plip_b200.datasets: the reference's resizeimg arithmetic, its PIL route, and the PanNuke labelling and
split, against tests/dataset_oracle.py and the frozen golden (no GPU)."""
import os

import numpy as np
import PIL.Image
import pytest

import dataset_oracle as O
from plip_b200 import datasets as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pannuke_golden.npz")


def _oracle_plan(w, h):
    if w == h:
        return 224, 224, 0, 0
    (nw, nh), box = O.resizeimg_box(w, h)
    return nw, nh, round(box[0]), round(box[1])


def test_resizeimg_plan_equals_reference_arithmetic():
    rng = np.random.default_rng(0)
    heights = np.concatenate([np.arange(1, 40), [207, 223, 224, 225, 256, 299, 301, 800, 1000, 2999],
                              rng.integers(1, 3000, 30)])
    for w in range(1, 601):
        for h in heights:
            assert D.resizeimg_plan(w, int(h)) == _oracle_plan(w, int(h)), (w, h)
    short223 = [s for s in range(1, 3000) if int(s * (224 / s)) == 223]
    assert len(short223) == 258 and 207 in short223
    assert D.resizeimg_plan(207, 300)[0] == 223
    assert D.resizeimg_plan(301, 200) == (337, 224, 38, -12)        # odd excess, 12 rows above the image
    assert D.resizeimg_plan(1000, 800) == (280, 224, 388, 288)      # the window misses the image
    assert D.resizeimg_plan(256, 256) == (224, 224, 0, 0)
    assert D.resizeimg_plan(50, 70) == (224, 313, -87, -77)


CASES = [(50, 70), (70, 50), (207, 300), (300, 207), (301, 200), (200, 301), (1000, 800), (800, 1000), (256, 256),
         (1000, 1000), (224, 300), (225, 224), (3, 1000), (1000, 3)]


@pytest.mark.parametrize("mode", ["RGB", "P", "L", "RGBA"])
def test_pil_tiles_from_plan_equal_oracle(mode):
    rng = np.random.default_rng(1)
    for w, h in CASES:
        img = PIL.Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        if mode == "P":
            img = img.quantize(colors=17)
        elif mode != "RGB":
            img = img.convert(mode)
        want = np.asarray(O.resizeimg(img).convert("RGB"))
        got = D._pil_tile(img)
        assert got.shape == (224, 224, 3) and np.array_equal(got, want), (mode, w, h)
    black = D._pil_tile(PIL.Image.fromarray(rng.integers(1, 256, (800, 1000, 3), dtype=np.uint8)))
    assert not black.any()


@pytest.fixture(scope="module")
def folds():
    from plip_b200.synthetic import PANNUKE_TISSUES, make_pannuke_folds
    f = make_pannuke_folds(0)
    assert set(np.concatenate([x[2] for x in f])) == set(PANNUKE_TISSUES)
    return f


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


def _rows(folds):
    masks = np.concatenate([f[1].astype(np.uint8) for f in folds])
    types = np.concatenate([f[2] for f in folds])
    return D.pannuke_rows(O.value_sets(masks), types)


def test_synthetic_folds_cover_the_rule_edges(folds):
    masks = np.concatenate([f[1] for f in folds])
    assert masks.dtype == np.float64 and masks.max() > 255
    u8 = masks.astype(np.uint8)
    counts = O.unique_counts(u8[..., :6])
    kept = ~np.all(u8[..., :5].reshape(len(u8), -1) == 0, axis=1)
    n0, total = counts[:, 0], counts.sum(axis=1)
    assert (~kept).any()
    assert ((n0 == 10) & (n0 / np.maximum(total, 1) > 0.3) & kept).any()
    assert ((n0 == 10) & (n0 / np.maximum(total, 1) < 0.3) & kept).any()
    assert ((n0 == 9) & kept).any()
    assert (u8[..., :5].reshape(len(u8), -1, 5).min(axis=1) > 0).any()       # a channel without a zero
    assert (u8[..., 5].reshape(len(u8), -1).max(axis=1) == 0).any() and (u8[..., 5].max() >= 1)


def test_pannuke_rows_equal_oracle(folds):
    pytest.importorskip("pandas")
    df, src, _ = O.pannuke_table(folds)
    got = _rows(folds)
    assert list(got["image"]) == [os.path.basename(x) for x in df["image"]]
    assert list(got["caption"]) == list(df["caption"])
    assert np.array_equal(got["source_index"], src)


def test_split_equals_oracle(folds):
    pytest.importorskip("pandas")
    df, _, _ = O.pannuke_table(folds)
    for seed, ratio in ((1, 0.7), (3, 0.5)):
        train, test = D.split_pannuke(_rows(folds), seed, ratio)
        for got, want in zip((train, test), O.process_pannuke(df, seed, ratio)):
            assert list(got["image"]) == [os.path.basename(x) for x in want["image"]]
            assert got["label"].dtype == np.float64 and np.array_equal(got["label"], want["label"].to_numpy())
            for col in ("label_text", "text_style_0", "text_style_1", "text_style_4"):
                assert list(got[col]) == list(want[col]), col


def test_rows_and_split_equal_golden(folds, golden):
    rows = _rows(folds)
    assert list(rows["image"]) == list(golden["table_image"])
    assert list(rows["caption"]) == list(golden["table_caption"])
    assert np.array_equal(rows["source_index"], golden["table_source_index"])
    for part, got in zip(("train", "test"), D.split_pannuke(rows, 1, 0.7)):
        assert list(got["image"]) == list(golden[f"{part}_image"])
        assert np.array_equal(got["label"], golden[f"{part}_label"])
        for col in ("label_text", "text_style_0", "text_style_1", "text_style_4"):
            assert list(got[col]) == list(golden[f"{part}_{col}"]), col
        src = dict(zip(golden["table_image"], golden["table_source_index"]))
        assert np.array_equal(got["source_index"], [src[x] for x in got["image"]])


def test_pannuke_rows_rejects_bad_shapes():
    with pytest.raises(ValueError):
        D.pannuke_rows(np.zeros((3, 5, 8), np.uint32), np.array(["Colon"] * 3))
    with pytest.raises(ValueError):
        D.pannuke_rows(np.zeros((3, 6, 8), np.uint32), np.array(["Colon"] * 2))
