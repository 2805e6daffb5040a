"""Slide regions without a GPU: the window grid and keep decision against the reference's crop loop (region_oracle),
score-map placement, band planning, and argument checks that must fire before any device call."""
import ctypes as C

import numpy as np
import pytest
import torch

import region_oracle as RO
from plip_b200 import _lib
from plip_b200.engine import Engine, check_origins, check_region
from plip_b200.regions import RegionEncoding, keep_windows, plan_bands, window_grid

SIZES = [224, 225, 300, 425, 426, 427, 448, 449, 626, 627, 1000]


@pytest.mark.parametrize("crop_overlap", [0.0, 0.1, 0.25, 0.5, -0.2])
def test_window_grid_is_the_reference_loop(crop_overlap):
    for h in SIZES:
        for w in SIZES[::3]:
            g = window_grid(h, w, crop_overlap)
            _, want, _ = RO.crops(np.zeros((h, w, 3), np.uint8), crop_overlap, non_bg_threshold=-np.inf)
            assert [tuple(o) for o in g.origins.tolist()] == want, (h, w, crop_overlap)
            assert g.origins.dtype == np.int32 and g.origins.shape == (len(want), 2)
            assert len(g.origins) == len(g.row_starts) * len(g.col_starts)


def test_window_grid_border_rule():
    # a window that ends exactly on the border is dropped (the reference's `x2 >= shape`)
    assert len(window_grid(224, 224).origins) == 0
    assert window_grid(225, 225).origins.tolist() == [[0, 0]]
    assert window_grid(425, 225).row_starts.tolist() == [0]          # 201 + 224 == 425: dropped
    assert window_grid(426, 225).row_starts.tolist() == [0, 201]
    assert window_grid(448, 448, 0.0).row_starts.tolist() == [0]       # 224 + 224 == 448
    assert window_grid(449, 449, 0.5).row_starts.tolist() == [0, 112, 224]
    with pytest.raises(ValueError, match="crop_overlap"):
        window_grid(500, 500, 1.0)


def test_keep_decision_matches_reference_at_the_boundary():
    # windows with an exact number of background pixels, around the tissue threshold
    for count in [0, 1, 25087, 25088, 25089, 37632, 50175, 50176]:
        patch = np.zeros((224, 224, 3), np.uint8)
        patch.reshape(-1, 3)[:count] = 200
        for thr in (0.5, 0.25, 0.75, 0.0, 1.0):
            keep, tissue = keep_windows(np.array([count]), thr)
            t_ref = 1 - RO.background_ratio(patch)
            assert tissue[0] == t_ref and tissue.dtype == np.float64
            assert bool(keep[0]) == (not t_ref < thr), (count, thr)


@pytest.mark.parametrize("seed", range(4))
def test_keep_decision_on_regions_with_white_blocks(seed):
    img = RO.region_with_blocks(700 + 37 * seed, 900 - 41 * seed, seed)
    g = window_grid(*img.shape[:2])
    counts = np.array([int(((img[r:r + 224, c:c + 224] >= 200).all(-1)).sum()) for r, c in g.origins])
    for thr in (0.5, 0.9):
        keep, tissue = keep_windows(counts, thr)
        _, want, t_want = RO.crops(img, 0.1, thr)
        assert [tuple(o) for o in g.origins[keep].tolist()] == want
        assert tissue[keep].tolist() == t_want                         # float64, bit for bit
        assert 0 < keep.sum() < len(keep) or thr == 0.9


class _FakeSimilarity:
    device = torch.device("cpu")

    def similarity(self, a, b, scale=None, normalize_image=True, normalize_text=True):
        assert scale == 1.0 and normalize_image and normalize_text
        return torch.nn.functional.normalize(a, dim=-1) @ torch.nn.functional.normalize(b, dim=-1).t()


def test_score_map_places_scores_at_grid_cells():
    g = torch.Generator().manual_seed(0)
    rows, cols = np.array([0, 201, 402]), np.array([0, 201, 402, 603])
    grid_index = np.array([0, 5, 6, 11])
    emb, txt = torch.randn(4, 512, generator=g), torch.randn(2, 512, generator=g)
    res = RegionEncoding(_FakeSimilarity(), emb, np.zeros((4, 2), np.int32), np.ones(4), rows, cols, grid_index)
    m = res.score_map(txt)
    assert m.shape == (2, 3, 4)
    cos = torch.nn.functional.normalize(emb, dim=-1) @ torch.nn.functional.normalize(txt, dim=-1).t()
    for i, gi in enumerate(grid_index):
        r, c = divmod(int(gi), 4)
        assert torch.equal(m[:, r, c], cos[i])
    assert int(torch.isnan(m).sum()) == 2 * (12 - 4)
    empty = RegionEncoding(_FakeSimilarity(), emb[:0], np.zeros((0, 2), np.int32), np.ones(0), rows, cols,
                           np.zeros(0, np.int64))
    assert torch.isnan(empty.score_map(txt)).all()


def test_bands_cover_whole_window_rows_within_budget():
    rows = window_grid(5000, 300).row_starts
    for budget in (1, 224 * 900, 1000 * 900, 10 ** 9):
        bands = plan_bands(rows, 300, budget)
        assert [i for a, b in bands for i in range(a, b)] == list(range(len(rows)))
        for a, b in bands:
            assert b - a == 1 or (rows[b - 1] + 224 - rows[a]) * 900 <= budget
    assert len(plan_bands(rows, 300, 10 ** 9)) == 1


def test_region_checks():
    big = torch.zeros(300, 400, 3, dtype=torch.uint8)
    assert check_region(big) == (300, 400, 1200)
    assert check_region(big[10:, 5:305]) == (290, 300, 1200)          # row-strided view
    assert check_region(np.zeros((230, 240, 3), np.uint8)[:, 3:]) == (230, 237, 720)
    for bad, msg in [(big.float(), "dtype"), (big[..., :2], "shape"), (big[0], "shape"), (big[None], "shape"),
                     (big[:200], "smaller"), (big[:, :100], "smaller"),
                     (torch.zeros(300, 800, 3, dtype=torch.uint8)[:, ::2], "strides"), (big.permute(1, 0, 2), "strides"),
                     (torch.zeros(300, 400, 4, dtype=torch.uint8)[..., :3], "strides")]:
        with pytest.raises(ValueError, match=msg):
            check_region(bad)
    assert check_origins([[0, 0], [76, 176]], 300, 400).dtype == np.int32
    for o, i in [([[0, 0], [77, 0]], 1), ([[0, 177]], 0), ([[0, 0], [0, 0], [-1, 3]], 2)]:
        with pytest.raises(ValueError, match=rf"window {i} at \({o[i][0]}, {o[i][1]}\) is outside the 300x400"):
            check_origins(o, 300, 400)
    with pytest.raises(ValueError, match=r"\[n, 2\]"):
        check_origins(np.zeros((3, 3), np.int32), 300, 400)


class _NoDevice:
    """Stands in for the C library: any call is a test failure."""

    def __getattr__(self, name):
        raise AssertionError(f"device call {name} reached")


def test_engine_window_methods_reject_before_any_device_call():
    eng = Engine.__new__(Engine)
    eng._L, eng._h, eng.device = _NoDevice(), None, torch.device("cuda", 0)
    host = torch.zeros(300, 400, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA tensor"):
        eng.encode_windows(host, [[0, 0]])
    with pytest.raises(ValueError, match="CUDA tensor"):
        eng.window_background_counts(host.numpy(), [[0, 0]])


def test_c_abi_checks_windows_before_anything_else():
    L = _lib.lib()
    buf = (C.c_char * 64)()
    addr = C.addressof(buf)

    def origins(*pairs):
        a = np.ascontiguousarray(pairs, dtype=np.int32)
        return a, a.ctypes.data

    keep, o = origins((0, 0), (10, 20), (77, 0))
    assert L.plip_encode_windows(None, addr, 300, 400, 1200, o, 3, addr, 0, None) != 0
    assert "window 2 at (77, 0) is outside the 300x400 region" in _lib.last_error()
    assert L.plip_window_background_counts(addr, 300, 400, 1200, o, 3, 200, addr, None) != 0
    assert "window 2 at (77, 0)" in _lib.last_error()
    _ok, o2 = origins((0, 0))
    assert L.plip_encode_windows(None, addr, 300, 400, 1200, o2, 1, addr, 0, None) != 0
    assert "null engine" in _lib.last_error()
    for args, msg in [((addr, 300, 400, 1199, o2, 1), "row pitch"), ((addr, 223, 400, 1200, o2, 1), "smaller"),
                      ((addr, 300, 400, 1200, o2, 0), "positive"), ((None, 300, 400, 1200, o2, 1), "null argument"),
                      ((addr, 300, 400, 1200, None, 1), "null argument")]:
        assert L.plip_window_background_counts(*args, 200, addr, None) != 0
        assert msg in _lib.last_error(), (msg, _lib.last_error())
    del keep, _ok
