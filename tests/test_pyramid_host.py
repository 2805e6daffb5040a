"""Region pyramids without a GPU: level sizes, the NEAREST mask map and the library's filter windows against Pillow,
the whole-image resize oracle against Pillow, the host band plan, the tumour-ratio arithmetic, and argument checks of
the new C ABI and Python entry points that must fire before any device call."""
import ctypes as C

import numpy as np
import pytest
import torch
from PIL import Image

import pyramid_oracle as PO
import region_oracle as RO
from oracle import resize_oracle as R
from plip_b200 import _lib
from plip_b200.engine import resize_filter_bounds, resize_region, resize_rows, window_mask_counts
from plip_b200.regions import (level_size, nearest_index, plan_pyramid_bands, tumor_ratios, WINDOW_PIXELS,
                               encode_region_pyramid)


def test_level_size_is_the_reference_new_size():
    g = np.random.default_rng(0)
    for _ in range(60):
        h, w = (int(x) for x in g.integers(1, 3000, 2))
        for ds in (2, 4, 8, 16, 32, 1.5, 3):
            new_size = (int(np.round(w / ds)), int(np.round(h / ds)))    # the reference: PIL's (width, height)
            want = Image.new("RGB", (w, h)).resize(new_size).size if min(new_size) > 0 else new_size
            assert level_size(h, w, ds) == (want[1], want[0]), (h, w, ds)
    # np.round rounds halves to even
    assert level_size(4999, 5001, 2) == (2500, 2500)
    assert level_size(4997, 4997, 2) == (2498, 2498)


def _pil_nearest(in_size: int, out_size: int) -> np.ndarray:
    idx = np.arange(in_size, dtype=np.int32)[None, :]                   # mode "I": every source index visible
    return np.asarray(Image.fromarray(idx, mode="I").resize((out_size, 1), Image.Resampling.NEAREST))[0]


def test_nearest_index_is_pillows_running_sum():
    g = np.random.default_rng(1)
    differs = 0
    for _ in range(300):
        n = int(g.integers(300, 9001))
        ds = float(g.uniform(2, 32))
        out = max(1, int(round(n / ds)))
        got = nearest_index(n, out)
        np.testing.assert_array_equal(got, _pil_nearest(n, out), err_msg=f"{n} -> {out}")
        differs += not np.array_equal(got, ((np.arange(out) + 0.5) * (n / out)).astype(np.int64))
    assert differs > 0                     # the multiply form is not the same map
    for n, out in [(300, 300), (301, 1000), (9000, 7), (7, 9000), (1, 5)]:   # identity, upscales, tiny
        np.testing.assert_array_equal(nearest_index(n, out), _pil_nearest(n, out))
    # both axes of a 2-D mask: Pillow steps rows the same way
    m = np.arange(37 * 53, dtype=np.int32).reshape(37, 53)
    got = np.asarray(Image.fromarray(m, mode="I").resize((11, 5), Image.Resampling.NEAREST))
    np.testing.assert_array_equal(got, m[nearest_index(37, 5)][:, nearest_index(53, 11)])


@pytest.mark.parametrize("in_size,out_size", [(8192, 256), (8192, 128), (9001, 281), (5000, 78), (700, 11)])
def test_library_filters_at_strong_shrinks_match_the_oracle(in_size, out_size):
    xm, xc, kk = R.coefficients(in_size, out_size)
    b = resize_filter_bounds(in_size, out_size)
    np.testing.assert_array_equal(b[:, 0], xm)
    np.testing.assert_array_equal(b[:, 1], xc)
    L = _lib.lib()
    k = np.zeros(kk.shape[1] + 8, np.int32)
    lo, cnt = C.c_int(), C.c_int()
    for xx in sorted({0, 1, out_size // 2, out_size - 2, out_size - 1}):
        assert L.plip_dbg_resize_filter(in_size, out_size, xx, k.ctypes.data, len(k), C.byref(lo), C.byref(cnt)) == \
            kk.shape[1]
        assert (lo.value, cnt.value) == (xm[xx], xc[xx])
        np.testing.assert_array_equal(k[:cnt.value], kk[xx, :cnt.value])


@pytest.mark.parametrize("ds", [2, 3, 4.5, 8, 16, 32])
def test_resize_oracle_equals_pil_on_whole_images(ds):
    img = np.random.default_rng(int(ds * 10)).integers(0, 256, (517, 771, 3), dtype=np.uint8)
    h, w = level_size(517, 771, ds)
    want = np.asarray(Image.fromarray(img).resize((w, h)))
    np.testing.assert_array_equal(R.resize_bicubic_u8(img, w, h), want)


def _check_plan(height, sizes, budget, row_bytes):
    bounds = [resize_filter_bounds(height, lh) for lh in sizes]
    bands = plan_pyramid_bands(bounds, height, row_bytes, budget)
    win = max(int(b[:, 1].max()) for b in bounds)
    seen = [np.zeros(lh, int) for lh in sizes]
    for r0, r1, ranges in bands:
        assert 0 <= r0 < r1 <= height
        assert r1 - r0 >= min(height, win) or r1 == height          # never less than the tallest window
        assert r1 - r0 <= max(budget // row_bytes, win)
        for b, s, (o0, o1) in zip(bounds, seen, ranges):
            s[o0:o1] += 1
            assert (b[o0:o1, 0] >= r0).all() and (b[o0:o1, 0] + b[o0:o1, 1] <= r1).all()
    for s in seen:
        assert (s == 1).all()                                        # every output row exactly once
    return bands


def test_pyramid_band_plan_covers_every_row_once():
    h, w = 8192, 8192
    sizes = [level_size(h, w, ds)[0] for ds in (2, 4, 8, 16, 32)]
    for budget in (1, 129 * 3 * w, 300 * 3 * w, 1000 * 3 * w, 1 << 28, 1 << 40):
        bands = _check_plan(h, sizes, budget, 3 * w)
        if budget == 1:                                              # the smallest band: the 32x window, 128 rows
            assert bands[0][1] - bands[0][0] == int(resize_filter_bounds(h, sizes[-1])[:, 1].max()) == 128
    assert len(_check_plan(h, sizes, 1 << 40, 3 * w)) == 1
    for h2, sizes2 in [(1111, [556, 370, 278, 139, 35]), (700, [700, 1400, 233]), (5, [1, 2, 10])]:
        for budget in (1, 50, 3000, 10 ** 9):
            _check_plan(h2, sizes2, budget, 30)


def test_tumour_ratios_are_the_reference_expressions():
    g = np.random.default_rng(2)
    counts = np.concatenate([[0, 1, 25088, 50176, 50177, 150528], g.integers(0, 150529, 200)])
    tissue = np.concatenate([[0.5, 1.0, 0.75, 0.5, 1.0, 0.9], g.uniform(0.5, 1.0, 200)])
    t2p, t2t = tumor_ratios(counts, tissue)
    for i, (c, t) in enumerate(zip(counts, tissue)):
        c = np.int64(c)                                               # np.sum(...) of the reference is an int64
        assert t2p[i] == c / (224 * 224) and t2t[i] == c / (224 * 224 * t)
    assert t2p[5] == 3.0 and t2p.dtype == t2t.dtype == np.float64   # an RGB mask counts 3 channels: ratios above 1
    z1, z2 = tumor_ratios(None, tissue)
    assert not z1.any() and not z2.any() and z1.shape == tissue.shape
    assert WINDOW_PIXELS == 50176


def test_region_oracle_at_downsample_1_is_the_plain_crop_loop():
    img = RO.region_with_blocks(700, 650, 3)
    crops, origins, tissue = RO.crops(img)
    ref = PO.random_crop(img)
    assert ref["origins"] == origins and ref["tissue"] == tissue and np.array_equal(ref["crops"], crops)
    assert PO.random_crop(img, downsample=4) is None                 # 175 x 162: under one window
    m = PO.tumour_mask(350, 325, 0)                                  # a mask of another size
    ref = PO.random_crop(img, m, 1)
    assert ref["origins"] == origins and max(ref["t2p"]) > 0 and min(ref["t2p"]) < 1


def test_c_abi_checks_resize_and_mask_arguments_before_anything_else():
    L = _lib.lib()
    buf = (C.c_char * 256)()
    addr = C.addressof(buf)
    n = C.c_uint64()
    for args, msg in [((0, 10, 5, 5, 0, 5), "source size 0x10"), ((10, 10, 5, 70000, 0, 5), "output size 5x70000"),
                      ((10, 10, 5, 5, 3, 3), "output rows [3, 3)"), ((10, 10, 5, 5, 0, 6), "output rows [0, 6)"),
                      ((10, 10000, 5, 10, 0, 5), "width 10000 -> 10 shrinks too much")]:
        assert L.plip_resize_region_workspace(*args, C.byref(n)) != 0
        assert msg in _lib.last_error(), (msg, _lib.last_error())
    assert L.plip_resize_region_workspace(100, 100, 50, 50, 0, 50, C.byref(n)) == 0 and n.value > 0
    ws_ok = n.value

    def resize(src_pitch=300, row0=0, rows=100, out_pitch=150, o=(0, 50), ws=None, ws_bytes=None, src=addr):
        return L.plip_resize_region_u8(src, src_pitch, row0, rows, 100, 100, addr, out_pitch, 50, 50, o[0], o[1],
                                       addr if ws is None else ws, ws_ok if ws_bytes is None else ws_bytes, None)

    aligned = addr + (-addr) % 16
    for kw, msg in [(dict(src_pitch=299), "source row pitch 299"), (dict(out_pitch=149), "output row pitch 149"),
                    (dict(row0=-1), "band of 100 rows at row -1"), (dict(row0=10, rows=91), "band of 91 rows at row 10"),
                    (dict(row0=10, rows=90), "output rows [0, 50) read source rows [0, 100), the band holds rows "
                                             "[10, 100)"),
                    (dict(ws=aligned + 4), "16-byte aligned"), (dict(ws=aligned, ws_bytes=ws_ok - 1), "workspace of"),
                    (dict(src=None), "null argument"), (dict(o=(10, 5)), "output rows [10, 5)")]:
        assert resize(**kw) != 0
        assert msg in _lib.last_error(), (msg, _lib.last_error())
    # a band that holds exactly the rows an output range reads passes the band check (fails later at the workspace)
    b = resize_filter_bounds(100, 50)
    s0, s1 = int(b[20, 0]), int(b[29, 0] + b[29, 1])
    assert resize(row0=s0, rows=s1 - s0, o=(20, 30), ws=aligned, ws_bytes=1) != 0
    assert "workspace of 1 bytes" in _lib.last_error()
    assert resize(row0=s0 + 1, rows=s1 - s0 - 1, o=(20, 30), ws=aligned, ws_bytes=1) != 0
    assert "the band holds" in _lib.last_error()

    o = np.ascontiguousarray([[0, 0], [0, 77]], dtype=np.int32)
    for args, msg in [((addr, 300, 300, 2, 300, o.ctypes.data, 1), "channels must be 1 or 3 (got 2)"),
                      ((addr, 300, 300, 1, 299, o.ctypes.data, 1), "row pitch 299 bytes < 1 * width"),
                      ((addr, 300, 300, 3, 899, o.ctypes.data, 1), "row pitch 899 bytes < 3 * width"),
                      ((addr, 300, 300, 1, 300, o.ctypes.data, 2), "window 1 at (0, 77) is outside the 300x300"),
                      ((addr, 223, 300, 1, 300, o.ctypes.data, 1), "smaller than one"),
                      ((None, 300, 300, 1, 300, o.ctypes.data, 1), "null argument"),
                      ((addr, 300, 300, 1, 300, o.ctypes.data, 0), "positive")]:
        assert L.plip_window_mask_counts(*args, 10, addr, None) != 0
        assert msg in _lib.last_error(), (msg, _lib.last_error())
    bnd = np.zeros((4, 2), np.int32)
    assert L.plip_resize_filter_bounds(0, 4, bnd.ctypes.data) != 0 and "outside 1..65536" in _lib.last_error()


class _NoDevice:
    def __getattr__(self, name):
        raise AssertionError(f"device call {name} reached")


def test_python_entry_points_reject_before_any_device_call(monkeypatch):
    import plip_b200.engine as E
    monkeypatch.setattr(E, "lib", lambda *a, **k: _NoDevice())
    host = torch.zeros(300, 400, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA tensor"):
        resize_region(host, 100, 100)
    with pytest.raises(ValueError, match="CUDA tensor"):
        resize_rows(host, 0, 300, 100, 100, (0, 100), host)
    with pytest.raises(ValueError, match="CUDA tensor"):
        window_mask_counts(host[..., 0], [[0, 0]])
    eng = object()
    for kw, msg in [(dict(downsample_list=[2, 0]), "positive"), (dict(downsample_list=[float("nan")]), "positive"),
                    (dict(crop_overlap=1.0), "crop_overlap"), (dict(mask=np.zeros((5, 5, 2), np.uint8)), "mask"),
                    (dict(mask=np.zeros((5, 5), np.float32)), "mask")]:
        with pytest.raises(ValueError, match=msg):
            encode_region_pyramid(eng, host.numpy(), **kw)
    with pytest.raises(ValueError, match="uint8 RGB"):
        encode_region_pyramid(eng, host.numpy()[..., :2])
