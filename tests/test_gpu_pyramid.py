"""Region pyramids on the GPU: the whole-image resize against Pillow bit for bit (whole images, strided views, stitched
row ranges), the mask counts against numpy on Pillow-NEAREST masks, ``encode_region`` with ``downsample`` and a mask and
``encode_region_pyramid`` on device and host regions against the reference's ``random_crop`` (pyramid_oracle), and
argument errors that launch nothing."""
import numpy as np
import pytest
import torch
from PIL import Image

import pyramid_oracle as PO
import region_oracle as RO
from plip_b200._lib import lib
from plip_b200.engine import resize_filter_bounds, resize_region, resize_rows, window_mask_counts
from plip_b200.regions import encode_region, encode_region_pyramid, level_size, window_grid

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def big():
    """A 1111 x 2049 region with white blocks, on the host and the device."""
    img = RO.region_with_blocks(1111, 2049, 21)
    return img, torch.from_numpy(img).cuda()


def _pil(img: np.ndarray, h: int, w: int) -> torch.Tensor:
    return torch.from_numpy(np.array(Image.fromarray(np.ascontiguousarray(img)).resize((w, h)))).cuda()


@pytest.mark.parametrize("ds", [1.5, 2, 3, 4, 8, 16, 32, 0.7])
def test_resize_region_is_pil(big, ds):
    img, dev = big
    for host, src in ((img, dev), (img[7:1000, 61:1900], dev[7:1000, 61:1900])):     # and a row-strided view
        h, w = level_size(host.shape[0], host.shape[1], ds)
        want = _pil(host, h, w)
        got = resize_region(src, h, w)
        assert got.shape == (h, w, 3) and torch.equal(got, want), (ds, host.shape)
    # into a row-strided output view, leaving the rest of the buffer alone
    h, w = level_size(700, 900, ds)
    small = img[:700, :900]
    buf = torch.full((h, w + 5, 3), 7, dtype=torch.uint8, device="cuda")
    resize_region(dev[:700, :900], h, w, out=buf[:, 2:w + 2])
    assert torch.equal(buf[:, 2:w + 2], _pil(small, h, w))
    assert (buf[:, :2] == 7).all() and (buf[:, w + 2:] == 7).all()


@pytest.mark.parametrize("ds", [2, 3, 32])
def test_row_ranges_stitch_to_the_whole_image(big, ds):
    img, dev = big
    H = img.shape[0]
    h, w = level_size(H, img.shape[1], ds)
    whole = resize_region(dev, h, w)
    b = resize_filter_bounds(H, h)
    cuts = sorted({0, h, 1, h // 3, h // 2 + 1, h - 1})
    out = torch.zeros_like(whole)
    for o0, o1 in zip(cuts, cuts[1:]):
        s0, s1 = int(b[o0, 0]), int(b[o1 - 1, 0] + b[o1 - 1, 1])
        band = dev[s0:s1].clone()                        # only the rows the range reads, as a band of its own
        resize_rows(band, s0, H, h, w, (o0, o1), out[o0:o1])
    assert torch.equal(out, whole)


def _np_mask_counts(m: np.ndarray, origins, thr):
    return np.array([int((m[r:r + 224, c:c + 224] > thr).sum()) for r, c in origins], np.int64)


def test_window_mask_counts_on_nearest_masks(big):
    img, _ = big
    for rgb in (False, True):
        mask = PO.tumour_mask(1111, 2049, 4, rgb)
        for (mh, mw) in ((555, 1024), (1111, 2049), (700, 500)):       # downsampled, same size, another aspect
            m = np.array(Image.fromarray(mask).resize((mw, mh), Image.Resampling.NEAREST))
            o = np.concatenate([window_grid(mh, mw).origins, [[mh - 224, mw - 224], [3, 5]]]).astype(np.int32)
            dm = torch.from_numpy(m).cuda()
            for thr in (10, 0, 254):
                got = window_mask_counts(dm, o, thr).cpu().numpy()
                np.testing.assert_array_equal(got, _np_mask_counts(m, o, thr))
    # a row-strided view
    m = PO.tumour_mask(600, 700, 5)
    o = window_grid(590, 600).origins
    got = window_mask_counts(torch.from_numpy(m).cuda()[10:, 50:650], o).cpu().numpy()
    np.testing.assert_array_equal(got, _np_mask_counts(m[10:, 50:650], o, 10))


@pytest.mark.parametrize("ds,mask_kind", [(2, "L"), (3, "RGB"), (2, "other-size")])
def test_encode_region_downsample_with_mask_is_the_reference(engine, big, ds, mask_kind):
    img, dev = big
    mask = {"L": PO.tumour_mask(1111, 2049, 6), "RGB": PO.tumour_mask(1111, 2049, 7, rgb=True),
            "other-size": PO.tumour_mask(800, 1500, 8)}[mask_kind]
    ref = PO.random_crop(img, mask, ds)
    for m in (mask, torch.from_numpy(mask).cuda()):
        res = encode_region(engine, dev, downsample=ds, mask=m)
        assert res.downsample == ds and res.level_size == ref["level"].shape[:2]
        assert [tuple(x) for x in res.origins.tolist()] == ref["origins"]
        assert res.tissue_ratio.tolist() == ref["tissue"]
        assert res.tumor_to_patch_ratio.tolist() == ref["t2p"]
        assert res.tumor_to_tissue_ratio.tolist() == ref["t2t"]
        assert torch.equal(res.embeddings, engine.encode_images(torch.from_numpy(ref["crops"]).cuda()))
    if mask_kind == "RGB":
        assert max(ref["t2p"]) > 1                              # every channel counted, over 224 * 224


def test_downsample_1_with_mask_changes_nothing_else(engine, big):
    img, dev = big
    mask = PO.tumour_mask(1111, 2049, 9)
    plain = encode_region(engine, dev)
    masked = encode_region(engine, dev, mask=mask)
    assert torch.equal(masked.embeddings, plain.embeddings)
    assert np.array_equal(masked.origins, plain.origins) and masked.tissue_ratio.tolist() == plain.tissue_ratio.tolist()
    ref = PO.random_crop(img, mask, 1)
    assert masked.tumor_to_patch_ratio.tolist() == ref["t2p"] and masked.tumor_to_tissue_ratio.tolist() == ref["t2t"]
    assert not plain.tumor_to_patch_ratio.any() and plain.level_size == (1111, 2049)
    host = encode_region(engine, img, mask=mask, band_bytes=(201 + 224) * 2049 * 3)     # the host band path too
    assert host.tumor_to_patch_ratio.tolist() == ref["t2p"] and host.origins.tolist() == plain.origins.tolist()


def test_pyramid_host_bands_equal_device(engine):
    img = RO.region_with_blocks(2300, 1900, 12)
    mask = PO.tumour_mask(2300, 1900, 13)
    dsl = [2, 4, 8, 16, 3]
    dev = encode_region_pyramid(engine, torch.from_numpy(img).cuda(), mask, dsl)
    assert [lv.downsample for lv in dev] == dsl
    assert [len(lv.origins) for lv in dev][3] == 0 and dev[3].level_size == (144, 119)   # under one window: empty
    for band_bytes in (1, 300 * 1900 * 3, 10 ** 9):                  # 1: the smallest bands the planner allows
        for region in (img, torch.from_numpy(img)):
            host = encode_region_pyramid(engine, region, mask, dsl, band_bytes=band_bytes)
            for a, b in zip(host, dev):
                assert a.level_size == b.level_size and np.array_equal(a.origins, b.origins)
                assert a.tissue_ratio.tolist() == b.tissue_ratio.tolist()
                assert a.tumor_to_patch_ratio.tolist() == b.tumor_to_patch_ratio.tolist()
                assert torch.equal(a.embeddings, b.embeddings)
    for lv, ds in zip(dev, dsl):
        ref = PO.random_crop(img, mask, ds)
        assert [tuple(x) for x in lv.origins.tolist()] == (ref["origins"] if ref else [])
        if ref:
            assert lv.tumor_to_tissue_ratio.tolist() == ref["t2t"]
            m = lv.score_map(torch.randn(2, 512, device="cuda"))
            assert m.shape == (2, len(lv.row_starts), len(lv.col_starts))


def test_small_and_background_regions(engine):
    white = np.full((900, 1000, 3), 255, np.uint8)
    for region in (white, torch.from_numpy(white).cuda()):
        levels = encode_region_pyramid(engine, region, np.zeros((900, 1000), np.uint8), [1, 2, 4, 8])
        for lv in levels:
            assert lv.embeddings.shape == (0, 512) and lv.origins.shape == (0, 2)
            assert len(lv.tumor_to_patch_ratio) == len(lv.tissue_ratio) == 0
        assert [lv.level_size for lv in levels] == [(900, 1000), (450, 500), (225, 250), (112, 125)]
    tiny = RO.region_with_blocks(300, 300, 1)
    res = encode_region(engine, torch.from_numpy(tiny).cuda(), downsample=2)
    assert res.embeddings.shape == (0, 512) and res.level_size == (150, 150)


def test_bad_inputs_launch_nothing(engine, big):
    _, dev = big
    L = lib()
    c0 = L.plip_launch_count()
    out = torch.empty(100, 100, 3, dtype=torch.uint8, device="cuda")
    cases = [
        (lambda: resize_region(dev, 0, 10), "outside 1..65536"),
        (lambda: resize_region(dev.float(), 10, 10), "uint8"),
        (lambda: resize_region(dev[:, ::2], 10, 10), "packed"),
        (lambda: resize_region(dev, 100, 100, out=out[:50]), "the output is 50x100"),
        (lambda: resize_region(dev, 100, 5), "shrinks too much"),
        (lambda: resize_rows(dev[100:300], 100, 1111, 555, 1024, (0, 100), out), "the output is 100x100"),
        (lambda: resize_rows(dev[100:300], 100, 1111, 555, 100, (0, 100), out), "the band holds rows"),
        (lambda: resize_rows(dev[100:300], 1000, 1111, 555, 100, (0, 100), out), "not inside the 1111 source rows"),
        (lambda: window_mask_counts(torch.zeros(300, 300, 2, dtype=torch.uint8, device="cuda"), [[0, 0]]), "shape"),
        (lambda: window_mask_counts(torch.zeros(300, 300, dtype=torch.uint8, device="cuda"), [[0, 77]]),
         r"window 0 at \(0, 77\)"),
        (lambda: encode_region_pyramid(engine, dev, downsample_list=[2, -1]), "positive"),
        (lambda: encode_region(engine, dev, downsample=2, mask=np.zeros((10, 10, 4), np.uint8)), "mask"),
    ]
    for fn, msg in cases:
        with pytest.raises(ValueError, match=msg):
            fn()
    torch.cuda.synchronize()
    assert L.plip_launch_count() == c0


def test_plip_encode_region_pyramid_is_the_reference_df_stat(state_dict):
    from plip_b200.plip import PLIP
    img = RO.region_with_blocks(1300, 1200, 14)
    mask = PO.tumour_mask(1300, 1200, 15)
    plip = PLIP.from_state_dict(state_dict, max_micro_batch=32)
    try:
        dsl = [2, 4, 8]
        emb, stats = plip.encode_region_pyramid(Image.fromarray(img), Image.fromarray(mask), dsl, 0.1, 0.5)
        rows = []
        crops = []
        for ds in dsl:
            ref = PO.random_crop(img, mask, ds)
            if ref is None:
                continue
            crops.append(ref["crops"])
            for (r, c), t, p, q in zip(ref["origins"], ref["tissue"], ref["t2p"], ref["t2t"]):
                rows.append((r, c, t, p, q, ds, 224, 0.1, 0.5))
        cols = ["origin_row", "origin_col", "tissue_ratio", "tumor_to_patch_ratio", "tumor_to_tissue_ratio",
                "downsample", "cropsize", "crop_overlap", "non_bg_threshold"]
        assert list(stats) == cols
        for j, name in enumerate(cols):
            assert stats[name].tolist() == [r[j] for r in rows], name
        assert emb.dtype == np.float32 and emb.shape == (len(rows), 512)
        # each level is encoded on its own (its own micro-batches), as encode_images of that level's crops
        want = np.concatenate([plip.model.engine.encode_images(torch.from_numpy(c).cuda()).cpu().numpy() for c in crops])
        assert np.array_equal(emb, want)
    finally:
        plip.model.engine.close()
