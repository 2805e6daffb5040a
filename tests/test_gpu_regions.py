"""Slide regions on the GPU: the background counts against numpy, windows encoded in place against the same windows
cut out as tiles (bit for bit), the oracle forward, launch counts, and ``encode_region`` end to end on device and host
regions against the reference's crop loop (region_oracle)."""
import ctypes as C

import numpy as np
import pytest
import torch

import region_oracle as RO
from oracle import clip_oracle as O
from plip_b200._lib import lib
from plip_b200.engine import Engine, window_background_counts
from plip_b200.regions import encode_region, window_grid

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine16(state_dict):
    eng = Engine(state_dict, max_micro_batch=64, operand_dtype="fp16")
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def wide():
    """A 700 x 900 region with white blocks, and a row-strided 693 x 800 view into it (pitch 2700 != 3 * 800)."""
    img = torch.from_numpy(RO.region_with_blocks(700, 900, 1))
    dev = img.cuda()
    return img, dev, img[7:, 61:861], dev[7:, 61:861]


def _crops(region: torch.Tensor, origins) -> torch.Tensor:
    return torch.stack([region[r:r + 224, c:c + 224] for r, c in np.asarray(origins).tolist()]).contiguous()


def _origins(h, w, n, seed, aligned=False):
    g = np.random.default_rng(seed)
    o = np.stack([g.integers(0, h - 224 + 1, n), g.integers(0, w - 224 + 1, n)], 1)
    if aligned:
        o = o // 8 * 8
    o[0] = (h - 224, w - 224)                         # touches the last row and column
    if n > 1:
        o[1] = (0, w - 224)
    return o.astype(np.int32)


def _bg_counts_numpy(img: np.ndarray, origins, thr):
    # exact window sums of the background mask through an integral image
    m = (img >= thr).all(-1).astype(np.int64)
    s = np.zeros((m.shape[0] + 1, m.shape[1] + 1), np.int64)
    s[1:, 1:] = m.cumsum(0).cumsum(1)
    r, c = origins[:, 0].astype(np.int64), origins[:, 1].astype(np.int64)
    return s[r + 224, c + 224] - s[r, c + 224] - s[r + 224, c] + s[r, c]


def test_background_counts_exact(wide):
    img, dev, img_v, dev_v = wide
    for host, region in ((img, dev), (img_v, dev_v)):
        h, w = host.shape[:2]
        o = np.concatenate([_origins(h, w, 2500, 5), window_grid(h, w).origins])   # > one 2048-window launch
        for thr in (200, 0, 1, 231, 255, 256):
            got = window_background_counts(region, o, thr).cpu().numpy()
            assert got.dtype == np.int32
            np.testing.assert_array_equal(got, _bg_counts_numpy(host.numpy(), o, thr))
    crop = img[:224, 3:227].numpy()
    assert window_background_counts(dev, [[0, 3]]).item() / 50176 == RO.background_ratio(crop)


@pytest.mark.parametrize("case", ["aligned", "odd", "strided", "ragged", "normalize", "fp16"])
def test_encode_windows_bit_identical_to_tiles(engine, engine16, wide, case):
    img, dev, _, dev_v = wide
    region = dev_v if case == "strided" else dev
    h, w = region.shape[:2]
    n = {"ragged": 150, "aligned": 12}.get(case, 9)   # 150 > max_micro_batch 64: passes of 64, 64, 22
    o = _origins(h, w, n, seed=len(case), aligned=case == "aligned")
    if case == "odd":
        o = np.where(o % 2 == 0, np.maximum(o - 1, 1), o).astype(np.int32)   # every row and column start odd
    eng = engine16 if case == "fp16" else engine
    norm = case == "normalize"
    got = eng.encode_windows(region, o, normalize=norm)
    ref = eng.encode_images(_crops(region, o), normalize=norm)
    assert got.shape == (n, 512)
    assert torch.equal(got, ref)
    assert torch.equal(eng.encode_windows(region, torch.from_numpy(o).cuda(), normalize=norm), got)


def test_windows_against_oracle_forward(engine, state_dict, wide):
    img, dev, _, _ = wide
    o = np.array([[3, 5], [201, 402], [476, 676]], np.int32)
    ref = O.get_image_features(state_dict, O.preprocess_u8(_crops(img, o)))
    err = (1 - O.cosine(engine.encode_windows(dev, o).cpu(), ref)).max().item()
    print(f"windows vs oracle 1-cos {err:.2e}")
    assert err <= 1e-4


def test_launch_count_equals_encode_images(engine, wide):
    _, dev, _, _ = wide
    L = lib()

    def launches(fn):
        fn()
        torch.cuda.synchronize()
        c0 = L.plip_launch_count()
        fn()
        torch.cuda.synchronize()
        return L.plip_launch_count() - c0

    per = {}
    for n in (3, 150):
        o = _origins(700, 900, n, seed=n)
        tiles = _crops(dev, o)
        per[n] = launches(lambda: engine.encode_windows(dev, o))
        assert per[n] == launches(lambda: engine.encode_images(tiles)), n
    assert per[150] == 3 * per[3]                              # one pass per 64 windows, same launches per pass


def test_encode_region_device_and_host(engine, state_dict):
    img = RO.region_with_blocks(1100, 1300, 7)
    crops, origins, tissue = RO.crops(img)
    assert 0 < len(origins) < len(window_grid(1100, 1300).origins)
    dev = encode_region(engine, torch.from_numpy(img).cuda())
    assert [tuple(x) for x in dev.origins.tolist()] == origins
    assert dev.tissue_ratio.tolist() == tissue
    assert torch.equal(dev.embeddings, engine.encode_images(torch.from_numpy(crops).cuda()))
    # host region in bands of two window rows: same windows, micro-batches of a band only
    for region in (img, torch.from_numpy(img)):
        host = encode_region(engine, region, band_bytes=(201 + 224) * 1300 * 3)
        assert host.origins.tolist() == dev.origins.tolist()
        assert host.tissue_ratio.tolist() == dev.tissue_ratio.tolist()
        assert np.array_equal(host.grid_index, dev.grid_index)
        err = (1 - O.cosine(host.embeddings.cpu(), dev.embeddings.cpu())).max().item()
        assert err < 1e-5, err
    # the score map puts each kept window's cosine at its grid cell
    txt = torch.randn(3, 512, generator=torch.Generator().manual_seed(0)).cuda()
    m = dev.score_map(txt)
    assert m.shape == (3, len(dev.row_starts), len(dev.col_starts))
    cos = engine.similarity(dev.embeddings, txt, scale=1.0)
    for i, gi in enumerate(dev.grid_index.tolist()):
        assert torch.equal(m[:, gi // len(dev.col_starts), gi % len(dev.col_starts)], cos[i])
    assert int(torch.isnan(m).sum()) == 3 * (len(window_grid(1100, 1300).origins) - len(origins))


def test_encode_region_all_background(engine):
    white = np.full((600, 700, 3), 255, np.uint8)
    for region in (torch.from_numpy(white).cuda(), white):
        res = encode_region(engine, region)
        assert res.embeddings.shape == (0, 512) and res.origins.shape == (0, 2) and len(res.tissue_ratio) == 0


def test_plip_encode_region(state_dict):
    from plip_b200.plip import PLIP
    img = RO.region_with_blocks(650, 700, 11)
    crops, origins, tissue = RO.crops(img, 0.5, 0.6)
    plip = PLIP.from_state_dict(state_dict, max_micro_batch=32)
    try:
        emb, org, tis = plip.encode_region(img, crop_overlap=0.5, non_bg_threshold=0.6)
        assert emb.dtype == np.float32 and emb.shape == (len(origins), 512)
        assert [tuple(x) for x in org.tolist()] == origins and tis.tolist() == tissue
        ref = plip.model.engine.encode_images(torch.from_numpy(crops).cuda()).cpu().numpy()
        assert (1 - O.cosine(torch.from_numpy(emb), torch.from_numpy(ref))).max().item() < 1e-5
    finally:
        plip.model.engine.close()


def test_out_of_range_origin_launches_nothing(engine, wide):
    _, dev, _, _ = wide
    L = lib()
    c0 = L.plip_launch_count()
    with pytest.raises(ValueError, match=r"window 1 at \(477, 0\)"):
        engine.encode_windows(dev, [[0, 0], [477, 0]])
    o = np.array([[0, 0], [0, 677]], np.int32)
    out = torch.empty(2, 512, device="cuda")
    rc = L.plip_encode_windows(engine._h, dev.data_ptr(), 700, 900, 2700, o.ctypes.data, 2, out.data_ptr(), 0,
                               C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc != 0 and L.plip_launch_count() == c0
