"""The similarity head (similarity.cu), its fused top-k and the L2 normalisation (elementwise.cu) against the float64
contracts of similarity_oracle.py, per element, on every dispatch path.

Constants of the kernels the cases derive from (revisit them when one changes):
  launch_similarity   tensor cores when m >= 256, ld >= m_pad (m rounded up to 128) and ld % 8 == 0; the fp32
                      64 x 64 tile kernel otherwise (float4 stores when ld % 4 == 0 and the 4 columns are in range)
  launch_similarity_tc  A rows split and multiplied 131072 at a time (kSimRowChunk): a new row-scale vector and
                      `out + i * ld` per chunk
  plip_similarity     launch_similarity on 65535 x 64 = 4194240 rows at a time (the fp32 kernel's grid.y limit)
  launch_similarity_topk  tensor-core score chunks when n >= 256 and m >= 8192 (chunk width 256 MB / 4n rounded down
                      to 256 columns, within [256, 32768]); one CTA per query when n m < 65536; 64-column tiles in
                      at most 64 splits of the space per 64-query tile otherwise
  l2_normalize_kernel one warp per row, grid capped at 16 x #SMs blocks of 8 warps (16896 rows per pass on 132 SMs)
Every output has 8 guard rows, and columns past what the kernel may write, holding SENT; their bits must survive.
"""
import ctypes as C
import json
import os

import pytest
import torch

from similarity_oracle import (ABI_CHUNK, OBSERVED, ROW_CHUNK, SENT, assert_within, golden_logit_scale,
                               l2_ref, make_pair, similarity_refs, topk_check, FAMILIES)

pytestmark = pytest.mark.gpu

DEV = "cuda"
FLAGS = [(1, 1), (0, 0), (1, 0), (0, 1)]


@pytest.fixture(scope="module")
def L():
    from plip_b200._lib import lib
    yield lib()
    path = os.environ.get("PLIP_EDGE_REPORT")
    if path and OBSERVED:
        with open(path, "w") as f:
            json.dump(OBSERVED, f, indent=1, sort_keys=True)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check(rc, what):
    from plip_b200._lib import check
    check(rc, what)


def _bits(t):
    return t.contiguous().view(torch.int32)


def scales():
    return (1.0, 100.0, golden_logit_scale())


def m_pad_of(m):
    return (m + 127) // 128 * 128


def tc_path(m, ld):
    return m >= 256 and ld >= m_pad_of(m) and ld % 8 == 0


def run_similarity(L, a, b, scale, na, nb, ld):
    """plip_similarity into a SENT-filled [n + 8, ld] buffer; checks that nothing outside what the path may write
    changed (the tensor-core path writes zeros into columns m .. m_pad, NaN in a normalised zero row) and returns
    the full buffer and the [n, m] logits."""
    n, m = a.shape[0], b.shape[0]
    out = torch.full((n + 8, ld), SENT, device=DEV)
    _check(L.plip_similarity(a.data_ptr(), n, b.data_ptr(), m, C.c_float(scale), na, nb, out.data_ptr(), ld,
                             _stream()), "plip_similarity")
    torch.cuda.synchronize()
    w = m_pad_of(m) if tc_path(m, ld) else m
    assert (_bits(out[n:]) == _bits(torch.tensor(SENT))).all(), f"stray write into the guard rows (n={n} m={m} ld={ld})"
    if ld > w:
        assert (_bits(out[:n, w:]) == _bits(torch.tensor(SENT))).all(), f"stray write past column {w} (n={n} m={m} ld={ld})"
    if w > m:   # cs = 0 there: zeros, NaN (inf x 0) in a normalised zero row
        nan_row = torch.isnan(out[:n, :m]).all(1)
        pad = out[:n, m:w]
        assert (pad[~nan_row] == 0).all() and torch.isnan(pad[nan_row]).all(), \
            f"padding columns {m}..{w} not zero (n={n} m={m} ld={ld})"
    return out, out[:n, :m]


def check_logits(out, r, tc, what, rows=slice(None)):
    if tc:
        assert_within(out, r["contract"][rows], r["contract_slack"][rows], 0.0,
                      "similarity tensor cores vs split contract (err / slack)", what)
        assert_within(out, r["plain"][rows], r["plain_slack"][rows], 0.0,
                      "similarity tensor cores vs float64 logits (err / contract + residual slack)", what)
    else:
        assert_within(out, r["plain"][rows], r["simt_slack"][rows], 0.0,
                      "similarity fp32 kernel vs float64 logits (err / slack)", what)


def refs(a, b, scale, na, nb, tc):
    return similarity_refs(a, b, scale, na, nb, need=("contract", "plain") if tc else ("simt",))


# ------------------------------------------------------------------------------------------------------------------
# plip_similarity
# ------------------------------------------------------------------------------------------------------------------
SIM_M = [1, 63, 64, 65, 255, 256, 257, 383, 384, 1000, 10000]
SIM_N = [1, 63, 64, 65, 127, 128, 129]


def lds_of(m):
    """m_pad and m_pad + 128 (tensor cores from m = 256 on), m (the fp32 kernel at m >= 256 unless m = m_pad), m + 1
    (scalar stores), m_pad + 4 (a multiple of 4 the GEMM cannot take: the fp32 kernel)."""
    mp = m_pad_of(m)
    return sorted({mp, mp + 128, m, m + 1, mp + 4})


@pytest.mark.parametrize("m", SIM_M)
def test_similarity_shapes(L, m):
    a_all, b = make_pair("randn", max(SIM_N), m, 100 + m, DEV)
    for na, nb in FLAGS:
        for scale in scales():
            r = {tc: refs(a_all, b, scale, na, nb, tc) for tc in {tc_path(m, ld) for ld in lds_of(m)}}
            for n in SIM_N:
                for ld in lds_of(m):
                    tc = tc_path(m, ld)
                    _, out = run_similarity(L, a_all[:n], b, scale, na, nb, ld)
                    check_logits(out, r[tc], tc, f"n={n} m={m} ld={ld} norm=({na},{nb}) scale={scale}", slice(0, n))


@pytest.mark.parametrize("path", ["tensor_cores", "fp32"])
@pytest.mark.parametrize("family", FAMILIES)
def test_similarity_input_families(L, family, path):
    n, m = 200, 300
    ld = m_pad_of(m) if path == "tensor_cores" else m + 1
    a, b = make_pair(family, n, m, 7, DEV)
    for na, nb in FLAGS:
        for scale in scales():
            r = refs(a, b, scale, na, nb, path == "tensor_cores")
            _, out = run_similarity(L, a, b, scale, na, nb, ld)
            check_logits(out, r, path == "tensor_cores", f"{family} {path} norm=({na},{nb}) scale={scale}")


@pytest.mark.parametrize("n", [ROW_CHUNK + 37, 2 * ROW_CHUNK + 1])
@pytest.mark.parametrize("m,ld", [(257, 384), (64, 64)])
def test_similarity_row_chunks_and_row_shards(L, n, m, ld):
    """Past the 131072-row A chunk of the tensor-core path (each chunk: its own row scales and output offset), rows of
    magnitudes 2^-20 .. 2^20 so that a scale taken from the wrong row shows; and rows i:j of a call equal a call on
    a[i:j] bit for bit (DESIGN §4.4), for slices inside and across the chunk boundary."""
    a, b = make_pair("logmag", n, m, n + m, DEV)
    tc = tc_path(m, ld)
    for na, nb in ((1, 1), (0, 0)):
        full, out = run_similarity(L, a, b, 100.0, na, nb, ld)
        step = 16384
        for i in range(0, n, step):
            j = min(n, i + step)
            check_logits(out[i:j], refs(a[i:j], b, 100.0, na, nb, tc), tc,
                         f"rows {i}:{j} of n={n} m={m} ld={ld} norm=({na},{nb})")
        for i, j in ((5, 1000), (ROW_CHUNK - 100, ROW_CHUNK + 20), (ROW_CHUNK, ROW_CHUNK + 37), (n - 37, n),
                     (ROW_CHUNK - 1, n)):
            _, part = run_similarity(L, a[i:j], b, 100.0, na, nb, ld)
            assert torch.equal(_bits(part), _bits(out[i:j])), f"rows {i}:{j} differ from the unsharded call (m={m})"
        del full, out


def test_similarity_past_abi_chunk(L):
    """n = 4194240 + 3 rows with m = 64 (the fp32 kernel, whose grid.y limits one launch to 4194240 rows): the rows
    around the boundary meet the contract and equal a call on the slice around it bit for bit."""
    n, m = ABI_CHUNK + 3, 64
    need = n * 512 * 4 + (n + 8) * m * 4 + (1 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    try:
        g = torch.Generator(device=DEV).manual_seed(17)
        a = torch.randn(n, 512, generator=g, device=DEV)
        b = torch.randn(m, 512, generator=g, device=DEV)
        full, out = run_similarity(L, a, b, 100.0, 1, 1, m)
        lo = ABI_CHUNK - 64
        r = refs(a[lo:], b, 100.0, 1, 1, False)
        check_logits(out[lo:], r, False, f"rows {lo}:{n} across the ABI chunk")
        check_logits(out[:64], refs(a[:64], b, 100.0, 1, 1, False), False, "rows 0:64")
        _, part = run_similarity(L, a[lo:], b, 100.0, 1, 1, m)
        assert torch.equal(_bits(part), _bits(out[lo:])), "rows across the ABI chunk differ from the call on the slice"
    finally:
        a = b = full = out = part = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# plip_similarity_topk
# ------------------------------------------------------------------------------------------------------------------
TOPK_K = [1, 31, 32, 33, 63, 64]


def topk_path(n, m):
    if n >= 256 and m >= 8192:
        return "tensor_cores"
    return "per_query" if n * m < 65536 else "tiled"


def run_topk(L, q, s, k, scale, nq=1, ns=1, with_val=True):
    n, m = q.shape[0], s.shape[0]
    idx = torch.full((n + 8, k), -7, device=DEV, dtype=torch.int32)
    val = torch.full((n + 8, k), SENT, device=DEV) if with_val else None
    _check(L.plip_similarity_topk(q.data_ptr(), n, s.data_ptr(), m, C.c_float(scale), nq, ns, k, idx.data_ptr(),
                                  val.data_ptr() if with_val else None, _stream()), "plip_similarity_topk")
    torch.cuda.synchronize()
    assert (idx[n:] == -7).all() and (val is None or (_bits(val[n:]) == _bits(torch.tensor(SENT))).all()), \
        "top-k wrote into the guard rows"
    return idx[:n], (val[:n] if with_val else None)


def check_topk_lists(q, s, scale, lists, path, what, nq=1, ns=1, slack_of=None):
    """topk_check of every (k, idx, val) in `lists` against the scores of `path`, in query chunks."""
    n, m = q.shape[0], s.shape[0]
    tc = path == "tensor_cores"
    step = max(1, (1 << 26) // m)
    for i in range(0, n, step):
        j = min(n, i + step)
        r = similarity_refs(q[i:j], s, scale, nq, ns, need=slack_of or (("contract",) if tc else ("simt",)))
        if slack_of:
            ref, slack = r["plain"], torch.maximum(r["plain_slack"], r["simt_slack"])
        elif tc:
            ref, slack = r["contract"], r["contract_slack"]
        else:
            ref, slack = r["plain"], r["simt_slack"]
        for k, idx, val in lists:
            topk_check(idx[i:j], val[i:j], ref, slack, k, f"{what} k={k} queries {i}:{j}",
                       key=f"top-k {path} values vs reference (err / slack)")
        del r, ref, slack


# (n, m): the dispatch boundaries, 64 splits of 2 tiles, 10 tensor-core chunks of 6656 columns with a last one of 96,
# and 131109 queries: every 256-column chunk of the space runs two A-row chunks
TOPK_CASES = [(255, 8192), (256, 8191), (256, 8192), (5, 13107), (4, 16384), (64, 8191), (10000, 60000),
              (ROW_CHUNK + 37, 8192)]


@pytest.mark.parametrize("n,m", TOPK_CASES)
def test_topk_dispatch(L, n, m):
    path = topk_path(n, m)
    q, s = make_pair("parallel", n, m, n + 3 * m, DEV)            # every query has one near-parallel space row
    scale = 100.0
    lists = []
    for k in TOPK_K:
        idx, val = run_topk(L, q, s, k, scale)
        idx2, _ = run_topk(L, q, s, k, scale, with_val=False)
        assert torch.equal(idx, idx2), f"{path} n={n} m={m} k={k}: val = NULL changes the indices"
        lists.append((k, idx, val))
    check_topk_lists(q, s, scale, lists, path, f"{path} n={n} m={m}")
    if path == "tensor_cores":
        # both run launch_similarity_tc on the same rows and columns: the scores are the same bits
        full, _ = run_similarity(L, q, s, scale, 1, 1, m_pad_of(m))
        for k, idx, val in lists:
            got = full[:n].gather(1, idx.long())
            assert torch.equal(_bits(got), _bits(val)), f"n={n} m={m} k={k}: top-k values differ from plip_similarity"
        del full


@pytest.mark.parametrize("shards", [2, 3, 8])
@pytest.mark.parametrize("m", [65536, 20000])
def test_topk_gallery_shards(L, shards, m):
    """ShardedCLIP.retrieval_topk on one device: top-k per gallery shard, global indices, merge_topk_candidates.
    Shards of >= 8192 rows take the tensor-core path as the whole gallery does, and the merged lists equal the
    unsharded ones bit for bit, ties included (copies of a row sit on both sides of every shard boundary).  Smaller
    shards take the fp32 tiled kernel: each list is then a top-k within the fp32 and the split bounds, and a near-tie
    may resolve otherwise than on one GPU."""
    from plip_b200.distributed import merge_topk_candidates, shard_range
    n, k, scale = 256, 32, 100.0
    q, s = make_pair("parallel", n, m, m + shards, DEV)
    bounds = [shard_range(m, r, shards) for r in range(shards)]
    for lo, _ in bounds[1:]:
        s[lo] = s[lo - 1]
    q[:2 * (shards - 1)] = torch.stack([s[lo - d] for lo, _ in bounds[1:] for d in (0, 1)])
    idx1, val1 = run_topk(L, q, s, k, scale)
    ci, cv = [], []
    for lo, hi in bounds:
        idx, val = run_topk(L, q, s[lo:hi], k, scale)
        ci.append(torch.where(idx < 0, torch.full_like(idx, -1), idx + lo).long())
        cv.append(val)
    gi, gv = merge_topk_candidates(torch.cat(ci, 1), torch.cat(cv, 1), k)
    if all(topk_path(n, hi - lo) == "tensor_cores" for lo, hi in bounds):
        assert torch.equal(gi, idx1.long()) and torch.equal(_bits(gv), _bits(val1)), \
            f"{shards} shards of {m}: merged lists differ from the one-device call"
    else:
        check_topk_lists(q, s, scale, [(k, gi.int(), gv)], "gallery shards (fp32 and split)",
                         f"{shards} shards of {m}", slack_of=("plain", "simt"))
    for lo, _ in bounds[1:]:                                       # a tie across a boundary: the lower index first
        rows = (gi[:, 0] == lo - 1).nonzero()[:, 0]
        assert rows.numel() > 0 and (gi[rows, 1] == lo).all(), f"{shards} shards of {m}: tie at {lo} out of order"


# ------------------------------------------------------------------------------------------------------------------
# Zero rows: x / |x| as transformers computes it; NaN scores are never selected
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["tensor_cores", "fp32"])
def test_similarity_zero_rows(L, path):
    n, m = 100, 300
    ld = m_pad_of(m) if path == "tensor_cores" else m + 1
    a, b = make_pair("randn", n, m, 5, DEV)
    a[[3, 17]] = 0
    b[[5, 299]] = 0
    for na, nb in FLAGS:
        _, out = run_similarity(L, a, b, 100.0, na, nb, ld)
        want = torch.zeros(n, m, dtype=torch.bool, device=DEV)
        if na:
            want[[3, 17]] = True
        if nb:
            want[:, [5, 299]] = True
        assert torch.equal(torch.isnan(out), want), f"{path} norm=({na},{nb}): NaN outside the zero rows / columns"
        zero = torch.zeros(n, m, dtype=torch.bool, device=DEV)
        zero[[3, 17]] = True
        zero[:, [5, 299]] = True
        assert (out[zero & ~want] == 0).all(), f"{path} norm=({na},{nb}): un-normalised zero row not zero"
        r = refs(a, b, 100.0, na, nb, path == "tensor_cores")
        clean = {key: torch.where(want, torch.zeros_like(t), t) for key, t in r.items()}
        check_logits(torch.where(want, torch.zeros_like(out), out), clean, path == "tensor_cores",
                     f"{path} zero rows norm=({na},{nb})")


@pytest.mark.parametrize("n,m", [(8, 4000), (200, 3000), (256, 8192)])
def test_topk_zero_rows(L, n, m):
    """A zero query gets index -1 and value -inf throughout; a zero space row is never selected (its scores are NaN)."""
    path = topk_path(n, m)
    q, s = make_pair("parallel", n, m, 9, DEV)
    q[[0, 5]] = 0
    s[[1, 7, m - 1]] = 0
    for k in (1, 33, 64):
        idx, val = run_topk(L, q, s, k, 100.0)
        assert (idx[[0, 5]] == -1).all() and (val[[0, 5]] == float("-inf")).all()
        check_topk_lists(q, s, 100.0, [(k, idx, val)], path, f"zero rows {path} n={n} m={m}")
        assert not torch.isin(idx, torch.tensor([1, 7, m - 1], device=DEV, dtype=idx.dtype)).any()


# ------------------------------------------------------------------------------------------------------------------
# plip_l2_normalize
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 33, 20000])
@pytest.mark.parametrize("dim", [1, 31, 32, 33, 512, 768, 1024])
def test_l2_normalize(L, dim, rows):
    g = torch.Generator(device=DEV).manual_seed(dim * rows)
    buf = torch.full((rows + 8, dim), SENT, device=DEV)
    x = torch.randn(rows, dim, generator=g, device=DEV) * torch.exp2(torch.randint(-20, 21, (rows, 1), device=DEV))
    zeros = [r for r in (0, rows // 2, rows - 1) if rows > 1]
    x[zeros] = 0
    buf[:rows] = x
    _check(L.plip_l2_normalize(buf.data_ptr(), rows, dim, _stream()), "plip_l2_normalize")
    torch.cuda.synchronize()
    assert (_bits(buf[rows:]) == _bits(torch.tensor(SENT))).all(), "l2_normalize wrote into the guard rows"
    ref, rel = l2_ref(x)
    nan = torch.zeros(rows, dtype=torch.bool, device=DEV)
    nan[zeros] = True
    assert torch.equal(torch.isnan(buf[:rows]).all(1), nan) and not torch.isnan(buf[:rows][~nan]).any()
    assert_within(buf[:rows][~nan], ref[~nan], 0.0, rel, "l2_normalize vs float64 (err / relative bound)",
                  f"dim={dim} rows={rows}")


# ------------------------------------------------------------------------------------------------------------------
# Rejections: an error naming the reason, nothing launched, the outputs untouched
# ------------------------------------------------------------------------------------------------------------------
def test_rejections(L):
    from plip_b200._lib import last_error
    a, b = make_pair("randn", 64, 300, 1, DEV)
    out = torch.full((72, 384), SENT, device=DEV)
    idx = torch.full((64, 65), -7, device=DEV, dtype=torch.int32)
    val = torch.full((64, 65), SENT, device=DEV)
    x = torch.full((8, 512), SENT, device=DEV)
    st = _stream()

    def sim(n=64, m=300, ld=384, da=0, db=0, do=0):
        return L.plip_similarity(a.data_ptr() + da, n, b.data_ptr() + db, m, C.c_float(1.0), 1, 1, out.data_ptr() + do,
                                 ld, st)

    def topk(k=5, m=300):
        return L.plip_similarity_topk(a.data_ptr(), 64, b.data_ptr(), m, C.c_float(1.0), 1, 1, k, idx.data_ptr(),
                                      val.data_ptr(), st)

    cases = [(lambda: sim(m=0), "empty operand"), (lambda: sim(ld=299), "ld_logits"),
             (lambda: sim(da=4), "16-byte aligned"), (lambda: sim(db=4), "16-byte aligned"),
             (lambda: sim(do=4), "16-byte aligned"), (lambda: sim(n=-1), "negative row count"),
             (lambda: topk(k=0), "out of range"), (lambda: topk(k=65), "out of range"),
             (lambda: topk(m=0), "empty operand"),
             (lambda: L.plip_l2_normalize(x.data_ptr(), 8, 0, st), "bad shape")]
    torch.cuda.synchronize()
    for call, fragment in cases:
        before = L.plip_launch_count()
        assert call() != 0, fragment
        assert fragment in last_error(), (fragment, last_error())
        assert L.plip_launch_count() == before, f"{fragment}: a kernel was launched"
    torch.cuda.synchronize()
    for t in (out, val, x):
        assert (_bits(t) == _bits(torch.tensor(SENT))).all()
    assert (idx == -7).all()
