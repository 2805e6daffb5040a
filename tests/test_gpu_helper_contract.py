"""The towers' helper kernels (elementwise.cu) against the float64 references of helper_oracle.py, per element:
LayerNorm, row statistics, im2col, text embeddings and pooled rows, key mask, class rows, row gather, position table.

Constants of the kernels the cases derive from (revisit them when one changes):
  grid_for            at most 16 blocks per SM of 256 threads, so the grid-stride loops take a second trip past
                      16 x #SMs x 8 rows (one warp per row: layernorm, rowstats_cast, text_embed, eos_row) or
                      16 x #SMs x 256 items (one thread per item: im2col, mask_to_i32, cls_rows, gather_rows)
  im2col_kernel       one item per 8 pixels of one image row (per channel for the NCHW formats); vector loads when
                      the base and every row start are aligned (W % 4 for f32, W % 8 for bf16 and u8), scalar loads
                      otherwise; a 224 x 224 batch (compile-time geometry) must be 16-byte aligned
  cls_rows_kernel     one item per float4 of the class row (192 per image)
  gather_rows_kernel  one item per 16-byte piece (dim / 8 + dim / 4 per row)
Every output sits in a buffer with guard rows (and unused slots) holding SENT; their bits must survive.
"""
import json
import os

import pytest
import torch

import helper_oracle as H
from attention_oracle import OBSERVED, SENT, _note

pytestmark = pytest.mark.gpu

DEV = "cuda"
DT = {0: torch.bfloat16, 1: torch.float16}
GUARD = 8


@pytest.fixture(scope="module")
def L():
    from plip_b200._lib import lib
    L = lib()
    yield L
    L.plip_dbg_set_operand_format(0)
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
    t = t.contiguous()
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _fmt(L, fmt):
    _check(L.plip_dbg_set_operand_format(fmt), "operand format")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def warp_cap():
    return 16 * _sms() * 8


def item_cap():
    return 16 * _sms() * 256


def _guarded(rows, cols, dtype=torch.float32, fill=SENT):
    return torch.full((rows + GUARD, cols), fill, device=DEV, dtype=dtype)


def _untouched(buf, start, what, fill=SENT):
    assert _same(buf[start:], torch.full_like(buf[start:], fill)), f"{what}: stray write past row {start}"


def _within(got, ref, slack, key, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= slack)
    assert not bad.any(), f"{what}: {int(bad.sum())} elements outside the bound, first at {bad.nonzero()[0].tolist()}"
    _note(key, (err / slack.clamp_min(1e-300)).max().item())


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------------------------
def _ln_rows(rows, D, seed):
    """Rows cycling through five kinds: N(0.5, 3); near-constant (variance below eps); mean 1e3 with std 1e-2; one
    channel at +-300 (make_state_dict(mode="outlier")); all equal."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(rows, D, generator=g, device=DEV)
    kind = torch.arange(rows, device=DEV) % 5
    x = torch.where((kind == 0)[:, None], x * 3 + 0.5, x)
    x = torch.where((kind == 1)[:, None], 0.25 + 1e-4 * x, x)
    x = torch.where((kind == 2)[:, None], 1e3 + 1e-2 * x, x)
    out_ch = (torch.arange(rows, device=DEV) * 37) % D
    sign = torch.where(torch.arange(rows, device=DEV) % 2 == 0, 300.0, -300.0)
    o = (kind == 3).nonzero()[:, 0]
    x[o, out_ch[o]] = sign[o]
    x = torch.where((kind == 4)[:, None], torch.full_like(x, -7.125), x)
    gam = 1 + 0.1 * torch.randn(D, generator=g, device=DEV)
    bet = 0.1 * torch.randn(D, generator=g, device=DEV)
    return x, gam, bet


def _ln_rows_list():
    c = warp_cap()
    return [1, 7, 8, 9, c - 1, c, c + 1]


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("D", [768, 512])
@pytest.mark.parametrize("rows_at", range(7))
def test_layernorm_contract(L, D, fmt, rows_at):
    """Every addressing mode the engine uses (contiguous, in place, the class rows at stride S * D, row_index with
    duplicates) x every output request (fp32, 16-bit, both): fp32 within layernorm_slack, the 16-bit output the RNE
    cast of the fp32 one whichever outputs were requested."""
    rows = _ln_rows_list()[rows_at]
    _fmt(L, fmt)
    dt = DT[fmt]
    P, gam, bet = _ln_rows(rows, D, rows * 3 + D + fmt)
    ref, slack = H.layernorm_ref(P, gam, bet), H.layernorm_slack(P, gam, bet)
    idx = ((torch.arange(rows, device=DEV) * 7 + 3) % rows).to(torch.int32)
    if rows > 1:
        idx[1] = idx[0]                                          # a duplicate
    modes = [("contiguous", None), ("row_index", None), ("in place", None)]
    modes += [(f"stride S={S}", S) for S in ((50, 65, 1025) if rows < 100 else (50,))]
    for mode, S in modes:
        want, want_slack = (ref[idx.long()], slack[idx.long()]) if mode == "row_index" else (ref, slack)
        results = {}
        for req in ("both", "f32", "16"):
            what = f"layernorm D={D} fmt={fmt} rows={rows} {mode} out={req}"
            if mode == "in place":
                if req == "16":
                    continue
                x = _guarded(rows, D)
                x[:rows] = P
                xp, stride, ri, of = x, D, None, x
            elif S is not None:
                x = torch.full((rows * S + GUARD, D), SENT, device=DEV)
                x[:rows * S].view(rows, S, D)[:, 0] = P
                xp, stride, ri, of = x, S * D, None, _guarded(rows, D)
            else:
                x = _guarded(rows, D)
                x[:rows] = P
                xp, stride, ri, of = x, D, (idx if mode == "row_index" else None), _guarded(rows, D)
            before = xp.clone()
            o16 = _guarded(rows, D, dt)
            _check(L.plip_dbg_layernorm_ex(xp.data_ptr(), ri.data_ptr() if ri is not None else None, stride, rows, D,
                                           gam.data_ptr(), bet.data_ptr(), of.data_ptr() if req != "16" else None,
                                           o16.data_ptr() if req != "f32" else None, _stream()), what)
            torch.cuda.synchronize()
            if req != "16":
                _within(of[:rows], want, want_slack, f"layernorm D={D} (err / layernorm_slack)", what)
                _untouched(of, rows, what + " (fp32 guard rows)")
                results["f32"] = of[:rows].clone()
            if req != "f32":
                _untouched(o16, rows, what + " (16-bit guard rows)")
                results.setdefault("16", []).append(o16[:rows].clone())
            else:
                _untouched(o16, 0, what + " (16-bit output not requested)")
            if mode != "in place":
                assert _same(xp, before), what + ": the input changed"
        if "16" in results:
            assert _same(results["16"][0], results["f32"].to(dt)), f"{mode}: 16-bit output is not the RNE cast"
            for o in results["16"][1:]:
                assert _same(o, results["16"][0]), f"{mode}: 16-bit-only call differs from the two-output call"


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("D", [768, 512])
@pytest.mark.parametrize("rows_at", range(7))
def test_rowstats_contract(L, D, fmt, rows_at):
    """rowstats_cast: the 16-bit copy exact, slot 0 within rowstats_ref's depth bound, slots 1..7 and the guard rows
    untouched."""
    rows = _ln_rows_list()[rows_at]
    _fmt(L, fmt)
    x, _, _ = _ln_rows(rows, D, rows + D * 5 + fmt)
    xb = _guarded(rows, D, DT[fmt])
    stats = torch.full((rows + GUARD, 8, 2), SENT, device=DEV)
    what = f"rowstats D={D} fmt={fmt} rows={rows}"
    _check(L.plip_dbg_rowstats_cast(x.data_ptr(), rows, D, xb.data_ptr(), stats.data_ptr(), _stream()), what)
    torch.cuda.synchronize()
    assert _same(xb[:rows], x.to(DT[fmt])), what + ": 16-bit copy"
    _untouched(xb, rows, what + " (16-bit guard rows)")
    s1, s2, t1, t2 = H.rowstats_ref(x)
    _within(stats[:rows, 0, 0], s1, t1, "row statistics sum (err / gamma(V+7) sum|x|)", what)
    _within(stats[:rows, 0, 1], s2, t2, "row statistics sum of squares (err / gamma(V+8) sum x^2)", what)
    keep = stats.clone()
    keep[:rows, 0] = SENT
    assert _same(keep, torch.full_like(keep, SENT)), what + ": statistics slots 1..7 or guard rows written"


# ------------------------------------------------------------------------------------------------------------------
# im2col
# ------------------------------------------------------------------------------------------------------------------
SIZES = [(224, 224), (32, 32), (256, 256), (448, 448), (320, 480), (266, 250), (63, 95), (1024, 1024)]
PIX = {0: torch.float32, 1: torch.bfloat16, 2: torch.uint8}


def _pixels(pix, n, h, w, seed, offset=0):
    """n images in pixel format pix, the rows and columns im2col must not read (H % 32, W % 32) set to NaN (255 for
    uint8); offset > 0 starts the batch that many elements into its allocation."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    shape = (n, h, w, 3) if pix == 2 else (n, 3, h, w)
    numel = n * 3 * h * w
    base = torch.empty(numel + offset, device=DEV, dtype=PIX[pix])
    px = base[offset:].view(shape)
    if pix == 2:
        px.copy_(torch.randint(0, 255, shape, generator=g, device=DEV, dtype=torch.uint8))   # 255 marks unread pixels
        px[:, (h // 32) * 32:] = 255
        px[:, :, (w // 32) * 32:] = 255
    else:
        px.copy_(torch.randn(shape, generator=g, device=DEV) * 2)
        px[:, :, (h // 32) * 32:] = float("nan")
        px[:, :, :, (w // 32) * 32:] = float("nan")
    return px


def _im2col_ns(pix, h, w):
    per = (1 if pix == 2 else 3) * (h // 32) * 32 * (w // 32) * 4
    k = item_cap() // per
    return sorted({1, k + 1, 2 * k + 1})


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("pix", [0, 1, 2])
@pytest.mark.parametrize("h,w", SIZES)
def test_im2col_contract(L, h, w, pix, fmt):
    """im2col_ref bit for bit at every n that ends a grid-stride trip, through the vector and the scalar loads; a
    batch one element off alignment takes the scalar path, or is refused at 224 x 224."""
    _fmt(L, fmt)
    dt = DT[fmt]
    P = (h // 32) * (w // 32)
    cases = [(n, 0) for n in _im2col_ns(pix, h, w)] + [(2, 1)]
    for n, off in cases:
        what = f"im2col {h}x{w} pix={pix} fmt={fmt} n={n} offset={off}"
        px = _pixels(pix, n, h, w, h * w + n + pix, off)
        out = _guarded(n * P, 3072, dt)
        count = _launches(L)
        rc = L.plip_dbg_im2col_hw(px.data_ptr(), pix, n, h, w, out.data_ptr(), _stream())
        if off and (h, w) == (224, 224):
            assert rc != 0 and _launches(L) == count, what + ": a misaligned 224 x 224 batch must be refused"
            torch.cuda.synchronize()
            _untouched(out, 0, what + " (refused)")
            continue
        _check(rc, what)
        torch.cuda.synchronize()
        assert _same(out[:n * P], H.im2col_ref(px, pix, dt)), what
        _untouched(out, n * P, what + " (guard rows)")


def test_im2col_hw_matches_224_hook(L):
    """plip_dbg_im2col (the 224 x 224 hook) and plip_dbg_im2col_hw at 224 x 224 are the same launch."""
    _fmt(L, 0)
    px = _pixels(2, 3, 224, 224, 5)
    a = _guarded(3 * 49, 3072, torch.bfloat16)
    b = a.clone()
    _check(L.plip_dbg_im2col(px.data_ptr(), 2, 3, a.data_ptr(), _stream()), "im2col")
    _check(L.plip_dbg_im2col_hw(px.data_ptr(), 2, 3, 224, 224, b.data_ptr(), _stream()), "im2col_hw")
    torch.cuda.synchronize()
    assert _same(a, b)


# ------------------------------------------------------------------------------------------------------------------
# Text embeddings and pooled rows
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tables():
    g = torch.Generator(device=DEV).manual_seed(77)
    return (torch.randn(H.VOCAB, 512, generator=g, device=DEV) * 0.02,
            torch.randn(77, 512, generator=g, device=DEV) * 0.01)


def _caption_ids(n, i64, seed):
    """n rows of 77 ids cycling through the patterns the pooling must get right: no eos; one eos at t in
    {0, 31, 32, 63, 64, 76} (past a shorter prefix: none seen); several eos; the largest id tied within one lane
    (t, t + 32, t + 64) and across lanes (t, t + 1); out-of-vocabulary ids (-1, 49408, 2^40 for int64)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    ids = torch.randint(1, 40000, (n, 77), generator=g, device=DEV, dtype=torch.int64)
    pat = torch.arange(n, device=DEV) % 12
    for k, t in enumerate((0, 31, 32, 63, 64, 76)):
        ids[pat == k + 1, t] = H.EOS_ID
    sel = pat == 7
    ids[sel, 5], ids[sel, 40], ids[sel, 70] = H.EOS_ID, H.EOS_ID, H.EOS_ID
    sel = pat == 8
    ids[sel, 3], ids[sel, 35], ids[sel, 67] = 49000, 49000, 49000
    sel = pat == 9
    ids[sel, 10], ids[sel, 11] = 49001, 49001
    sel = pat == 10
    ids[sel, 0], ids[sel, 1] = -1, 49408
    if i64:
        ids[sel, 2] = 2 ** 40
    sel = pat == 11
    ids[sel, 33], ids[sel, 34] = 49406, 49406                      # tie of the largest id in the 2nd warp-wide pass
    return ids if i64 else ids.to(torch.int32)


def _run_text(L, tables, ids, n, S, mode):
    tok, pos = tables
    x = _guarded(n * S, 512)
    rows = torch.full((n + GUARD,), -7, device=DEV, dtype=torch.int32)
    dtype = 1 if ids.dtype == torch.int64 else 0
    what = f"text_embed {'i64' if dtype else 'i32'} n={n} seq_len={S} mode={mode}"
    _check(L.plip_dbg_text_embed(ids.data_ptr(), dtype, n, S, ids.shape[1], tok.data_ptr(), pos.data_ptr(), x.data_ptr(),
                                 rows.data_ptr(), mode, _stream()), what)
    torch.cuda.synchronize()
    assert _same(x[:n * S], H.text_embed_ref(ids, S, tok, pos)), what + ": embedding rows"
    _untouched(x, n * S, what + " (guard rows)")
    want = H.pooled_rows_ref(ids.cpu(), S, mode).to(torch.int32)
    assert torch.equal(rows[:n].cpu(), want), what + ": pooled rows"
    assert (rows[n:] == -7).all(), what + ": stray pooled-row write"


@pytest.mark.parametrize("i64", [False, True])
@pytest.mark.parametrize("S", [1, 31, 32, 33, 64, 65, 77])
def test_text_embed_and_pooling(L, tables, S, i64):
    ids = _caption_ids(48, i64, S)
    for mode in (0, 1):
        _run_text(L, tables, ids, 48, S, mode)


@pytest.mark.parametrize("S,n_of", [(77, lambda c: c // 77), (77, lambda c: c // 77 + 1), (77, lambda c: 2 * (c // 77) + 1),
                                    (1, lambda c: c - 1), (1, lambda c: c), (1, lambda c: c + 1),
                                    (33, lambda c: c + 1)])
def test_text_embed_trip_edges(L, tables, S, n_of):
    """The embedding grid (n * seq_len warps) and the pooling grid (n warps) across their cap of 16 x #SMs x 8."""
    n = n_of(warp_cap())
    ids = _caption_ids(n, True, n)
    _run_text(L, tables, ids, n, S, 1)


# ------------------------------------------------------------------------------------------------------------------
# Key mask, class rows, row gather
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("i64", [False, True])
@pytest.mark.parametrize("S,n_of", [(77, lambda c: 50), (40, lambda c: c // 40 + 1), (1, lambda c: c - 1),
                                    (1, lambda c: c), (1, lambda c: c + 1)])
def test_mask_to_i32(L, S, n_of, i64):
    n = n_of(item_cap())
    stride = 77
    vals = torch.tensor([0, 1, 2, -1] + ([2 ** 33, 2 ** 32] if i64 else [2 ** 31 - 1, -2 ** 31]), device=DEV)
    g = torch.Generator(device=DEV).manual_seed(S + n)
    m = vals[torch.randint(0, len(vals), (n, stride), generator=g, device=DEV)].to(torch.int64 if i64 else torch.int32)
    out = torch.full((n * S + 64,), -7, device=DEV, dtype=torch.int32)
    what = f"mask {'i64' if i64 else 'i32'} n={n} seq_len={S}"
    _check(L.plip_dbg_mask_to_i32(m.data_ptr(), int(i64), n * S, S, stride, out.data_ptr(), _stream()), what)
    torch.cuda.synchronize()
    assert torch.equal(out[:n * S], H.mask_ref(m, S)), what
    assert (out[n * S:] == -7).all(), what + ": stray write"


@pytest.mark.parametrize("S", [50, 65, 1025])
def test_cls_rows(L, S):
    g = torch.Generator(device=DEV).manual_seed(S)
    cls, pos0 = torch.randn(768, generator=g, device=DEV), torch.randn(768, generator=g, device=DEV)
    k = item_cap() // 192
    for n in ([1, 3, 7] if S == 1025 else [1, k, k + 1, 2 * k + 1]):
        x = _guarded(n * S, 768)
        what = f"cls_rows S={S} n={n}"
        _check(L.plip_dbg_cls_rows(cls.data_ptr(), pos0.data_ptr(), n, S, x.data_ptr(), _stream()), what)
        torch.cuda.synchronize()
        want = torch.full_like(x, SENT)
        want[:n * S].view(n, S, 768)[:, 0] = H.cls_rows_ref(cls, pos0)
        assert _same(x, want), what + ": class rows, patch rows or guard rows"


@pytest.mark.parametrize("D", [768, 512])
def test_gather_rows(L, D):
    dt = torch.bfloat16                                                  # the 16-bit rows are copied as bits
    k = item_cap() // (D // 8 + D // 4)
    for n in (1, k, k + 1, 2 * k + 1):
        for by_index in (False, True):
            S = 50
            g = torch.Generator(device=DEV).manual_seed(n + D)
            src = n * S
            a16 = torch.randn(src, D, generator=g, device=DEV).to(dt)
            x32 = torch.randn(src, D, generator=g, device=DEV)
            idx = torch.randint(0, src, (n,), generator=g, device=DEV, dtype=torch.int32)
            if n > 1:
                idx[1] = idx[0]
            ao, xo = _guarded(n, D, dt), _guarded(n, D)
            what = f"gather_rows D={D} n={n} {'row_index' if by_index else 'stride'}"
            _check(L.plip_dbg_gather_rows(a16.data_ptr(), x32.data_ptr(), idx.data_ptr() if by_index else None, S, n, D,
                                          ao.data_ptr(), xo.data_ptr(), _stream()), what)
            torch.cuda.synchronize()
            ri = idx if by_index else None
            assert _same(ao[:n], H.gather_rows_ref(a16, n, ri, S)), what + ": 16-bit rows"
            assert _same(xo[:n], H.gather_rows_ref(x32, n, ri, S)), what + ": fp32 rows"
            _untouched(ao, n, what)
            _untouched(xo, n, what)


# ------------------------------------------------------------------------------------------------------------------
# Position table
# ------------------------------------------------------------------------------------------------------------------
GRIDS = [(g, g) for g in range(1, 33)] + [(1, 32), (32, 1), (7, 8), (10, 15), (31, 17)]


def test_pos_interp_contract(L):
    """Every grid: the class row copied, the 7 x 7 grid the stored table bit for bit, every other value within
    gamma(8) sum |w||p| of the float64 sum with the kernel's fp32 weights."""
    g = torch.Generator().manual_seed(11)
    pos = torch.randn(50, 768, generator=g) * 0.02
    pos[3, 5], pos[40, 700] = 3.0, -2.5                                  # outliers reach many output rows
    pd = pos.to(DEV)
    for gh, gw in GRIDS:
        rows = 1 + gh * gw
        out = _guarded(rows, 768)
        what = f"pos_interp {gh}x{gw}"
        _check(L.plip_dbg_pos_interp(pd.data_ptr(), gh, gw, out.data_ptr(), _stream()), what)
        torch.cuda.synchronize()
        got = out.cpu()
        ref, slack = H.pos_interp_ref(pos, gh, gw)
        assert _same(got[0], pos[0]), what + ": class row"
        if (gh, gw) == (7, 7):
            assert _same(got[:rows], pos), what + ": the stored table"
        _within(got[1:rows], ref[1:], slack[1:], "position table (err / gamma(8) sum|w||p|)", what)
        _untouched(got, rows, what + " (guard rows)")


# ------------------------------------------------------------------------------------------------------------------
# Rejected arguments launch nothing
# ------------------------------------------------------------------------------------------------------------------
def _launches(L):
    return int(L.plip_launch_count())


def test_rejections_launch_nothing(L, tables):
    _fmt(L, 0)
    f = torch.zeros(64 * 768 + 16, device=DEV)
    h = torch.zeros(64 * 768 + 16, device=DEV, dtype=torch.bfloat16)
    i32 = torch.zeros(64 * 77 + 4, device=DEV, dtype=torch.int32)
    i64 = torch.zeros(64 * 77 + 4, device=DEV, dtype=torch.int64)
    u8 = torch.zeros(4 * 224 * 224 * 3 + 16, device=DEV, dtype=torch.uint8)
    tok, pos = tables
    F, F1, Hp, H2 = f.data_ptr(), f.data_ptr() + 4, h.data_ptr(), h.data_ptr() + 2
    s = _stream()
    calls = {
        "layernorm x misaligned": lambda: L.plip_dbg_layernorm_ex(F1, None, 768, 4, 768, F, F, F, None, s),
        "layernorm gamma misaligned": lambda: L.plip_dbg_layernorm_ex(F, None, 768, 4, 768, F1, F, F, None, s),
        "layernorm beta misaligned": lambda: L.plip_dbg_layernorm_ex(F, None, 768, 4, 768, F, F1, F, None, s),
        "layernorm out_f32 misaligned": lambda: L.plip_dbg_layernorm_ex(F, None, 768, 4, 768, F, F, F1, None, s),
        "layernorm out16 misaligned": lambda: L.plip_dbg_layernorm_ex(F, None, 768, 4, 768, F, F, None, H2, s),
        "layernorm null gamma": lambda: L.plip_dbg_layernorm_ex(F, None, 768, 4, 768, None, F, F, None, s),
        "layernorm stride": lambda: L.plip_dbg_layernorm_ex(F, None, 766, 4, 768, F, F, F, None, s),
        "layernorm rows": lambda: L.plip_dbg_layernorm_ex(F, None, 768, 0, 768, F, F, F, None, s),
        "layernorm dim": lambda: L.plip_dbg_layernorm_ex(F, None, 640, 4, 640, F, F, F, None, s),
        "rowstats x misaligned": lambda: L.plip_dbg_rowstats_cast(F1, 4, 768, Hp, F, s),
        "rowstats xb misaligned": lambda: L.plip_dbg_rowstats_cast(F, 4, 768, H2, F, s),
        "rowstats stats misaligned": lambda: L.plip_dbg_rowstats_cast(F, 4, 768, Hp, F1, s),
        "im2col 224 misaligned": lambda: L.plip_dbg_im2col_hw(u8.data_ptr() + 1, 2, 1, 224, 224, Hp, s),
        "im2col f32 off its element size": lambda: L.plip_dbg_im2col_hw(F + 2, 0, 1, 64, 64, Hp, s),
        "im2col out misaligned": lambda: L.plip_dbg_im2col_hw(F, 0, 1, 64, 64, H2, s),
        "im2col size": lambda: L.plip_dbg_im2col_hw(F, 0, 1, 31, 64, Hp, s),
        "im2col format": lambda: L.plip_dbg_im2col_hw(F, 3, 1, 64, 64, Hp, s),
        "text_embed tok misaligned": lambda: L.plip_dbg_text_embed(i32.data_ptr(), 0, 2, 77, 77, tok.data_ptr() + 4,
                                                                   pos.data_ptr(), F, i32.data_ptr(), 0, s),
        "text_embed ids misaligned": lambda: L.plip_dbg_text_embed(i64.data_ptr() + 4, 1, 2, 77, 77, tok.data_ptr(),
                                                                   pos.data_ptr(), F, i32.data_ptr(), 0, s),
        "text_embed stride": lambda: L.plip_dbg_text_embed(i32.data_ptr(), 0, 2, 77, 76, tok.data_ptr(),
                                                           pos.data_ptr(), F, i32.data_ptr(), 0, s),
        "text_embed dtype": lambda: L.plip_dbg_text_embed(i32.data_ptr(), 2, 2, 77, 77, tok.data_ptr(),
                                                          pos.data_ptr(), F, i32.data_ptr(), 0, s),
        "mask count": lambda: L.plip_dbg_mask_to_i32(i32.data_ptr(), 0, 0, 77, 77, i32.data_ptr(), s),
        "mask seq_len": lambda: L.plip_dbg_mask_to_i32(i32.data_ptr(), 0, 77, 0, 77, i32.data_ptr(), s),
        "mask stride": lambda: L.plip_dbg_mask_to_i32(i32.data_ptr(), 0, 154, 77, 76, i32.data_ptr(), s),
        "mask partial row": lambda: L.plip_dbg_mask_to_i32(i32.data_ptr(), 0, 100, 77, 77, i32.data_ptr(), s),
        "mask dtype": lambda: L.plip_dbg_mask_to_i32(i32.data_ptr(), 5, 77, 77, 77, i32.data_ptr(), s),
        "mask misaligned": lambda: L.plip_dbg_mask_to_i32(i64.data_ptr() + 4, 1, 77, 77, 77, i32.data_ptr(), s),
        "cls_rows n": lambda: L.plip_dbg_cls_rows(F, F, 0, 50, F, s),
        "cls_rows seq": lambda: L.plip_dbg_cls_rows(F, F, 1, 0, F, s),
        "cls_rows null": lambda: L.plip_dbg_cls_rows(None, F, 1, 50, F, s),
        "cls_rows cls misaligned": lambda: L.plip_dbg_cls_rows(F1, F, 1, 50, F, s),
        "cls_rows x misaligned": lambda: L.plip_dbg_cls_rows(F, F, 1, 50, F1, s),
        "gather_rows a16 misaligned": lambda: L.plip_dbg_gather_rows(H2, F, None, 1, 2, 768, Hp, F, s),
        "gather_rows x32 misaligned": lambda: L.plip_dbg_gather_rows(Hp, F1, None, 1, 2, 768, Hp, F, s),
        "gather_rows outputs misaligned": lambda: L.plip_dbg_gather_rows(Hp, F, None, 1, 2, 768, H2, F1, s),
        "gather_rows stride": lambda: L.plip_dbg_gather_rows(Hp, F, None, -1, 2, 768, Hp, F, s),
        "gather_rows dim": lambda: L.plip_dbg_gather_rows(Hp, F, None, 1, 2, 766, Hp, F, s),
    }
    torch.cuda.synchronize()
    snap = [t.clone() for t in (f, h, i32, i64, u8)]
    from plip_b200._lib import last_error
    for what, call in calls.items():
        count = _launches(L)
        assert call() != 0, what + ": accepted"
        assert last_error(), what + ": no error message"
        assert _launches(L) == count, what + ": launched a kernel"
    torch.cuda.synchronize()
    for a, b in zip((f, h, i32, i64, u8), snap):
        assert _same(a, b), "a refused call wrote memory"
