"""Kernel parity at the edges of the wgmma GEMM, the attention core and the fused top-k: later trips of the persistent
tile loops, tiles that start in the middle of the shared-memory ring, IEEE-half operands, strided operands, guard
bands around every output, slot boundaries and tile neighbours of the attention kernel, and the tie order of top-k.

Everything goes through the C ABI test hooks.  References are plain torch in float64, built from the same 16-bit
inputs the kernel reads, and acceptance is per element (no ulp-of-the-largest-value tolerances).

Constants of the kernels the shapes below are derived from (revisit the cases when one of them changes):
  gemm_wgmma.cu   BM = 128 rows per CTA tile, BK = 64, ring stages Cfg<BN>::STAGES = 4 (BN 256), 4 (BN 192), 6 (BN 128);
                  resident groups = #SMs / CG: 132 CTAs (CG 1) or at most 66 clusters (CG 2) on an H100 SXM
  attention.cu    128-row tiles, slot = 32 / 64 / 128 rows per sequence (G = 4 / 2 / 1 sequences per tile),
                  NK = 64 keys per warpgroup for slot <= 64 else 128; grid <= occupancy (3 resp. 2) x #SMs
  similarity.cu   one CTA per query when n m < 65536; tensor-core chunks of <= 32768 columns when n >= 256 and
                  m >= 8192; 64-column tiles split over gridDim.y CTAs otherwise
"""
import ctypes as C
import json
import math
import os

import pytest
import torch

from attention_oracle import (ATT_ABS, DT, OBSERVED, REL, SENT, U32, _bits, _note, _round_to,
                              assert_within, attention_contract_ref)
from similarity_oracle import similarity_refs, topk_check

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from plip_b200._lib import lib
    yield lib()
    path = os.environ.get("PLIP_EDGE_REPORT")
    if path and OBSERVED:
        with open(path, "w") as f:
            json.dump(OBSERVED, f, indent=1, sort_keys=True)


@pytest.fixture
def fmt_guard(L):
    """Lets a test switch the handle-free hooks to fp16 operands; bf16 is restored whatever happens."""
    def set_fmt(fmt):
        _check(L.plip_dbg_set_operand_format(fmt), "set_operand_format")
    try:
        yield set_fmt
    finally:
        L.plip_dbg_set_operand_format(0)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check(rc, what):
    from plip_b200._lib import check
    check(rc, what)


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _randn(shape, g, dev):
    return torch.randn(shape, generator=g, device=dev)


# ------------------------------------------------------------------------------------------------------------------
# References
# ------------------------------------------------------------------------------------------------------------------
def quick_gelu64(x):
    return x * torch.sigmoid(1.702 * x)


def gemm_ref(A, W, bias, epi, x0=None, pos=None, ln=None):
    """float64 result of plip_dbg_gemm's epilogue `epi` on the [M, N] problem, from the 16-bit operands as stored, and
    the absolute slack the kernel's fp32 arithmetic is entitled to.  Returns (ref, slack), both [M, N] float64.

      0 acc + bias            1 quick_gelu(acc + bias)      2 x0 + acc + bias      3 acc + pos[1 + row % 49]
      4 acc                   5 / 6  rstd (acc - mean colsum) + bias  (6: quick_gelu of it), ln = (s1, s2, colsum)
    (the scatter of 3 to rows b * 50 + 1 + p is left to the caller)

    Accumulation slack: the tensor core adds the 16 exact products of a k16 step to the fp32 accumulator with one
    rounding (or truncation: 2^-23 relative to the running sum) per step, K / 16 steps.  For operands with random
    signs the errors add like a random walk and the running sum stays far below sum_k |a_k w_k|, so
        |acc_kernel - acc| <= 2 x 2^-23 sqrt(K / 16) sum_k |a_k| |w_k|
    (the worst case, K / 16 instead of its root, needs same-signed products).  On an H100 the fp32-output cases
    below reach 0.31 of this bound, the factor 2 being the margin.  Every fp32 operation of the epilogue adds 2^-23
    of the magnitude of its operands."""
    A64, W64 = A.double(), W.double()
    K = A.shape[1]
    acc = A64 @ W64.t()
    slack = 2 * U32 * math.sqrt(K / 16) * (A64.abs() @ W64.abs().t())
    if epi == 4:
        return acc, slack
    if epi == 3:
        p = torch.arange(A.shape[0], device=A.device) % 49
        e = pos.double()[1 + p]
        return acc + e, slack + U32 * (acc.abs() + e.abs())
    b = bias.double()[None]
    if epi in (5, 6):
        s1, s2, colsum = (t.double() for t in ln)
        mean = s1 / K
        msq = s2 / K
        var = (msq - mean * mean).clamp_min(0.0)
        rstd = (var + 1e-5).rsqrt()
        t_acc, t_cs = rstd[:, None] * acc, (rstd * mean)[:, None] * colsum[None]
        pre = t_acc - t_cs + b
        # the kernel forms mean, var and rstd in fp32: var loses 2^-23 (E[x^2] + mean^2), rsqrtf is good to 2 ulp
        rstd_rel = 4 * U32 + U32 * (msq + mean * mean) / (var + 1e-5)
        slack = rstd[:, None] * slack + (4 * U32 + rstd_rel[:, None]) * (t_acc.abs() + t_cs.abs()) + U32 * b.abs()
    else:
        pre = acc + b
        slack = slack + U32 * (acc.abs() + b.abs())
    if epi == 2:
        x = x0.double()
        return x + pre, slack + U32 * (x.abs() + (x + pre).abs())
    if epi in (1, 6):
        # quick_gelu in the kernel is h + h tanh.approx(0.851 x), h = x / 2; tanh.approx is specified to 2^-11
        # relative, and |d quick_gelu / dx| <= 1.1 carries the slack of the argument through
        half_t = (0.5 * pre * torch.tanh(0.851 * pre)).abs()
        return quick_gelu64(pre), 1.1 * slack + 2.0 ** -11 * half_t + 2 * U32 * pre.abs()
    return pre, slack


def test_references_against_torch_functional():
    """The float64 helpers agree with torch.nn.functional on small inputs (runs without a GPU)."""
    F = torch.nn.functional
    g = torch.Generator().manual_seed(1)
    M, N, K = 98, 128, 192
    A = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16)
    W = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    bias, x0, pos = torch.randn(N, generator=g), torch.randn(M, N, generator=g), torch.randn(50, N, generator=g)
    lin = F.linear(A.double(), W.double(), bias.double())
    for epi, want in ((0, lin), (1, lin * torch.sigmoid(1.702 * lin)), (2, x0.double() + lin),
                      (3, F.linear(A.double(), W.double()) + pos.double()[1:].repeat(2, 1)),
                      (4, F.linear(A.double(), W.double()))):
        ref, slack = gemm_ref(A, W, bias, epi, x0=x0, pos=pos)
        assert torch.allclose(ref, want, rtol=1e-12, atol=1e-12), epi
        assert (slack > 0).all() and slack.max().item() < 1e-2, epi
    # LayerNorm fold: with exact statistics and an unrounded folded weight it is LayerNorm -> linear
    x = (torch.randn(M, K, generator=g) * 1.5 + 0.4).double()
    gam, bet = 1 + 0.1 * torch.randn(K, generator=g).double(), 0.05 * torch.randn(K, generator=g).double()
    Wd = W.double()
    Wf = Wd * gam[None]
    ln = (x.sum(-1), (x * x).sum(-1), Wf.sum(1))
    want = F.linear(F.layer_norm(x, (K,), gam, bet, 1e-5), Wd, bias.double())
    ref, _ = gemm_ref(x, Wf, bias.double() + Wd @ bet, 5, ln=ln)
    assert torch.allclose(ref, want, rtol=1e-9, atol=1e-9)
    ref, _ = gemm_ref(x, Wf, bias.double() + Wd @ bet, 6, ln=ln)
    assert torch.allclose(ref, want * torch.sigmoid(1.702 * want), rtol=1e-9, atol=1e-9)

    for fmt in (0, 1):
        for n_seq, S, heads, causal, use_mask in ((3, 20, 2, True, True), (2, 33, 1, False, True), (2, 7, 2, True, False)):
            qkv = torch.randn(n_seq * S, 3 * heads * 64, generator=g).to(DT[fmt])
            mask = None
            bias_mask = torch.zeros(n_seq, 1, S, S, dtype=torch.float64)
            if use_mask:
                lens = torch.randint(1, S + 1, (n_seq,), generator=g)
                mask = (torch.arange(S)[None] < lens[:, None]).to(torch.int32)
                bias_mask = bias_mask.masked_fill((mask == 0)[:, None, None, :], float("-inf"))
            if causal:
                bias_mask = bias_mask + torch.full((S, S), float("-inf"), dtype=torch.float64).triu(1)
            contract, plain, flip = attention_contract_ref(qkv, n_seq, S, heads, causal, mask, fmt)
            q, k, v = qkv.double().view(n_seq, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
            want = F.scaled_dot_product_attention(q, k, v, attn_mask=bias_mask, scale=1.0)
            want = want.permute(0, 2, 1, 3).reshape(n_seq * S, heads * 64)
            assert torch.allclose(plain, want, rtol=1e-10, atol=1e-12)
            # rounding p moves the output by at most one ulp of the weights times |v|
            assert ((contract - plain).abs() <= REL[fmt] * 0.5 * 1.01 * v.abs().amax()).all()
            assert (flip >= 0).all() and torch.isfinite(flip).all()


def test_long_and_probs_references_against_torch_functional(monkeypatch):
    """The block-wise references of the long and the probabilities kernel against torch.nn.functional and against
    the one-block reference (runs without a GPU)."""
    import attention_oracle as AO
    F = torch.nn.functional
    g = torch.Generator().manual_seed(2)
    for fmt in (0, 1):
        for n_seq, S, heads in ((2, 7, 2), (1, 64, 2), (2, 65, 1), (2, 129, 2), (1, 200, 1)):
            qkv = torch.randn(n_seq * S, 3 * heads * 64, generator=g).to(DT[fmt])
            q, k, v = qkv.double().view(n_seq, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
            want = F.scaled_dot_product_attention(q, k, v, scale=1.0).permute(0, 2, 1, 3).reshape(n_seq * S, heads * 64)
            contract, plain, flip = AO.long_attention_contract_ref(qkv, n_seq, S, heads, fmt)
            assert torch.allclose(plain, want, rtol=0, atol=1e-10)
            assert ((contract - plain).abs() <= REL[fmt] * 0.5 * 1.01 * v.abs().amax()).all()
            assert (flip >= 0).all() and torch.isfinite(flip).all()
            if S <= 64:                                       # one block: the short kernel's contract, bit for bit
                short = attention_contract_ref(qkv, n_seq, S, heads, False, None, fmt)
                assert torch.equal(contract, short[0]) and torch.equal(flip, short[2])
            elif fmt == 0:                                    # rounded against m_b, not against the final maximum
                assert not torch.equal(contract, attention_contract_ref(qkv, n_seq, S, heads, False, None, fmt)[0])
            slack = AO.long_chain_slack(qkv, n_seq, S, heads)
            assert (slack > 0).all() == (S > 64) and slack.max().item() < 1e-4
            with monkeypatch.context() as mp:                 # rounding taken out: the block weights are exact
                mp.setattr(AO, "_round_to", lambda x64, dt: x64)
                assert torch.allclose(AO.long_attention_contract_ref(qkv, n_seq, S, heads, fmt)[0], want, rtol=0, atol=1e-10)
            for causal, use_mask in ((False, False), (True, False), (True, True)):
                mask = None
                bias_mask = torch.zeros(n_seq, 1, S, S, dtype=torch.float64)
                if use_mask:
                    mask = (torch.rand(n_seq, S, generator=g) > 0.3).to(torch.int32)
                    mask[:, 0] = 1
                    bias_mask = bias_mask.masked_fill((mask == 0)[:, None, None, :], float("-inf"))
                if causal:
                    bias_mask = bias_mask + torch.full((S, S), float("-inf"), dtype=torch.float64).triu(1)
                probs, rel = AO.probs_contract_ref(qkv, n_seq, S, heads, causal, mask)
                want_p = torch.softmax(q @ k.transpose(-1, -2) + bias_mask, -1)
                assert torch.allclose(probs, want_p, rtol=0, atol=1e-12)
                assert torch.equal(rel > 0, want_p > 0) and rel.max().item() < 1e-3
    # a row whose first block holds no visible key: no rescale link before its first key, probabilities from there on
    S = 150
    s = torch.full((1, S, S), float("-inf"), dtype=torch.float64)
    s[0, :, 100:] = torch.linspace(0.0, 5.0, 50, dtype=torch.float64)
    m_key, m_last, chain = AO.running_block_max(s)
    assert torch.isinf(m_key[..., :64]).all() and (m_key[..., 64:128] == s[..., 127:128]).all()
    assert (m_key[..., 128:] == 5.0).all() and (m_last == 5.0).all()
    assert torch.allclose(chain, torch.full_like(chain, 2.0 ** -24 * 5.0 + 3 * U32), rtol=1e-12, atol=0)


# ------------------------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------------------------
def assert_guards(buf, before, rows, cols, what, keep_rows=None):
    """Everything of `buf` outside [:rows, :cols] (pad columns, guard rows) — and, with keep_rows, those rows of the
    payload as well — still holds the bits it held before the launch."""
    a, b = _bits(buf).clone(), _bits(before).clone()
    payload = torch.ones(rows, dtype=torch.bool, device=buf.device)
    if keep_rows is not None:
        payload[keep_rows] = False
    a[:rows, :cols][payload] = 0
    b[:rows, :cols][payload] = 0
    diff = a != b
    assert not diff.any(), f"{what}: stray write at (row, col) {diff.nonzero()[0].tolist()}, {int(diff.sum())} elements changed"


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tile_of(cg, bn, N):
    def where(r, c):
        nb = N // bn
        t = (r // (128 * cg)) * nb + c // bn
        return (f"tile {t} (m-block {r // 128}, n-block {c // bn}, cta rank {(r // 128) % cg}), "
                f"trip {t // max(1, _sm_count() // cg)} of its group if all groups are resident, "
                f"warp {(r % 128) // 16} row {r % 16} of the tile")
    return where


def _operands(M, N, K, lda, ldw, fmt, g, dev, wide):
    """A [M, K] and W [N, K] as views into [rows, ld] buffers whose pad columns hold a value that would wreck the
    result if the kernel read it.  `wide` scales one k-block of A so results reach ~1e3 (fp16: spacing 0.5)."""
    dt = DT[fmt]
    Ab = torch.full((M, lda), 1000.0, device=dev, dtype=dt)
    Wb = torch.full((N, ldw), 1000.0, device=dev, dtype=dt)
    a = _randn((M, K), g, dev) * 0.5
    if wide:
        a[:, :64] *= 300.0
    Ab[:, :K] = a.to(dt)
    Wb[:, :K] = (_randn((N, K), g, dev) * 0.05).to(dt)
    return Ab, Wb


def run_gemm(L, cg, bn, epi, M, N, K, fmt=0, lda=None, ldw=None, ldo=None, emit=False, wide=False, key=None):
    """One launch of epilogue 0 / 1 / 2 / 3 / 4 into guarded buffers; parity per element, guards bit-unchanged."""
    dev = "cuda"
    lda, ldw, ldo = lda or K, ldw or K, ldo or N
    g = _gen(dev, M * 7 + N + K + epi + 13 * fmt)
    Ab, Wb = _operands(M, N, K, lda, ldw, fmt, g, dev, wide)
    A, W = Ab[:, :K], Wb[:, :K]
    bias = _randn((N,), g, dev) * (30.0 if wide else 1.0)
    pos = _randn((50, N), g, dev) if epi == 3 else None
    out_dt = DT[fmt] if epi in (0, 1) else torch.float32
    out_rows = M // 49 * 50 if epi == 3 else M
    out = torch.full((out_rows + 8, ldo), SENT, device=dev, dtype=out_dt)
    x0 = None
    if epi == 2:
        x0 = _randn((M, N), g, dev)
        out[:M, :N] = x0
    xb = stats = None
    if emit:
        xb = torch.full((M + 8, ldo), SENT, device=dev, dtype=DT[fmt])
        stats = torch.full((M + 8, 8, 2), SENT, device=dev)
    before = out.clone()
    _check(L.plip_dbg_gemm(Ab.data_ptr(), lda, Wb.data_ptr(), ldw, M, N, K, bias.data_ptr(), out.data_ptr(), ldo,
                           pos.data_ptr() if pos is not None else None, epi, cg, bn, None, None, 0,
                           xb.data_ptr() if emit else None, stats.data_ptr() if emit else None, _stream()), "gemm")
    torch.cuda.synchronize()
    ref, slack = gemm_ref(A, W, bias, epi, x0=x0, pos=pos)
    what = f"gemm cg={cg} bn={bn} epi={epi} M={M} N={N} K={K} fmt={fmt} ld=({lda},{ldw},{ldo})"
    key = key or f"gemm epi {epi} {'bf16' if fmt == 0 else 'fp16'} operands"
    rel = REL[fmt] if epi in (0, 1) else 0.0
    eff_bn = bn if N % bn == 0 else 128
    if epi == 3:
        nb = M // 49
        got = out[:nb * 50].view(nb, 50, ldo)[:, 1:, :N].reshape(M, N)
        assert_within(got, ref, slack, rel, key, what, _tile_of(cg, eff_bn, N))
        cls_rows = torch.arange(0, nb * 50, 50, device=dev)
        assert_guards(out, before, nb * 50, N, what + " (class rows, pad columns, guard rows)", keep_rows=cls_rows)
        return
    assert_within(out[:M, :N], ref, slack, rel, key, what, _tile_of(cg, eff_bn, N))
    assert_guards(out, before, M, N, what + " (pad columns, guard rows)")
    if emit:
        x = out[:M, :N]
        assert torch.equal(xb[:M, :N], x.to(DT[fmt])), what + ": xb_out is not the 16-bit cast of the updated rows"
        assert_guards(xb, torch.full_like(xb, SENT), M, N, what + " (xb_out)")
        npart = 2 * (N // eff_bn)                              # one slot per (N tile, half of the tile's columns)
        x64 = x.double()
        s = stats[:M, :npart].double().sum(1)
        # each slot is an fp32 sum of <= 128 values: 2^-23 sqrt(128) of the absolute sum is a wide bound
        tol1 = U32 * math.sqrt(128) * x64.abs().sum(-1) + 1e-6
        tol2 = U32 * math.sqrt(128) * (x64 * x64).sum(-1) + 1e-6
        e1, e2 = (s[:, 0] - x64.sum(-1)).abs(), (s[:, 1] - (x64 * x64).sum(-1)).abs()
        assert (e1 <= tol1).all() and (e2 <= tol2).all(), (what, (e1 / tol1).max().item(), (e2 / tol2).max().item())
        _note("row statistics (sum, sum of squares)", max((e1 / tol1).max().item(), (e2 / tol2).max().item()))
        sb = torch.full_like(stats, SENT)
        sb[:M, :npart] = stats[:M, :npart]
        assert torch.equal(_bits(stats), _bits(sb)), what + ": statistics slots >= npart or guard rows were written"


# M = 8192 + 37 = 65 row blocks.  CG 2: 33 clusters per column of tiles, the second CTA of the last one owns rows
# 8320.. only (past M: zero fill, nothing stored).  Tiles / resident groups at N = 2304:
#   (1,256) 65 x 9 = 585 / 132     (2,256) 33 x 9 = 297 / <=66     (2,192) 33 x 12 = 396 / <=66
#   (1,128) 65 x 18 = 1170 / 132   (2,128) 33 x 18 = 594 / <=66    -> 4.4 to 9 trips per group
M_PERSIST = 8192 + 37
CONFIGS = [(1, 256), (2, 256), (2, 192), (1, 128), (2, 128)]


FP16_CONFIGS = [(2, 256), (2, 192), (1, 128)]                  # fp16 operands: one configuration per BN


@gpu
@pytest.mark.parametrize("cg,bn,epi,fmt", [(cg, bn, epi, fmt) for fmt, cfgs in ((0, CONFIGS), (1, FP16_CONFIGS))
                                           for cg, bn in cfgs for epi in (0, 1)])
def test_gemm_persistent_16bit_store(L, fmt_guard, cg, bn, epi, fmt):
    """Second and later tiles of the TMA-store epilogue: stage_sel carried across tiles, two staging boxes per warp."""
    fmt_guard(fmt)
    run_gemm(L, cg, bn, epi, M_PERSIST, 2304, 768, fmt=fmt, wide=(fmt == 1))


# Residual epilogue with the bf16 copy and row statistics.  M = 16384 + 37 = 129 row blocks (65 clusters, the last one
# half empty), K = 320 = 5 k-blocks (not a multiple of 4 or 6 stages: tiles start mid-ring as well).
#   N 768: BN 256 -> 3 tiles per row block, 6 slots; BN 192 -> 4, 8 slots (BN 128 would need 12 > 8: rejected)
#   N 512: BN 256 -> 2, 4 slots; BN 128 -> 4, 8 slots.   Fewest tiles: (2,256) at N 512, 130 clusters / <= 66.
@gpu
@pytest.mark.parametrize("cg,bn,N,fmt", [(1, 256, 768, 0), (2, 256, 768, 0), (2, 192, 768, 0), (2, 256, 512, 0),
                                         (1, 128, 512, 0), (2, 128, 512, 0), (2, 192, 768, 1), (2, 128, 512, 1)])
def test_gemm_persistent_residual_with_statistics(L, fmt_guard, cg, bn, N, fmt):
    fmt_guard(fmt)
    run_gemm(L, cg, bn, 2, 16384 + 37, N, 320, fmt=fmt, emit=True)


# Patch scatter: 200 images x 49 patches = 9800 rows = 77 row blocks, K = 3072 = 48 k-blocks.
#   (2,256): 39 clusters x 3 = 117 / <= 66        (1,128): 77 x 6 = 462 / 132
@gpu
@pytest.mark.parametrize("cg,bn", [(2, 256), (1, 128)])
def test_gemm_persistent_patch_scatter(L, cg, bn):
    run_gemm(L, cg, bn, 3, 49 * 200, 768, 3072)


# Ring carry-over: 3, 5, 7, 13 k-blocks, never a multiple of the stage count (4, 4, 6), so the 2nd, 3rd, ... tile of a
# CTA enters the ring at slot (i k) mod STAGES != 0 and the barrier phase flips inside a tile.
# M = 8357 = 66 row blocks (33 clusters, the last CTA has 37 rows), N = 1536 = 6 x 256 = 8 x 192 = 12 x 128:
#   (1,256) 396 / 132 = 3 trips   (2,256) 198 / <=66 = 3   (2,192) 264 / <=66 = 4   (1,128) 792 / 132   (2,128) 396 / <=66
@gpu
@pytest.mark.parametrize("cg,bn,K,epi,fmt", [(cg, bn, K, epi, fmt) for fmt, Ks in ((0, (192, 320, 448, 832)), (1, (320,)))
                                             for cg, bn in CONFIGS for K in Ks for epi in (4, 0)])
def test_gemm_ring_carry_over(L, fmt_guard, cg, bn, K, epi, fmt):
    fmt_guard(fmt)
    run_gemm(L, cg, bn, epi, 8357, 1536, K, fmt=fmt, wide=(fmt == 1 and epi == 0))


@gpu
@pytest.mark.parametrize("cg,bn,epi,ldo", [(cg, bn, epi, ldo) for cg, bn in ((2, 256), (1, 128))
                                           for epi, ldo in ((0, 768 + 8), (0, 768 + 128), (2, 768 + 8), (4, 768 + 8), (4, 768 + 128))
                                           if not (epi == 2 and bn == 128)])      # statistics at N 768 need BN >= 192
def test_gemm_strided_operands(L, cg, bn, epi, ldo):
    """lda, ldw, ldo larger than the logical widths: pad columns are neither read nor written."""
    run_gemm(L, cg, bn, epi, 1000, 768, 320, lda=320 + 8, ldw=320 + 8, ldo=ldo, emit=(epi == 2))


@gpu
@pytest.mark.parametrize("epi", [0, 4])
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("M", [1, 63, 64, 65, 127, 128, 129, 255, 257])
def test_gemm_small_m_under_clusters(L, M, bn, epi):
    """CG 2 with one to three row blocks: the peer CTA is empty, half full or holds a single row."""
    run_gemm(L, 2, bn, epi, M, 256, 128)


def _ln_inputs(M, D, N, fmt, dev):
    g = _gen(dev, D + N + fmt)
    x = _randn((M, D), g, dev) * 1.5 + 0.4
    gam = 1 + 0.1 * _randn((D,), g, dev)
    bet = 0.05 * _randn((D,), g, dev)
    W = _randn((N, D), g, dev) * 0.05
    bias = _randn((N,), g, dev) * 0.1
    return x, gam, bet, W, bias


# LayerNorm fold at M = 8229 (see M_PERSIST), D = 768 -> N = 2304 (epilogue 5) and 3072 (6): ln_row_terms re-read for
# every tile of the persistent loop.  Tiles at N = 3072: (2,256) 33 x 12 = 396, (2,192) 33 x 16, (1,128) 65 x 24.
@gpu
@pytest.mark.parametrize("epi,N", [(5, 2304), (6, 3072)])
@pytest.mark.parametrize("cg,bn", [(2, 256), (2, 192), (1, 128)])
def test_gemm_persistent_layernorm_fold(L, cg, bn, epi, N):
    dev, M, D, fmt = "cuda", M_PERSIST, 768, 0
    x, gam, bet, W, bias = _ln_inputs(M, D, N, fmt, dev)
    xb = torch.zeros(M, D, device=dev, dtype=DT[fmt])
    stats = torch.full((M, 8, 2), float("nan"), device=dev)    # only slot 0 is valid: n_partials = 1
    _check(L.plip_dbg_rowstats_cast(x.data_ptr(), M, D, xb.data_ptr(), stats.data_ptr(), _stream()), "rowstats")
    torch.cuda.synchronize()
    assert torch.equal(xb, x.to(DT[fmt]))
    x64 = x.double()
    s1, s2 = stats[:, 0, 0].double(), stats[:, 0, 1].double()
    assert ((s1 - x64.sum(-1)).abs() <= U32 * math.sqrt(D) * x64.abs().sum(-1)).all()
    assert ((s2 - (x64 * x64).sum(-1)).abs() <= U32 * math.sqrt(D) * (x64 * x64).sum(-1)).all()
    assert torch.isnan(stats[:, 1:]).all()
    Wf = (W * gam[None]).to(DT[fmt])
    colsum = Wf.float().sum(1).contiguous()
    biasf = (bias + W @ bet).contiguous()
    out = torch.full((M + 8, N), SENT, device=dev, dtype=DT[fmt])
    before = out.clone()
    _check(L.plip_dbg_gemm(xb.data_ptr(), D, Wf.data_ptr(), D, M, N, D, biasf.data_ptr(), out.data_ptr(), N, None, epi,
                           cg, bn, colsum.data_ptr(), stats.data_ptr(), 1, None, None, _stream()), "ln gemm")
    torch.cuda.synchronize()
    what = f"ln-fold gemm cg={cg} bn={bn} epi={epi} M={M} N={N}"
    # (a) the fold identity from the SAME 16-bit operands and statistics: isolates the kernel from the fold's own
    #     cancellation and from the rounding of x and gamma o W
    ref, slack = gemm_ref(xb, Wf, biasf, epi, ln=(stats[:, 0, 0], stats[:, 0, 1], colsum))
    assert_within(out[:M], ref, slack, REL[fmt], "gemm LayerNorm fold vs fold identity", what, _tile_of(cg, bn, N))
    assert_guards(out, before, M, N, what + " (guard rows)")
    # (b) LayerNorm -> linear in float64 from the unrounded inputs: bounds of the existing chain test
    full = torch.nn.functional.layer_norm(x64, (D,), gam.double(), bet.double(), 1e-5) @ W.double().t() + bias.double()
    if epi == 6:
        full = quick_gelu64(full)
    err = (out[:M].double() - full).abs()
    assert err.max().item() < 0.06 and err.mean().item() < 6e-3, (what, err.max().item(), err.mean().item())
    _note("gemm LayerNorm fold vs float64 LayerNorm -> linear (max abs err / 0.06)", err.max().item() / 0.06)


@gpu
def test_gemm_rejections_launch_nothing(L):
    from plip_b200._lib import last_error
    dev = "cuda"
    M, N, K = 256, 768, 128
    A = torch.zeros(M + 1, K, device=dev, dtype=torch.bfloat16)
    W = torch.zeros(N, K, device=dev, dtype=torch.bfloat16)
    bias = torch.zeros(N, device=dev)
    out = torch.full((M, N + 8), SENT, device=dev)
    out16 = torch.full((M, N), SENT, device=dev, dtype=torch.bfloat16)
    xb = torch.full((M, N), SENT, device=dev, dtype=torch.bfloat16)
    stats = torch.full((M, 8, 2), SENT, device=dev)

    def call(a_ptr=None, ldo=N, epi=4, cg=0, bn=0, colsum=None, stats_in=None, npart=0, emit=False, o=None):
        o = out if o is None else o
        return L.plip_dbg_gemm(a_ptr or A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(), o.data_ptr(), ldo, None,
                               epi, cg, bn, colsum, stats_in, npart, xb.data_ptr() if emit else None,
                               stats.data_ptr() if emit else None, _stream())

    for kw, fragment in ((dict(cg=1, bn=192), "bad config"),
                         (dict(ldo=N + 4), "multiples of 8"),
                         (dict(a_ptr=A.data_ptr() + 2), "16-byte aligned"),
                         (dict(epi=2, bn=128, emit=True), "statistics slots"),     # 2 x 768 / 128 = 12 slots > 8
                         (dict(epi=5, stats_in=stats.data_ptr(), npart=1, o=out16), "needs colsum"),
                         (dict(epi=5, colsum=bias.data_ptr(), stats_in=stats.data_ptr(), npart=9, o=out16), "partials")):
        assert call(**kw) != 0, kw
        assert fragment in last_error(), (kw, last_error())
    torch.cuda.synchronize()
    for t in (out, out16, xb, stats):
        assert (t == SENT).all()


# ------------------------------------------------------------------------------------------------------------------
# Attention
# ------------------------------------------------------------------------------------------------------------------
PLAIN_BOUNDS = {0: (0.03, 2e-3), 1: (6e-3, 4e-4)}   # (max, mean) |out - softmax(s) v| for N(0,1) inputs: P rounding


def _ragged_mask(n_seq, S, g, dev, holes=False):
    """Key padding mask [n_seq, S] int32: visible prefix of 1..S keys (key 0 always visible), optionally with holes."""
    lens = torch.randint(1, S + 1, (n_seq,), generator=g, device=dev)
    lens[0] = 1                                                # the shortest and the longest prefix always occur
    lens[-1] = S
    mask = torch.arange(S, device=dev)[None] < lens[:, None]
    if holes:
        mask &= torch.rand(n_seq, S, generator=g, device=dev) > 0.3
        mask[:, 0] = True
    return mask.to(torch.int32).contiguous()


def run_attention(L, qkv, n_seq, S, heads, causal, mask, fmt):
    D = heads * 64
    out = torch.full((n_seq * S + 8, D), SENT, device=qkv.device, dtype=DT[fmt])
    _check(L.plip_dbg_attention(qkv.data_ptr(), n_seq, S, heads, int(causal),
                                mask.data_ptr() if mask is not None else None, out.data_ptr(), _stream()), "attention")
    torch.cuda.synchronize()
    assert (out[n_seq * S:] == SENT).all(), "attention wrote past the last sequence"
    return out[:n_seq * S]


def check_attention(L, n_seq, S, heads, causal, mask_kind, fmt, seed=0, key=None):
    dev = "cuda"
    D = heads * 64
    g = _gen(dev, n_seq * 131 + S + seed)
    qkv = _randn((n_seq * S, 3 * D), g, dev).to(DT[fmt])
    mask = None if mask_kind is None else _ragged_mask(n_seq, S, g, dev, holes=(mask_kind == "holes"))
    out = run_attention(L, qkv, n_seq, S, heads, causal, mask, fmt)
    contract, plain, flip = attention_contract_ref(qkv, n_seq, S, heads, causal, mask, fmt)
    G = 128 // (32 if S <= 32 else 64 if S <= 64 else 128)

    def where(r, c):
        seq, h = r // S, c // 64
        tile = (seq // G) * heads + h
        return f"sequence {seq} (position {seq % G} of its tile) row {r % S} head {h} dim {c % 64}; tile {tile}"
    what = f"attention n_seq={n_seq} S={S} heads={heads} causal={causal} mask={mask_kind} fmt={fmt}"
    assert_within(out, contract, ATT_ABS + flip, REL[fmt], key or f"attention vs contract ({'bf16' if fmt == 0 else 'fp16'})",
                  what, where)
    err = (out.double() - plain).abs()
    mx, mean = PLAIN_BOUNDS[fmt]
    assert err.max().item() < mx and err.mean().item() < mean, (what, err.max().item(), err.mean().item())
    _note(f"attention vs plain softmax ({'bf16' if fmt == 0 else 'fp16'}, max abs err / {mx})", err.max().item() / mx)
    return qkv, mask, out


# Tiles (= ceil(n_seq / G) x heads) against a grid of at most 3 x 132 = 396 CTAs (NK 64) or 2 x 132 = 264 (NK 128):
#   (1024, 50, 12): 512 x 12 = 6144     (1024, 77, 8): 1024 x 8 = 8192 (NK 128)
#   (700, 20, 8):   175 x 8 = 1400      (300, 128, 8): 300 x 8 = 2400 (NK 128)        -> 3.5 to 31 trips per CTA
@gpu
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("n_seq,S,heads,causal,mask_kind", [(1024, 50, 12, False, None), (1024, 77, 8, True, "ragged"),
                                                            (700, 20, 8, True, "ragged"), (300, 128, 8, True, None)])
def test_attention_persistent(L, fmt_guard, n_seq, S, heads, causal, mask_kind, fmt):
    """Later trips of the tile loop: barrier parity it & 1, Q buffer refilled after it staged the output."""
    fmt_guard(fmt)
    check_attention(L, n_seq, S, heads, causal, mask_kind, fmt)


@gpu
@pytest.mark.parametrize("mask_kind", [None, "ragged"])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("S", [1, 2, 31, 32, 33, 63, 64, 65, 127, 128])
def test_attention_slot_edges(L, S, causal, mask_kind):
    """Both sides of the 32 / 64 / 128 slot choice (and of NK 64 / 128), with full, short and over-full last tiles."""
    G = 128 // (32 if S <= 32 else 64 if S <= 64 else 128)
    for n_seq in sorted({1, G - 1, G, G + 1, 4 * G + 3} - {0}):
        check_attention(L, n_seq, S, 3, causal, mask_kind, 0, key="attention vs contract (bf16)")


@gpu
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("S,causal", [(20, True), (50, False), (77, True), (128, False)])
def test_attention_mask_shapes(L, fmt_guard, S, causal, fmt):
    """Visible prefixes down to one key, holes inside the prefix, and two masks that must change nothing.
    (A query row without any visible key is outside this test: the kernel returns zeros for it, a float softmax NaN.)"""
    fmt_guard(fmt)
    n_seq, heads = 37, 4
    qkv, _, _ = check_attention(L, n_seq, S, heads, causal, "holes", fmt)
    qkv1, mask1, _ = check_attention(L, n_seq, S, heads, causal, "ragged", fmt, seed=1)
    assert mask1.sum(1).min().item() == 1
    plain = run_attention(L, qkv, n_seq, S, heads, causal, None, fmt)
    ones = torch.ones(n_seq, S, device="cuda", dtype=torch.int32)
    assert torch.equal(run_attention(L, qkv, n_seq, S, heads, causal, ones, fmt), plain), "all-ones mask != no mask"
    if causal:
        # keys from `cut` on are hidden: rows before `cut` never looked at them
        cut = torch.randint(1, S + 1, (n_seq,), generator=_gen("cuda", S), device="cuda")
        m = (torch.arange(S, device="cuda")[None] < cut[:, None]).to(torch.int32).contiguous()
        got = run_attention(L, qkv, n_seq, S, heads, True, m, fmt).view(n_seq, S, -1)
        rows_before = torch.arange(S, device="cuda")[None] < cut[:, None]
        assert torch.equal(got[rows_before], plain.view(n_seq, S, -1)[rows_before]), "a mask behind the causal limit changed a row"


@gpu
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("S,causal,use_mask", [(20, True, True), (32, False, False), (50, False, False), (64, True, True),
                                               (77, True, True), (100, False, False)])
def test_attention_neighbour_independence(L, fmt_guard, S, causal, use_mask, fmt):
    """Sequences share a 128-row tile (and, through the slot-sized TMA box, see the rows of the next sequences) and
    are separated by masking alone: a sequence's output may not depend on what the others hold."""
    fmt_guard(fmt)
    dev, heads = "cuda", 4
    G = 128 // (32 if S <= 32 else 64 if S <= 64 else 128)
    n_seq = 6 * G + 1
    g = _gen(dev, S)
    qkv = _randn((n_seq * S, 3 * heads * 64), g, dev).to(DT[fmt])
    mask = _ragged_mask(n_seq, S, g, dev) if use_mask else None
    base = run_attention(L, qkv, n_seq, S, heads, causal, mask, fmt).view(n_seq, S, -1)
    seq = torch.arange(n_seq, device=dev)
    for pos in range(max(G, 2)):
        keep = (seq % max(G, 2)) == pos                        # G = 1: every other sequence (its box neighbours)
        poisoned = qkv.clone().view(n_seq, S, -1)
        sign = torch.where(torch.rand(poisoned.shape, generator=g, device=dev) < 0.5, -1.0, 1.0).to(DT[fmt])
        poisoned[~keep] = (3e4 * sign)[~keep]
        got = run_attention(L, poisoned.view(n_seq * S, -1), n_seq, S, heads, causal, mask, fmt).view(n_seq, S, -1)
        assert torch.equal(got[keep], base[keep]), f"S={S} position {pos}: output depends on the tile neighbours"


@gpu
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("S,causal", [(50, False), (77, True), (128, True)])
def test_attention_peaked_and_flat_softmax(L, fmt_guard, S, causal, fmt):
    fmt_guard(fmt)
    dev, heads, n_seq = "cuda", 4, 9
    D = heads * 64
    g = _gen(dev, 3 * S + fmt)
    # flat: q = 0 -> every visible key weighs 1 / count exactly (p = 1, representable), output = mean of visible v
    qkv = _randn((n_seq * S, 3 * D), g, dev).to(DT[fmt])
    qkv[:, :D] = 0
    mask = _ragged_mask(n_seq, S, g, dev, holes=True)
    out = run_attention(L, qkv, n_seq, S, heads, causal, mask, fmt)
    vis = (mask != 0)[:, None, :].expand(n_seq, S, S)
    if causal:
        vis = vis & torch.ones(S, S, device=dev, dtype=torch.bool).tril()[None]
    w = vis.double() / vis.double().sum(-1, keepdim=True)
    v = qkv[:, 2 * D:].double().view(n_seq, S, D)
    mean_v = (w @ v).view(n_seq * S, D)
    slack = 8 * U32 * (w @ v.abs()).view(n_seq * S, D)        # fp32 sum of <= 128 terms, 1 / count, product
    assert_within(out, mean_v, slack, REL[fmt], "attention flat softmax (mean of visible V)", f"flat S={S} fmt={fmt}")
    # peaked: unit-norm keys, q = 80 k_target: the target scores 80, every other key at most ~ +-30, so its weight
    # is 1 to within e^-50 and ex2 sees arguments down to -230 (flushed to zero): output = v_target
    k = _randn((n_seq, S, heads, 64), g, dev).double()
    k = _round_to(k / k.norm(dim=-1, keepdim=True), DT[fmt])
    tgt = torch.randint(0, S, (n_seq, S), generator=g, device=dev)
    if causal:
        tgt = torch.minimum(tgt, torch.arange(S, device=dev)[None])
    q = 80.0 * torch.gather(k, 1, tgt[:, :, None, None].expand(n_seq, S, heads, 64))
    vv = _randn((n_seq, S, heads, 64), g, dev)
    qkv = torch.stack([q.float(), k.float(), vv], 2).reshape(n_seq * S, 3 * D).to(DT[fmt])
    out = run_attention(L, qkv, n_seq, S, heads, causal, None, fmt)
    contract, plain, flip = attention_contract_ref(qkv, n_seq, S, heads, causal, None, fmt)
    assert_within(out, contract, ATT_ABS + flip, REL[fmt], "attention peaked softmax vs contract", f"peaked S={S} fmt={fmt}")
    qs = qkv[:, :D].double().view(n_seq, S, heads, 64)
    ks = qkv[:, D:2 * D].double().view(n_seq, S, heads, 64)
    sc = torch.einsum("nihd,njhd->nhij", qs, ks)
    assert (sc.amax(-1) - sc.gather(-1, tgt[:, None, :, None].expand(n_seq, heads, S, 1))[..., 0]).abs().max().item() < 1e-9
    v_t = torch.gather(qkv[:, 2 * D:].double().view(n_seq, S, heads, 64), 1, tgt[:, :, None, None].expand(n_seq, S, heads, 64))
    second = sc.masked_fill(torch.nn.functional.one_hot(tgt, S).bool()[:, None], float("-inf"))
    if causal:
        second = second.masked_fill(torch.ones(S, S, device=dev, dtype=torch.bool).triu(1), float("-inf"))
    gap = (sc.amax(-1) - second.amax(-1)).clamp_max(745.0)     # S = 1-key rows: gap = inf
    leak = (S * torch.exp(-gap) * 6.0).permute(0, 2, 1)[..., None].expand(n_seq, S, heads, 64)   # |v| < 6
    assert_within(out, v_t.reshape(n_seq * S, D), (1e-6 + leak).reshape(n_seq * S, D), REL[fmt],
                  "attention peaked softmax vs v_target", f"peaked closed form S={S} fmt={fmt}")


# ------------------------------------------------------------------------------------------------------------------
# Fused top-k: documented order = higher score first, equal scores by lower index
# ------------------------------------------------------------------------------------------------------------------
def _topk_reference(q, s, scale):
    """float64 scores and the slack of the path plip_similarity_topk takes for these shapes (similarity_oracle)."""
    if q.shape[0] >= 256 and s.shape[0] >= 8192:
        r = similarity_refs(q, s, scale, 1, 1, need=("contract",))
        return r["contract"], r["contract_slack"]
    r = similarity_refs(q, s, scale, 1, 1, need=("simt",))
    return r["plain"], r["simt_slack"]


def _topk(L, q, s, k, scale=10.0, with_val=True):
    n, m = q.shape[0], s.shape[0]
    idx = torch.full((n + 1, k), -7, device=q.device, dtype=torch.int32)
    val = torch.full((n + 1, k), SENT, device=q.device) if with_val else None
    _check(L.plip_similarity_topk(q.data_ptr(), n, s.data_ptr(), m, C.c_float(scale), 1, 1, k, idx.data_ptr(),
                                  val.data_ptr() if with_val else None, _stream()), "topk")
    torch.cuda.synchronize()
    assert (idx[n] == -7).all() and (val is None or (val[n] == SENT).all()), "top-k wrote past the last query"
    return idx[:n], (val[:n] if with_val else None)


# (n, m, duplicated pairs (a, b): space[b] = space[a]) per dispatch path
#   one CTA per query  n m = 32000 < 65536; its 4 warps take columns c % 4, so (8, 9) sits in two warps' lists and
#                      (3, 3999) at both ends of one warp's
#   tiled              200 x 3000: 4 query tiles -> 47 splits of one 64-column tile each on a 132-SM part, so (63, 64)
#                      and (100, 2000) and (0, 2999) are merged from different CTAs' partial lists
#   tensor-core chunks 256 x 40000: chunks [0, 32768) and [32768, 40000): (32767, 32768) and (5, 39999) straddle the
#                      chunk boundary, (100, 101) share a chunk
TOPK_PATHS = {"cta_per_query": (8, 4000, [(8, 9), (3, 3999), (1000, 2001)]),
              "tiled": (200, 3000, [(63, 64), (100, 2000), (0, 2999)]),
              "tensor_core_chunks": (256, 40000, [(32767, 32768), (5, 39999), (100, 101)])}


@gpu
@pytest.mark.parametrize("k", [64, 5, 1])
@pytest.mark.parametrize("path", list(TOPK_PATHS))
def test_topk_tie_order_across_boundaries(L, path, k):
    dev = "cuda"
    n, m, pairs = TOPK_PATHS[path]
    g = _gen(dev, n + m)
    s = _randn((m, 512), g, dev)
    for a, b in pairs:
        s[b] = s[a]
    # query i points at pair i % 3: the two copies are its best matches by a wide margin, with equal scores
    q = torch.stack([s[pairs[i % len(pairs)][0]] for i in range(n)]) + 0.05 * _randn((n, 512), g, dev)
    idx, val = _topk(L, q, s, k)
    first = torch.tensor([pairs[i % len(pairs)][0] for i in range(n)], device=dev, dtype=torch.int32)
    second = torch.tensor([pairs[i % len(pairs)][1] for i in range(n)], device=dev, dtype=torch.int32)
    assert torch.equal(idx[:, 0], first), f"{path}: the lower index of a tie must come first"
    if k > 1:
        assert torch.equal(idx[:, 1], second)
        assert torch.equal(_bits(val[:, 0].contiguous()), _bits(val[:, 1].contiguous())), f"{path}: copies of a row score differently"
        # the whole list obeys the order: scores descend, equal scores ascend in index
        dv, di = val[:, 1:] - val[:, :-1], idx[:, 1:] - idx[:, :-1]
        assert (dv <= 0).all() and (di[dv == 0] > 0).all()
    ref, slack = _topk_reference(q, s, 10.0)
    topk_check(idx, val, ref, slack, k, path)                  # beyond the planted ties: near-ties within the bounds
    idx2, _ = _topk(L, q, s, k, with_val=False)
    assert torch.equal(idx2, idx), f"{path}: val = NULL changes the indices"


@gpu
@pytest.mark.parametrize("n,m,k", [(4, 5, 8), (4, 1, 64), (2000, 40, 64), (1100, 63, 64)])
def test_topk_short_space_pads(L, n, m, k):
    """m < k: the tail of every list is index -1 / value -inf (one CTA per query for n m < 65536, tiled otherwise; the
    tensor-core path needs m >= 8192 > k and cannot get here)."""
    dev = "cuda"
    g = _gen(dev, n + m + k)
    q, s = _randn((n, 512), g, dev), _randn((m, 512), g, dev)
    idx, val = _topk(L, q, s, k)
    assert (idx[:, m:] == -1).all() and (val[:, m:] == float("-inf")).all()
    ref, slack = _topk_reference(q, s, 10.0)
    topk_check(idx, val, ref, slack, k, f"short space n={n} m={m} k={k}")
    assert torch.equal(idx[:, :m].sort(-1).values, torch.arange(m, device=dev, dtype=torch.int32).expand(n, m))
    idx2, _ = _topk(L, q, s, k, with_val=False)
    assert torch.equal(idx2, idx)
