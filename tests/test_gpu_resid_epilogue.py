"""Bit-exactness of the fp32 residual epilogue of the wgmma GEMM (EPI_BIAS_RESID_F32: x += acc + bias in place, with
the optional 16-bit copy of the new rows and their row statistics).

The epilogue loads x and stores y as TMA boxes of [16 rows x 32 fp32] staged in shared memory.  Whatever the path, the data
must be exactly y = x + (acc + bias) in fp32: acc is taken from the EPI_F32 output of the same operands and tile
configuration, y is computed by torch in fp32 and compared bit for bit, and xb_out must be the 16-bit rounding of y.
Guard rows past M and pad columns past N hold a sentinel that must keep its bits; statistics slots are checked against
float64 sums.

Shapes (BM = 128 rows per tile, 16 rows per consumer warp, BN in {128, 192, 256}):
  M = 16384 + 37: 129 row blocks, the last one has 37 rows (its third warp holds a partial 16-row box, the warps after
      it only rows past M); 387 tiles at N 768 / BN 256, so every CTA runs several tiles and each warp's two staging
      blocks go round many times (8 boxes per tile at BN 256).
  M = 300: 3 row blocks, the last one 44 rows; fewer tiles than CTAs.
  K = 768 (12 k-blocks) and K = 320 (5 k-blocks: tiles start in the middle of the operand ring).
"""
import math

import pytest
import torch

gpu = pytest.mark.gpu

DT = {0: torch.bfloat16, 1: torch.float16}
SENT = -1536.0        # exactly representable in bf16, fp16 and fp32; no operand or result below comes near it
U32 = 2.0 ** -23      # one fp32 ulp, relative
EPI_RESID, EPI_F32 = 2, 4
M_BIG = 16384 + 37


@pytest.fixture(scope="module")
def L():
    from plip_b200._lib import lib
    return lib()


@pytest.fixture
def fmt_guard(L):
    """Switches the handle-free hooks to the requested 16-bit format; bf16 is restored whatever happens."""
    from plip_b200._lib import check

    def set_fmt(fmt):
        check(L.plip_dbg_set_operand_format(fmt), "set_operand_format")
    try:
        yield set_fmt
    finally:
        L.plip_dbg_set_operand_format(0)


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _first_diff(a, b):
    d = (_bits(a) != _bits(b)).nonzero()
    return d[0].tolist() if len(d) else None


def run_resid(L, cg, bn, N, fmt, M=M_BIG, K=768, ldo=None, emit=True):
    from plip_b200._lib import check
    dev = "cuda"
    ldo = ldo or N
    stream = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device=dev).manual_seed(M * 7 + N * 3 + K + 11 * fmt + cg + bn)
    dt = DT[fmt]
    A = (torch.randn((M, K), generator=g, device=dev) * 0.5).to(dt)
    W = (torch.randn((N, K), generator=g, device=dev) * 0.05).to(dt)
    bias = torch.randn((N,), generator=g, device=dev)
    x0 = torch.randn((M, N), generator=g, device=dev) * 4.0

    def launch(epi, out, xb=None, stats=None):
        check(L.plip_dbg_gemm(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(), out.data_ptr(), ldo, None, epi,
                              cg, bn, None, None, 0, xb.data_ptr() if xb is not None else None,
                              stats.data_ptr() if stats is not None else None, stream), f"gemm epi {epi}")

    acc = torch.full((M, ldo), SENT, device=dev)
    launch(EPI_F32, acc)
    out = torch.full((M + 8, ldo), SENT, device=dev)
    out[:M, :N] = x0
    before = out.clone()
    xb = torch.full((M + 8, ldo), SENT, device=dev, dtype=dt) if emit else None
    stats = torch.full((M + 8, 8, 2), SENT, device=dev) if emit else None
    launch(EPI_RESID, out, xb, stats)
    torch.cuda.synchronize()
    what = f"cg={cg} bn={bn} M={M} N={N} K={K} ldo={ldo} fmt={fmt} emit={emit}"

    y = x0 + (acc[:, :N] + bias)                     # the kernel's per-element arithmetic, in torch fp32
    got = out[:M, :N]
    assert torch.equal(_bits(got), _bits(y)), f"{what}: y != x + (acc + b) at (row, col) {_first_diff(got, y)}"
    guard = before.clone()
    guard[:M, :N] = y
    assert torch.equal(_bits(out), _bits(guard)), f"{what}: guard row or pad column changed at {_first_diff(out, guard)}"
    if not emit:
        return
    yb = y.to(dt)
    assert torch.equal(_bits(xb[:M, :N]), _bits(yb)), f"{what}: xb_out is not the 16-bit rounding of y at {_first_diff(xb[:M, :N], yb)}"
    xg = torch.full_like(xb, SENT)
    xg[:M, :N] = yb
    assert torch.equal(_bits(xb), _bits(xg)), f"{what}: xb_out guard changed at {_first_diff(xb, xg)}"
    eff_bn = bn if N % bn == 0 else 128
    npart = 2 * (N // eff_bn)                           # one slot per (N tile, half of the tile's columns)
    y64 = y.double()
    s = stats[:M, :npart].double().sum(1)
    # each slot is an fp32 sum of <= 128 values: 2^-23 sqrt(128) of the absolute sum is a wide bound
    tol1 = U32 * math.sqrt(128) * y64.abs().sum(-1) + 1e-6
    tol2 = U32 * math.sqrt(128) * (y64 * y64).sum(-1) + 1e-6
    e1, e2 = (s[:, 0] - y64.sum(-1)).abs(), (s[:, 1] - (y64 * y64).sum(-1)).abs()
    assert (e1 <= tol1).all() and (e2 <= tol2).all(), (what, (e1 / tol1).max().item(), (e2 / tol2).max().item())
    sg = torch.full_like(stats, SENT)
    sg[:M, :npart] = stats[:M, :npart]
    assert torch.equal(_bits(stats), _bits(sg)), f"{what}: statistics slots >= {npart} or guard rows were written"


# every (cg, bn) that accepts statistics: N 768 -> BN 256 / 192 (BN 128 would need 12 > 8 slots); N 512 -> all four
STATS_CASES = [(1, 256, 768), (2, 256, 768), (2, 192, 768), (1, 256, 512), (2, 256, 512), (1, 128, 512), (2, 128, 512)]
# without statistics: cg 1 / bn 128, and N 1536 (too many tiles per row for the statistics slots at any BN)
PLAIN_CASES = [(1, 128, 768), (1, 128, 1536), (1, 256, 1536), (2, 256, 1536), (2, 192, 1536)]


@gpu
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("cg,bn,N", STATS_CASES)
def test_resid_with_statistics_bitwise(L, fmt_guard, cg, bn, N, fmt):
    fmt_guard(fmt)
    run_resid(L, cg, bn, N, fmt)


@gpu
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("cg,bn,N", PLAIN_CASES)
def test_resid_without_copy_bitwise(L, fmt_guard, cg, bn, N, fmt):
    """xb_out == nullptr (the last layer's fc2): only x changes."""
    fmt_guard(fmt)
    run_resid(L, cg, bn, N, fmt, emit=False)


@gpu
@pytest.mark.parametrize("cg,bn,N,ldo,emit", [(2, 256, 768, 768 + 40, True), (2, 192, 768, 1024, True),
                                              (1, 128, 512, 520, True), (2, 256, 1536, 1536 + 8, False)])
def test_resid_row_stride_beyond_n(L, cg, bn, N, ldo, emit):
    run_resid(L, cg, bn, N, 0, ldo=ldo, emit=emit)


@gpu
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("cg,bn,N,emit", [(2, 256, 768, True), (1, 256, 512, True), (2, 128, 512, True),
                                          (2, 192, 1536, False)])
def test_resid_small_m_short_k(L, fmt_guard, cg, bn, N, emit, fmt):
    """M = 300 (last tile 44 rows: one partial 16-row box, the rest past M), K = 320 (5 k-blocks)."""
    fmt_guard(fmt)
    run_resid(L, cg, bn, N, fmt, M=300, K=320, ldo=N + 8, emit=emit)
