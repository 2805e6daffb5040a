"""Edges of the ping-pong schedule of the wgmma GEMM (gemm_wgmma.cu): each consumer warpgroup owns a whole 64-row
tile, warpgroup w takes the CTA's tiles i with i % 2 == w, and the two main loops take turns through two named
barriers.  The cases below reach what 128-row tiles never had to: a CTA whose second warpgroup gets no tile, a last
round with warpgroup 0 alone, fewer tiles than consumer warpgroups on the grid, 64-row tiles with 1 or 63 valid rows,
and k-block counts that make the two warpgroups enter the ring at different slots and phases.  Each case runs the
16-bit-store epilogue (0), the residual epilogue with the 16-bit copy and row statistics (2) and the fp32 epilogue (4).

Tile counts: ceil(M / (64 CG)) x N / BN tiles over min(tiles, resident groups) groups; resident groups = #SMs for CG 1
(132 on an H100 SXM) and at most #SMs / 2 clusters for CG 2.
"""
import pytest
import torch

from test_gpu_kernel_edges import _check, _gen, _operands, _sm_count, _stream, run_gemm

gpu = pytest.mark.gpu

EPIS = [(0, False), (2, True), (4, False)]   # (epilogue, emit the 16-bit copy and statistics)


@pytest.fixture(scope="module")
def L():
    from plip_b200._lib import lib
    return lib()


# One tile per CTA (its second warpgroup only passes the turn): M = 1000, N = 768 -> 16 x 3 = 48 tiles (CG 1) and
# 8 x 3 = 24 (CG 2), fewer than the resident groups, so the grid has one CTA per tile.
@gpu
@pytest.mark.parametrize("epi,emit", EPIS)
@pytest.mark.parametrize("cg", [1, 2])
def test_pingpong_one_tile_per_cta(L, cg, epi, emit):
    run_gemm(L, cg, 256, epi, 1000, 768, 320, emit=emit)


# Three tiles per CTA (the last round has warpgroup 0 only): 3 x groups tiles with one N block.  CG 2 assumes #SMs / 2
# resident clusters; with fewer, most clusters still get an odd count.  The last tile holds 27 valid rows.
@gpu
@pytest.mark.parametrize("epi,emit", EPIS)
@pytest.mark.parametrize("cg", [1, 2])
def test_pingpong_odd_tiles_per_cta(L, cg, epi, emit):
    groups = _sm_count() // cg
    M = 3 * groups * 64 * cg - 37
    run_gemm(L, cg, 256, epi, M, 256, 448, emit=emit)


# Between one and two tiles per group: some CTAs run two tiles, the rest one (fewer tiles than consumer warpgroups).
@gpu
@pytest.mark.parametrize("epi,emit", EPIS)
@pytest.mark.parametrize("cg", [1, 2])
def test_pingpong_fewer_tiles_than_warpgroups(L, cg, epi, emit):
    groups = _sm_count() // cg
    M = (groups + groups // 2) * 64 * cg - 5
    run_gemm(L, cg, 256, epi, M, 256, 192, emit=emit)


# 1 and 63 valid rows in the last 64-row tile, 1 and 63 rows past a 64-row boundary; CG 2 puts them on either CTA.
@gpu
@pytest.mark.parametrize("epi,emit", EPIS)
@pytest.mark.parametrize("cg,bn", [(1, 256), (2, 256), (1, 128), (2, 128)])
@pytest.mark.parametrize("M", [1, 63, 65, 127])
def test_pingpong_partial_last_tile(L, M, cg, bn, epi, emit):
    N = 512 if (emit and bn == 128) else 768      # at most 8 statistics slots: 2 per N tile
    run_gemm(L, cg, bn, epi, M, N, 320, emit=emit)


# 3, 5 and 13 k-blocks: with 4 ring stages (BN 256) or 8 (BN 128) warpgroup 1 starts its first tile at slot k mod S
# and later tiles at other slots and phases.  M = 4157 -> 65 (CG 1) / 33 (CG 2) row blocks x 3 N blocks: several
# tiles per warpgroup, an odd count on some CTAs.
@gpu
@pytest.mark.parametrize("epi,emit", EPIS)
@pytest.mark.parametrize("cg,bn", [(1, 256), (2, 256), (2, 128)])
@pytest.mark.parametrize("K", [192, 320, 832])
def test_pingpong_ring_entry(L, K, cg, bn, epi, emit):
    N = 512 if (emit and bn == 128) else 768
    run_gemm(L, cg, bn, epi, 4157, N, K, emit=emit)


# The tile -> warpgroup assignment changes with CG (and with the grid); no output element may change with it.
@gpu
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("M,K", [(1000, 320), (8229, 832), (127, 192)])
def test_pingpong_f32_bitwise_across_cluster_sizes(L, M, K, bn):
    dev, N = "cuda", 768
    g = _gen(dev, M + K + bn)
    Ab, Wb = _operands(M, N, K, K, K, 0, g, dev, False)
    bias = torch.zeros(N, device=dev)
    outs = []
    for cg in (1, 2):
        out = torch.full((M, N), -1536.0, device=dev)
        _check(L.plip_dbg_gemm(Ab.data_ptr(), K, Wb.data_ptr(), K, M, N, K, bias.data_ptr(), out.data_ptr(), N, None, 4,
                               cg, bn, None, None, 0, None, None, _stream()), "gemm")
        torch.cuda.synchronize()
        outs.append(out)
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), \
        f"EPI_F32 M={M} N={N} K={K} bn={bn}: CG 1 and CG 2 differ in {int((outs[0] != outs[1]).sum())} elements"
