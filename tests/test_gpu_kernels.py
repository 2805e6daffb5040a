"""Per-kernel parity on the GPU, through the C ABI test hooks, against plain torch fp32 references."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from plip_b200._lib import lib
    return lib()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check(rc, what):
    from plip_b200._lib import check
    check(rc, what)


GEMM_CASES = [
    # cg, bn, epi, M, N, K      (epi: 0 bias->bf16, 1 bias+quickgelu->bf16, 2 bias+residual f32, 3 patch scatter, 4 f32)
    (1, 128, 4, 128, 128, 64),
    (1, 256, 4, 300, 512, 768),      # ragged M (TMA zero fill + row guard)
    (2, 128, 4, 256, 128, 64),
    (2, 256, 4, 1000, 768, 3072),
    (1, 256, 0, 1000, 768, 768),
    (2, 256, 0, 1111, 2304, 768),
    (2, 256, 1, 1000, 3072, 768),
    (2, 256, 2, 1000, 768, 3072),
    (1, 256, 2, 77, 512, 2048),
    (2, 256, 3, 980, 768, 3072),
    (2, 256, 4, 1, 512, 768),        # single row (projection of one image)
    (0, 0, 2, 4097, 1536, 512),      # auto config
]


@pytest.mark.parametrize("cg,bn,epi,M,N,K", GEMM_CASES)
def test_gemm_epilogues(L, cg, bn, epi, M, N, K):
    dev = "cuda"
    g = torch.Generator().manual_seed(M * 7 + N + K + epi)
    A = (torch.randn(M, K, generator=g) * 0.5).to(dev).to(torch.bfloat16)
    W = (torch.randn(N, K, generator=g) * 0.05).to(dev).to(torch.bfloat16)
    bias = torch.randn(N, generator=g).to(dev)
    pos = torch.randn(50, N, generator=g).to(dev)
    ref = A.float() @ W.float().t()
    if epi in (0, 1, 2):
        ref = ref + bias
    if epi == 1:
        ref = ref * torch.sigmoid(1.702 * ref)
    if epi in (0, 1):
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        tol = 2.0 ** -8 * max(1.0, ref.abs().max().item())   # one bf16 ulp of the largest value
    elif epi == 2:
        x0 = torch.randn(M, N, generator=g).to(dev)
        out = x0.clone()
        ref = ref + x0
        tol = 2e-4
    elif epi == 3:
        nb = M // 49
        out = torch.full((nb * 50, N), 7.0, device=dev)
        r = torch.full((nb * 50, N), 7.0, device=dev)        # class rows must stay untouched
        r.view(nb, 50, N)[:, 1:, :] = ref.view(nb, 49, N) + pos[1:]
        ref = r
        tol = 2e-4
    else:
        out = torch.zeros(M, N, device=dev)
        tol = 2e-4
    _check(L.plip_dbg_gemm(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(), out.data_ptr(), N,
                           pos.data_ptr(), epi, cg, bn, None, None, 0, None, None, _stream()), "gemm")
    torch.cuda.synchronize()
    assert (out.float() - ref).abs().max().item() <= tol


@pytest.mark.parametrize("D,N,gelu,bn_prod", [(768, 2304, False, 256), (768, 3072, True, 192), (512, 1536, False, 256),
                                               (512, 2048, True, 128)])
def test_layernorm_folded_gemm_chain(L, D, N, gelu, bn_prod):
    """Residual GEMM epilogue emits bf16(x') + row statistics; the next GEMM applies LayerNorm through the
    fold  rstd (x' W'^T - mean colsum) + bias'  ==  LN(x') W^T + bias   (TF:371/380 + 310-312/348-349)."""
    dev = "cuda"
    M, K0 = 1000, 256
    g = torch.Generator().manual_seed(D + N)
    A0 = (torch.randn(M, K0, generator=g) * 0.5).to(dev).to(torch.bfloat16)
    W0 = (torch.randn(D, K0, generator=g) * 0.1).to(dev).to(torch.bfloat16)
    b0 = torch.randn(D, generator=g).to(dev) * 0.1
    x0 = (torch.randn(M, D, generator=g) * 1.5 + 0.4).to(dev)
    x = x0.clone()
    xb = torch.zeros(M, D, device=dev, dtype=torch.bfloat16)
    stats = torch.full((M, 8, 2), float("nan"), device=dev)
    _check(L.plip_dbg_gemm(A0.data_ptr(), K0, W0.data_ptr(), K0, M, D, K0, b0.data_ptr(), x.data_ptr(), D, None, 2, 2,
                           bn_prod, None, None, 0, xb.data_ptr(), stats.data_ptr(), _stream()), "resid gemm")
    xr = x0 + A0.float() @ W0.float().t() + b0
    npart = 2 * (D // bn_prod)      # one slot per (N tile, epilogue-warp half)
    assert (x - xr).abs().max().item() < 2e-4
    assert torch.equal(xb, x.to(torch.bfloat16))
    s = stats[:, :npart].sum(1)
    assert torch.allclose(s[:, 0], x.sum(-1), atol=2e-3) and torch.allclose(s[:, 1], (x * x).sum(-1), rtol=1e-5, atol=1e-2)
    # standalone producer of the same quantities (start of a tower)
    xb2 = torch.zeros_like(xb)
    st2 = torch.zeros(M, 8, 2, device=dev)
    _check(L.plip_dbg_rowstats_cast(x.data_ptr(), M, D, xb2.data_ptr(), st2.data_ptr(), _stream()), "rowstats")
    assert torch.equal(xb2, xb) and torch.allclose(st2[:, 0, 0], x.sum(-1), atol=2e-3)
    # consumer with the fold
    gam = 1 + 0.1 * torch.randn(D, generator=g).to(dev)
    bet = 0.05 * torch.randn(D, generator=g).to(dev)
    W = (torch.randn(N, D, generator=g) * 0.05).to(dev)
    bias = torch.randn(N, generator=g).to(dev) * 0.1
    Wf = (W * gam[None]).to(torch.bfloat16)
    colsum = Wf.float().sum(1).contiguous()
    biasf = (bias + W @ bet).contiguous()
    out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    _check(L.plip_dbg_gemm(xb.data_ptr(), D, Wf.data_ptr(), D, M, N, D, biasf.data_ptr(), out.data_ptr(), N, None,
                           6 if gelu else 5, 0, 0, colsum.data_ptr(), stats.data_ptr(), npart, None, None, _stream()), "ln gemm")
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x, (D,), gam, bet, 1e-5) @ W.t() + bias
    if gelu:
        ref = ref * torch.sigmoid(1.702 * ref)
    err = (out.float() - ref).abs()
    assert err.max().item() < 0.06 and err.mean().item() < 6e-3, (err.max().item(), err.mean().item())


def test_gemm_rejects_bad_shapes(L):
    a = torch.zeros(128, 100, device="cuda", dtype=torch.bfloat16)
    o = torch.zeros(128, 128, device="cuda")
    assert L.plip_dbg_gemm(a.data_ptr(), 100, a.data_ptr(), 100, 128, 128, 100, None, o.data_ptr(), 128, None, 4, 0, 0,
                           None, None, 0, None, None, _stream()) != 0
    from plip_b200._lib import last_error
    assert "multiple of 64" in last_error()


@pytest.mark.parametrize("D", [768, 512])
def test_layernorm(L, D):
    x = torch.randn(1003, D, device="cuda") * 3 + 0.5
    g, b = torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    of = torch.empty_like(x)
    ob = torch.empty(1003, D, device="cuda", dtype=torch.bfloat16)
    _check(L.plip_dbg_layernorm(x.data_ptr(), 1003, D, D, g.data_ptr(), b.data_ptr(), of.data_ptr(), ob.data_ptr(),
                                _stream()), "ln")
    from helper_oracle import layernorm_ref, layernorm_slack
    err = (of.double() - layernorm_ref(x, g, b)).abs()
    assert (err <= layernorm_slack(x, g, b)).all()      # the kernel's fp32 op order, bounded per element
    assert torch.allclose(of, torch.nn.functional.layer_norm(x, (D,), g, b, 1e-5), rtol=0, atol=1e-5)
    assert torch.equal(ob, of.to(torch.bfloat16))          # same rounding as torch's RNE cast


def test_im2col_formats(L):
    from oracle import clip_oracle as O
    n = 5
    px = torch.randn(n, 3, 224, 224, device="cuda")
    ref = px.reshape(n, 3, 7, 32, 7, 32).permute(0, 2, 4, 1, 3, 5).reshape(n * 49, 3072)
    out = torch.empty(n * 49, 3072, device="cuda", dtype=torch.bfloat16)
    _check(L.plip_dbg_im2col(px.data_ptr(), 0, n, out.data_ptr(), _stream()), "im2col f32")
    assert torch.equal(out, ref.to(torch.bfloat16))
    pb = px.to(torch.bfloat16)
    _check(L.plip_dbg_im2col(pb.data_ptr(), 1, n, out.data_ptr(), _stream()), "im2col bf16")
    assert torch.equal(out, ref.to(torch.bfloat16))
    u8 = torch.randint(0, 256, (n, 224, 224, 3), dtype=torch.uint8)
    pref = O.preprocess_u8(u8).cuda()
    ref8 = pref.reshape(n, 3, 7, 32, 7, 32).permute(0, 2, 4, 1, 3, 5).reshape(n * 49, 3072)
    u8d = u8.cuda()
    _check(L.plip_dbg_im2col(u8d.data_ptr(), 2, n, out.data_ptr(), _stream()), "im2col u8")
    assert (out.float() - ref8).abs().max().item() < 2.0 ** -7     # bf16 rounding of values up to ~2.7
    from helper_oracle import im2col_ref
    assert torch.equal(out, im2col_ref(u8d, 2, torch.bfloat16))   # bit for bit: the kernel's FFMA + FMUL, then RNE


ATT_CASES = [(7, 50, 12, False, False), (64, 50, 12, False, False), (1, 50, 12, False, False),
             (5, 77, 8, True, False), (33, 77, 8, True, False), (6, 20, 8, True, False),
             (9, 77, 8, True, True), (4, 128, 8, True, False), (3, 33, 8, False, True)]


@pytest.mark.parametrize("n_seq,S,heads,causal,use_mask", ATT_CASES)
def test_attention(L, n_seq, S, heads, causal, use_mask):
    dev = "cuda"
    D = heads * 64
    g = torch.Generator().manual_seed(n_seq * 131 + S)
    qkv = torch.randn(n_seq * S, 3 * D, generator=g).to(dev).to(torch.bfloat16)
    out = torch.zeros(n_seq * S, D, device=dev, dtype=torch.bfloat16)
    mask = None
    if use_mask:
        lens = torch.randint(3, S + 1, (n_seq,), generator=g)
        mask = (torch.arange(S)[None] < lens[:, None]).to(torch.int32).to(dev).contiguous()
    _check(L.plip_dbg_attention(qkv.data_ptr(), n_seq, S, heads, int(causal),
                                mask.data_ptr() if mask is not None else None, out.data_ptr(), _stream()), "attention")
    torch.cuda.synchronize()
    q, k, v = qkv.float().view(n_seq, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
    att = q @ k.transpose(-1, -2)      # the dh^-0.5 scale lives in the packed q weights, not in the kernel
    if causal:
        att = att + torch.full((S, S), float("-inf"), device=dev).triu(1)
    if mask is not None:
        att = att.masked_fill((mask == 0)[:, None, None, :], float("-inf"))
    ref = (torch.softmax(att, -1) @ v).permute(0, 2, 1, 3).reshape(n_seq * S, D)
    assert not torch.isnan(out.float()).any()
    err = (out.float() - ref).abs()
    # P and the output are rounded to bf16 (as an HF bf16 model does); inputs are N(0,1) so |out| <= ~5
    assert err.max().item() < 0.03 and err.mean().item() < 2e-3


@pytest.mark.parametrize("n,m,k", [(200, 3000, 50), (1000, 777, 10), (3, 40000, 64), (130, 64, 1),
                                   (300, 20000, 50), (257, 8192, 10)])   # the last two: tensor-core score chunks + row merge
def test_similarity_topk_tiled(L, n, m, k):
    """GEMM-shaped fused top-k (never materialises [n,m]): a top-k of the float64 scores within the fp32 kernels'
    bound (similarity_oracle.simt_ref), or the split contract on the tensor-core path (the last two cases)."""
    from similarity_oracle import similarity_refs, topk_check
    dev = "cuda"
    g = torch.Generator().manual_seed(n + m + k)
    a = torch.randn(n, 512, generator=g).to(dev)
    b = torch.randn(m, 512, generator=g).to(dev)
    idx = torch.empty(n, k, device=dev, dtype=torch.int32)
    val = torch.empty(n, k, device=dev)
    _check(L.plip_similarity_topk(a.data_ptr(), n, b.data_ptr(), m, C.c_float(10.0), 1, 1, k, idx.data_ptr(),
                                  val.data_ptr(), _stream()), "topk")
    torch.cuda.synchronize()
    if n >= 256 and m >= 8192:
        r = similarity_refs(a, b, 10.0, 1, 1, need=("contract",))
        topk_check(idx, val, r["contract"], r["contract_slack"], k, f"tensor-core top-k n={n} m={m}")
    else:
        r = similarity_refs(a, b, 10.0, 1, 1, need=("simt",))
        topk_check(idx, val, r["plain"], r["simt_slack"], k, f"fp32 top-k n={n} m={m}")
