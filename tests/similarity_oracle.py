"""float64 references of the similarity head (similarity.cu), the L2 normalisation (elementwise.cu) and the per-element
acceptance of a top-k list.

`split_contract_ref` is what the tensor-core path (split_embed_kernel + the EPI_SIM_F32 GEMM) is specified to compute,
`plain_ref` the mathematical result `scale * norm(a) . norm(b)^T` with the slack the split path is entitled to against
it, `simt_ref` the same result with the slack of the fp32 FMA kernels (similarity_kernel, similarity_topk_kernel,
similarity_topk_tiled_kernel), `topk_check` the acceptance of a top-k list against any of them and `l2_ref` what
l2_normalize_kernel computes.  Every function works on the device of its inputs.  They live in their own module so
that several test modules can import them without pytest collecting one test module from another.

`scale` is taken as the fp32 value the kernels receive (ctypes.c_float of the Python float).
"""
import math

import numpy as np
import torch

from attention_oracle import OBSERVED, SENT, U32, _note, assert_within  # noqa: F401  (re-exported for the suites)

K_PROJ = 512
SPLIT_K = 3 * K_PROJ                     # [hi|lo|hi] . [hi|hi|lo]
U24 = 2.0 ** -24                         # one rounding to nearest in fp32, relative
SUB16 = 2.0 ** -14                       # smallest normal fp16
ROW_CHUNK = 131072                       # kSimRowChunk: A rows split + multiplied per pass of launch_similarity_tc
ABI_CHUNK = 65535 * 64                   # plip_similarity's rows per launch_similarity call (SIMT grid.y limit)
TEMP_ELEMS = 1 << 26                     # float64 elements per [rows, m] temporary (512 MB)

# Tensor-core path, relative error of the fp32 scale vectors (derivation in split_contract_ref)
SS_SPLIT = 12 * U24                      # split_embed_kernel's warp sum of squares
RS_NORM = SS_SPLIT / 2 + 4 * U24         # rsqrtf of it (2 ulp)
# fp32 kernels (derivation in simt_ref)
SS_SIMT = 40 * U24                       # the per-thread sum of squares of similarity_kernel, 32 k-steps of 4 terms
INV_SIMT = SS_SIMT / 2 + 2 * U24         # 1.0f / sqrtf(ss)


def f32(scale):
    """The fp32 value a c_float argument carries."""
    return float(np.float32(scale))


def split_rows(x):
    """split_embed_kernel's operands of the fp32 rows x [r, 512], bit for bit: p = 2^(6 - e) with frexp(max|x|) = (., e)
    (1 for a zero row), f = p x (exact), hi = rn16(f), lo = rn16(f - hi) (f - hi is exact in fp32), both with fp16
    subnormals as __float2half_rn.  Returns (p [r] float64, f [r, 512] float32, hi, lo [r, 512] float16)."""
    x = x.float()
    mx = x.abs().amax(-1)
    _, e = torch.frexp(mx)
    p = torch.where(mx > 0, torch.exp2((6 - e).double()), torch.ones_like(mx, dtype=torch.float64))
    f = (x.double() * p[:, None]).float()
    hi = f.half()
    lo = (f - hi.float()).half()
    return p, f, hi, lo


def _norms(x):
    return x.double().pow(2).sum(-1).sqrt()


def _chunks(n, m):
    step = max(1, TEMP_ELEMS // max(1, m))
    return [(i, min(n, i + step)) for i in range(0, n, step)]


def similarity_refs(a, b, scale, norm_a, norm_b, need=("contract", "plain", "simt")):
    """The three references at once (they share the float64 products).  Returns a dict with the [n, m] float64 tensors
    'contract', 'contract_slack', 'plain', 'plain_slack', 'resid' (the split residual alone) and 'simt_slack', as
    far as `need` asks for them.  Rows are processed in chunks so that no [rows, m] temporary exceeds 512 MB."""
    n, m = a.shape[0], b.shape[0]
    s = f32(scale)
    out = {}
    want_split = "contract" in need or "plain" in need
    want_plain = "plain" in need or "simt" in need
    keys = []
    if want_split:
        keys += ["contract", "contract_slack"]
    if "plain" in need:
        keys += ["resid", "plain_slack"]
    if want_plain:
        keys += ["plain"]
    if "simt" in need:
        keys += ["simt_slack"]
    for key in keys:
        out[key] = torch.empty(n, m, dtype=torch.float64, device=a.device)

    nb = _norms(b)
    ib = 1.0 / nb if norm_b else torch.ones_like(nb)
    b64 = b.double()
    if want_split:
        pb, fb, hb, lb = split_rows(b)
        Bs = torch.cat([hb, hb, lb], 1).double()
        cs = ib / pb                                          # float64 column scales
        fb64 = fb.double()
        sub_b = ((fb - hb.float()).abs() < SUB16).double()
    for i, j in _chunks(n, m):
        ac = a[i:j]
        na = _norms(ac)
        ia = s / na if norm_a else torch.full_like(na, s)
        if want_split:
            pa, fa, ha, la = split_rows(ac)
            As = torch.cat([ha, la, ha], 1).double()
            rs = ia / pa
            w = rs[:, None].abs() * cs[None].abs()
            # exact partial sums of the k16 steps; run = sum over steps of the running sum each step adds into
            acc = torch.zeros(j - i, m, dtype=torch.float64, device=a.device)
            run = torch.zeros_like(acc)
            for k0 in range(0, SPLIT_K, 16):
                run += acc.abs()
                acc.addmm_(As[:, k0:k0 + 16], Bs[:, k0:k0 + 16].t())
            contract = acc * rs[:, None] * cs[None]
            run += As.abs() @ Bs.abs().t()
            rel = 3 * U24 + (RS_NORM + U24 if norm_a else 0.0) + (RS_NORM if norm_b else 0.0)
            cslack = 2 * U32 * run * w + rel * contract.abs()
            out["contract"][i:j] = contract
            out["contract_slack"][i:j] = cslack
            del acc, run
            if "plain" in need:
                fa64 = fa.double()
                sub_a = ((fa - ha.float()).abs() < SUB16).double()
                resid = (3 * 2.0 ** -22 * (fa64.abs() @ fb64.abs().t())
                         + 2.0 ** -25 * (sub_a @ fb64.abs().t() + fa64.abs() @ sub_b.t())) * (1 + 2.0 ** -10) * w
                out["resid"][i:j] = resid
                out["plain_slack"][i:j] = cslack + resid
                del resid
        if want_plain:
            a64 = ac.double()
            plain = (a64 @ b64.t()) * ia[:, None] * ib[None]
            out["plain"][i:j] = plain
            if "simt" in need:
                rel = 3 * U24 + (INV_SIMT if norm_a else 0.0) + (INV_SIMT if norm_b else 0.0)
                out["simt_slack"][i:j] = (2 * U24 * math.sqrt(K_PROJ) * (a64.abs() @ b64.abs().t()) * ia[:, None].abs()
                                          * ib[None].abs() + rel * plain.abs())
    return out


def split_contract_ref(a, b, scale, norm_a, norm_b):
    """What the tensor-core path computes, in float64, and the slack of its fp32 arithmetic.  Returns (ref, slack).

    The operands are split_rows(a), split_rows(b).  The GEMM sums hi_a hi_b + lo_a hi_b + hi_a lo_b over K = 1536; each
    fp16 x fp16 product is exact, so the float64 sum is the exact one (its own rounding is 2^-53 of sum |terms|).  The
    epilogue writes (acc * rs[r]) * cs[c] with
         rs = undo_a * (norm_a ? rsqrtf(ss_a) : 1) * scale,    cs = undo_b * (norm_b ? rsqrtf(ss_b) : 1),    undo = 1 / p.
    Slack, per element:
      accumulation   the tensor core adds the exact products of a k16 step (k ascending) to the fp32 running sum
                     s_(j-1) and truncates: at most one ulp, 2^-23, of the magnitudes the step adds, and as much again
                     for the alignment of its 16 products.  Over the 96 steps
                         2 x 2^-23 (sum_j |s_(j-1)| + sum_k |terms_k|) x |rs cs|
                     with the partial sums s_j taken exactly in float64.  gemm_ref's random-walk model,
                     2 x 2^-23 sqrt(96) sum |terms|, does not hold here: truncation errors share the sign of the running
                     sum, and when one product dominates it (the spike family) they add up linearly over the steps
                     that follow (an H100 reached 1.02 of that model there).
      epilogue       two fp32 products: 2 x 2^-24 |out|.
      rs, cs         ss is a warp sum of 16 squares per lane, (x^2 + y^2) + (z^2 + w^2) added into ss four times,
                     then 5 shuffle adds: every term passes at most 3 + 4 + 5 = 12 roundings, and a sum of
                     positive terms is then within 12 x 2^-24 of the exact one (SS_SPLIT).  rsqrtf halves that
                     and adds its 2 ulp = 4 x 2^-24 (RS_NORM).  undo * rsqrtf is exact (a power of two);
                     * scale rounds once more for rs.  Without normalisation undo * 1 * scale is exact.
      higher order   1 x 2^-24 of |out| covers the products of the first-order terms.
    A zero row gives NaN where it is normalised (0 x inf), as the kernel does."""
    r = similarity_refs(a, b, scale, norm_a, norm_b, need=("contract",))
    return r["contract"], r["contract_slack"]


def plain_ref(a, b, scale, norm_a, norm_b):
    """scale . norm(a) . norm(b)^T in float64 from the fp32 rows, and the slack of the tensor-core path against it:
    the contract slack plus the split residual.  Returns (ref, slack, resid).

    The split represents f = p x as hi + lo + d, d the rounding of lo: |lo| <= half an ulp of hi <= 2^-11 |f|, so
    |d| <= 2^-11 |lo| <= 2^-22 |f| for a normal lo and |d| <= 2^-25 for a subnormal lo (fp16 subnormals are 2^-24
    apart).  What the GEMM leaves out of f_a f_b is lo_a lo_b + d_a f_b + d_b f_a (to first order), hence per element
         resid = (3 x 2^-22 sum_k |f_a||f_b| + 2^-25 sum_k ([lo_a subnormal] |f_b| + |f_a| [lo_b subnormal])) |rs cs|
    with 2^-10 of it for the higher-order terms.  The bound follows each term's magnitude, not the largest logit."""
    r = similarity_refs(a, b, scale, norm_a, norm_b, need=("plain",))
    return r["plain"], r["plain_slack"], r["resid"]


def simt_ref(a, b, scale, norm_a, norm_b):
    """The float64 result (as plain_ref) and the slack of the fp32 FMA kernels against it.  Returns (ref, slack).

    similarity_kernel runs one sequential fmaf chain over k = 0 .. 511 per output.  Each step rounds the running sum
    once (2^-24 of it); with random signs the errors add like a random walk, gemm_ref's model with a factor-2 margin:
         2 x 2^-24 sqrt(512) sum_k |a_k||b_k| x |scale inv_a inv_b|.
    The sums of squares are positive: a thread adds 32 k-steps of 4 squares (contracted to fmas) and two shuffles
    combine 4 threads, so every term passes at most 4 + 32 + 2 = 38 roundings: 40 x 2^-24 relative (SS_SIMT).
    inv = 1.0f / sqrtf(ss) is IEEE (no fast-math): half of that plus 2 x 2^-24 (INV_SIMT).  The output is
    acc * (scale * inv_a) * inv_b: three roundings, 3 x 2^-24 of |out|.  The two top-k kernels form the same score
    with fewer roundings in every term (the per-query kernel: 16 fmas per lane and a 5-level shuffle tree; the tiled
    kernel: similarity_kernel's tile with ((acc * scale) * inv_a) * inv_b), so this slack bounds them too."""
    r = similarity_refs(a, b, scale, norm_a, norm_b, need=("simt",))
    return r["plain"], r["simt_slack"]


def l2_ref(x):
    """x / |x| in float64 and the per-element relative bound of l2_normalize_kernel.  Returns (ref, rel) with rel a
    Python float.  Lane l adds c = ceil(dim / 32) squares (one rounding per term: fmaf, or the product of the
    first), 5 shuffle adds follow: every term passes at most c + 5 roundings, the positive sum is within (c + 5) 2^-24
    of the exact one.  1 / sqrtf halves that and adds 2 roundings, x * inv one more:
         rel = ((c + 5) / 2 + 3) x 2^-24,
    with 2^-10 of it for the higher-order terms.  A lane missing from the reduction moves a row by ~1/64 of itself,
    far outside.  A zero row gives NaN (0 x inf), as x / x.norm() does."""
    dim = x.shape[-1]
    c = (dim + 31) // 32
    x64 = x.double()
    return x64 / x64.pow(2).sum(-1, keepdim=True).sqrt(), ((c + 5) / 2 + 3) * U24 * (1 + 2.0 ** -10)


def topk_check(idx, val, ref, slack, k, what, key=None):
    """Acceptance of a top-k list (idx int32 [n, k], val [n, k] fp32 or None) against float64 scores ref [n, m] with
    per-element slack, NaN where the kernel's score is NaN (skipped by every path):
      * indices lie in [-1, m), are distinct, and are -1 exactly past the number of non-NaN scores of the row
        (with value -inf there);
      * values do not increase, and equal values ascend in index;
      * each value is within the slack of ref at its index;
      * the set is a top-k of some scores within the slack: no left-out score can exceed a chosen one, i.e.
        max over left-out c of (ref - slack) <= min over chosen r of (ref + slack).  A candidate may be exchanged
        only with one whose float64 gap is within the sum of their two slacks.
    Records the largest value error / slack under `key`."""
    n, m = ref.shape
    dev = ref.device
    idx = idx.long()
    pos = torch.arange(k, device=dev)[None]
    valid = (~torch.isnan(ref)).sum(1, keepdim=True)
    neg = idx < 0
    assert ((idx >= -1) & (idx < m)).all(), f"{what}: index out of range"
    pad = pos >= valid.clamp(max=k)
    bad = neg != pad
    assert not bad.any(), f"{what}: -1 at the wrong places, first at {bad.nonzero()[0].tolist()}"
    srt = idx.sort(1).values
    dup = (srt[:, 1:] == srt[:, :-1]) & (srt[:, 1:] >= 0)
    assert not dup.any(), f"{what}: repeated index in row {dup.nonzero()[0, 0].item()}"
    g = idx.clamp(min=0)
    r_at = ref.gather(1, g)
    s_at = slack.gather(1, g)
    if val is not None:
        v = val.double()
        assert (v[neg] == float("-inf")).all(), f"{what}: padding entry without value -inf"
        down = v[:, 1:] <= v[:, :-1]
        tie = (v[:, 1:] == v[:, :-1]) & ~neg[:, 1:]
        assert down.all(), f"{what}: values increase at {(~down).nonzero()[0].tolist()}"
        assert (idx[:, 1:] > idx[:, :-1])[tie].all(), f"{what}: equal values not in ascending index order"
        err = (v - r_at).abs()
        bad = ~(err <= s_at) & ~neg
        if bad.any():
            rr, cc = bad.nonzero()[0].tolist()
            raise AssertionError(f"{what}: {int(bad.sum())} values out of bound; first at query {rr} rank {cc} index "
                                 f"{idx[rr, cc].item()}: val {v[rr, cc].item():.9g} ref {r_at[rr, cc].item():.9g} "
                                 f"err {err[rr, cc].item():.3g} tol {s_at[rr, cc].item():.3g}")
        if key is not None and (~neg).any():
            _note(key, (err / s_at)[~neg].max().item())
    chosen = torch.zeros(n, m, dtype=torch.int32, device=dev).scatter_add_(1, g, (~neg).int()) > 0
    lo_chosen = torch.where(neg, torch.full_like(r_at, float("inf")), r_at + s_at).amin(1)
    left = torch.where(chosen | torch.isnan(ref), torch.full_like(ref, float("-inf")), ref - slack).amax(1)
    full = valid[:, 0] >= k
    bad = full & (left > lo_chosen)
    if bad.any():
        rr = bad.nonzero()[0, 0].item()
        c = torch.where(chosen[rr] | torch.isnan(ref[rr]), float("-inf"), ref[rr] - slack[rr]).argmax().item()
        raise AssertionError(f"{what}: query {rr} leaves out index {c} (ref {ref[rr, c].item():.9g} slack "
                             f"{slack[rr, c].item():.3g}) though it beats a chosen score ({lo_chosen[rr].item():.9g} "
                             f"with slack)")


# ------------------------------------------------------------------------------------------------------------------
# Input families
# ------------------------------------------------------------------------------------------------------------------
FAMILIES = ("randn", "logmag", "exact_max", "spike", "parallel", "orthogonal", "golden")
EXACT_MAX = (1.0, 32.0, 64.0, 2.0 ** -10)


def _golden_embeds():
    import os
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "clip_golden.npz"))
    return (torch.from_numpy(d["image_embeds"]), torch.from_numpy(d["text_embeds"]),
            float(d["logit_scale_exp"]))


def golden_logit_scale():
    return _golden_embeds()[2]


def make_pair(family, n, m, seed, device):
    """fp32 operands a [n, 512], b [m, 512] of one input family:
      randn       N(0, 1)
      logmag      N(0, 1) rows times 2^u, u uniform in [-20, 20] per row
      exact_max   rows whose max |x| is exactly 1, 32, 64 or 2^-10 (in turn): the frexpf edge of the [32, 64) scaling
      spike       N(0, 1) 2^-12 with one entry +-1 per row, at a different position in a and b: lo parts of the
                  other entries are fp16 subnormals, and the spike of b meets a's subnormal lo parts
      parallel    a_i = b_(i mod m) + 1e-3 relative noise: cos within 1e-6 of 1, the top-1 regime of retrieval
      orthogonal  a_i orthogonal to b_(i mod m) up to fp32 rounding: logits near zero next to N(0, 1) ones
      golden      the reference's image_embeds (a) and text_embeds (b), replicated with 1e-4 relative noise"""
    g = torch.Generator().manual_seed(seed)
    if family == "golden":
        img, txt, _ = _golden_embeds()
        a = img[torch.arange(n) % img.shape[0]]
        b = txt[torch.arange(m) % txt.shape[0]]
        a = a + 1e-4 * a.abs().mean() * torch.randn(n, K_PROJ, generator=g)
        b = b + 1e-4 * b.abs().mean() * torch.randn(m, K_PROJ, generator=g)
        return a.float().contiguous().to(device), b.float().contiguous().to(device)
    a = torch.randn(n, K_PROJ, generator=g)
    b = torch.randn(m, K_PROJ, generator=g)
    if family == "logmag":
        a = a * torch.exp2(torch.rand(n, 1, generator=g) * 40 - 20)
        b = b * torch.exp2(torch.rand(m, 1, generator=g) * 40 - 20)
    elif family == "exact_max":
        for x in (a, b):
            x /= x.abs().amax(-1, keepdim=True)                   # the largest entry becomes exactly +-1
            x *= torch.tensor(EXACT_MAX)[torch.arange(x.shape[0]) % len(EXACT_MAX)][:, None]
    elif family == "spike":
        for x, step, off in ((a, 7, 0), (b, 13, 5)):
            x *= 2.0 ** -12
            r = torch.arange(x.shape[0])
            x[r, (r * step + off) % K_PROJ] = torch.where(torch.rand(x.shape[0], generator=g) < 0.5, -1.0, 1.0)
    elif family == "parallel":
        base = b[torch.arange(n) % m]
        a = base + 1e-3 * base.norm(dim=-1, keepdim=True) / math.sqrt(K_PROJ) * torch.randn(n, K_PROJ, generator=g)
    elif family == "orthogonal":
        base = b[torch.arange(n) % m].double()
        a64 = a.double()
        a = (a64 - (a64 * base).sum(-1, keepdim=True) / (base * base).sum(-1, keepdim=True) * base).float()
    else:
        assert family == "randn", family
    return a.float().contiguous().to(device), b.float().contiguous().to(device)
