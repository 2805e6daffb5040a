"""float64 references of the attention kernels (attention.cu) and the per-element acceptance the GPU suites share.

`attention_contract_ref` is what attention_kernel (S <= 128, one key block) is specified to compute,
`long_attention_contract_ref` / `long_chain_slack` what attention_long_kernel (128 < S <= 1025, 64-key blocks with an
online softmax) is, and `probs_contract_ref` what attention_probs_kernel writes.  All of them start from the 16-bit
q, k, v the kernel reads.  They live in their own module so that several test modules can import them without pytest
collecting one test module from another.
"""
import torch

DT = {0: torch.bfloat16, 1: torch.float16}
REL = {0: 2.0 ** -8, 1: 2.0 ** -11}      # round-to-nearest into the 16-bit output: half an ulp <= this much of |x|
U32 = 2.0 ** -23                         # one fp32 ulp, relative
SENT = -1536.0        # exactly representable in bf16, fp16 and fp32; no operand or result below comes near it

# Absolute slack of the attention output next to one ulp of the 16-bit result: the kernel's p carries ~1e-5 relative
# error (fp32 scores of magnitude <= ~100, ex2.approx), so the output moves by that much of sum_k p_k |v_k| / rowsum
# <= max |v| ~ 5 for N(0,1) inputs; the fp32 accumulation of P V adds 2^-23-ish of the same.  2e-4 covers both.
ATT_ABS = 2e-4

KEY_BLOCK = 64                           # keys per block of the long and the probabilities kernel

# largest err / tolerance seen per bound in this run; the GPU suites write it to $PLIP_EDGE_REPORT (JSON) when set
OBSERVED = {}


def _note(key, ratio):
    OBSERVED[key] = max(OBSERVED.get(key, 0.0), float(ratio))


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _round_to(x64, dt):
    return x64.float().to(dt).double()


def _ulp_of(x64, fmt):
    """Spacing of the 16-bit format in the binade of |x|; fp16 subnormals have a fixed spacing."""
    _, e = torch.frexp(x64)                                   # x = m 2^e, m in [0.5, 1)
    e = e.double() - (8 if fmt == 0 else 11)
    if fmt == 1:
        e = e.clamp_min(-24.0)
    return torch.exp2(e)


def attention_contract_ref(qkv, n_seq, S, heads, causal, mask, fmt):
    """What attention_kernel is specified to compute, in float64, per (sequence, head):
         s = q k^T (no scale: dh^-0.5 lives in the packed q weights), masked keys -> -inf,
         p = exp(s - rowmax),  rowsum over the UNROUNDED p,  o = (round16(p) @ v) / rowsum.
    Returns (contract, plain, flip), [n_seq * S, heads * 64] float64 each: `plain` is the ordinary softmax(s) @ v, and
    `flip` bounds what the output may move when p values that sit on a rounding boundary of the 16-bit format round
    the other way in the kernel: sum over such keys of ulp(p) |v| / rowsum.  The kernel's p differs from the float64
    one by the error of its fp32 score and of the row maximum (4 k16 steps, each 2^-23 of at most sum_d |q_d k_d|),
    by the rounding of the exp2 argument (2^-24 of its magnitude) and by ex2.approx (2 ulp).  A row without a visible key gives NaN here (the kernel returns zeros;
    the cases below keep key 0 visible)."""
    D = heads * 64
    q, k, v = qkv.double().view(n_seq, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2)
    if causal:
        s = s + torch.full((S, S), float("-inf"), device=qkv.device, dtype=torch.float64).triu(1)
    if mask is not None:
        s = s.masked_fill((mask == 0)[:, None, None, :], float("-inf"))
    p = torch.exp(s - s.amax(-1, keepdim=True))
    rowsum = p.sum(-1, keepdim=True)
    pr = _round_to(p, DT[fmt])
    ulp = _ulp_of(p, fmt)                                     # of p, not pr: just below a power of two the grid is finer
    mag = q.abs() @ k.abs().transpose(-1, -2)
    p_rel = 4 * U32 * (mag + mag.amax(-1, keepdim=True)) + 1.5 * 2.0 ** -24 * (s - s.amax(-1, keepdim=True)).abs() + 1e-6
    near = (0.5 - (p - pr).abs() / ulp) < p_rel * p / ulp     # distance from the rounding boundary, in ulps
    near &= p > 0
    flip = ((ulp * near) @ v.abs()) / rowsum
    contract = (pr @ v) / rowsum
    plain = (p / rowsum) @ v

    def rows(t):
        return t.permute(0, 2, 1, 3).reshape(n_seq * S, D)
    return rows(contract), rows(plain), rows(flip)


def _heads_view(qkv, n_seq, S, heads):
    """q, k, v as float64 [n_seq, heads, S, 64]."""
    return qkv.double().view(n_seq, S, 3, heads, 64).permute(2, 0, 3, 1, 4)


def _rows(t, n_seq, S, heads):
    return t.permute(0, 2, 1, 3).reshape(n_seq * S, heads * 64)


def running_block_max(s):
    """The online softmax's row maxima over 64-key blocks taken in order.  s: float64 [..., S_q, S_k], masked keys -inf.
    Returns (m_key, m_last, chain): m_key [..., S_q, S_k] is m_b, the running maximum after the block that holds the
    key; m_last [..., S_q, 1] the maximum over all keys; chain [..., S_q, 1] the relative error budget of the
    kernel's rescale chain (derivation in long_attention_contract_ref): per block transition c = 1 .. n_kb - 1 after
    a visible key,  2^-24 (|m_{c-1}| + |m_c - m_{c-1}|) + 3 x 2^-23."""
    S = s.shape[-1]
    n_kb = (S + KEY_BLOCK - 1) // KEY_BLOCK
    pad = torch.full(s.shape[:-1] + (n_kb * KEY_BLOCK - S,), float("-inf"), dtype=s.dtype, device=s.device)
    m = torch.cat([s, pad], -1).view(*s.shape[:-1], n_kb, KEY_BLOCK).amax(-1).cummax(-1).values
    m_key = m.repeat_interleave(KEY_BLOCK, -1)[..., :S]
    prev, cur = m[..., :-1], m[..., 1:]
    link = 2.0 ** -24 * (prev.abs() + (cur - prev).abs()) + 3 * U32
    chain = torch.where(torch.isfinite(prev), link, torch.zeros_like(link)).sum(-1, keepdim=True)
    return m_key, m[..., -1:], chain


def long_attention_contract_ref(qkv, n_seq, S, heads, fmt):
    """What attention_long_kernel is specified to compute, in float64, per (sequence, head): keys in blocks
    b = 0, 1, .. of 64 taken in order, s = q k^T, m_b the running row maximum after block b (running_block_max),
         l = sum_b exp(m_b - m_last) sum_{k in b} exp(s_k - m_b)          over the UNROUNDED p,
         o = sum_b exp(m_b - m_last) round16(exp(s_b - m_b)) @ v_b,      out = o / l.
    The 16-bit P of a block is rounded against the block's running maximum, before any later rescale:
    round16(exp(s - m_b)) e^(m_b - m_last) is not round16(exp(s - m_last)), so attention_contract_ref (rounded against
    the final maximum) is this reference only when S <= 64.  Returns (contract, plain, flip) as attention_contract_ref
    does, `flip` built per block against p = exp(s - m_b) and carried by the block's weight exp(m_b - m_last).

    The rescale chain (long_chain_slack).  The kernel weighs block b by alpha_{b+1} ... alpha_last with
    alpha_c = ex2(m_{c-1} log2e - ms_c) and takes the block's exps as ex2(s log2e - ms_b), ms_c = m_c log2e rounded to
    fp32 (row_shift).  The score error of m_c cancels between consecutive factors and the exps, so exactly rounded, the
    product would be exp(s - m_last) up to one factor common to every block (which cancels in o / l).  What does not
    cancel, per factor alpha_c, relative:
         the rounding of ms_{c-1}                 <= 2^-24 |m_{c-1} log2e| ln 2 = 2^-24 |m_{c-1}|
         the rounding of the fmaf argument        <= 2^-24 |m_c - m_{c-1}|   (+ 2^-24 |ms_c - m_c log2e|, negligible)
         ex2.approx                               <= 2 ulp = 2 x 2^-23
         the products l *= alpha and o *= alpha   <= 2^-24 each
    S = 1025 has 17 key blocks and so 17 factors in a chain; the first multiplies the zeros the row starts from, which
    leaves 16 that count.  With every block weight off by a relative delta_b, |delta_b| <= chain (summed over the
    factors), the output o / l moves by at most
         chain (sum_b w_b |round16(p_b)| @ |v_b| + |out| l) / l <= 2 (1 + 2^-8) chain (p @ |v|) / l,
    which long_chain_slack returns (with 2.1 for the factor and e^chain - 1 > chain).  The per-key errors of p (score,
    exp2 argument, ex2.approx of the exps) are those of attention_kernel and stay in ATT_ABS."""
    q, k, v = _heads_view(qkv, n_seq, S, heads)
    s = q @ k.transpose(-1, -2)
    m_key, m_last, _ = running_block_max(s)
    p = torch.exp(s - m_key)                                  # against the block's running maximum
    w = torch.exp(m_key - m_last)                             # what the later rescales make of the block
    rowsum = (w * p).sum(-1, keepdim=True)
    pr = _round_to(p, DT[fmt])
    ulp = _ulp_of(p, fmt)
    mag = q.abs() @ k.abs().transpose(-1, -2)
    p_rel = 4 * U32 * (mag + mag.amax(-1, keepdim=True)) + 1.5 * 2.0 ** -24 * (s - m_key).abs() + 1e-6
    near = (0.5 - (p - pr).abs() / ulp) < p_rel * p / ulp
    near &= p > 0
    flip = ((w * ulp * near) @ v.abs()) / rowsum
    contract = ((w * pr) @ v) / rowsum
    pf = torch.exp(s - m_last)
    plain = (pf / pf.sum(-1, keepdim=True)) @ v
    return _rows(contract, n_seq, S, heads), _rows(plain, n_seq, S, heads), _rows(flip, n_seq, S, heads)


def long_chain_slack(qkv, n_seq, S, heads):
    """Absolute slack of attention_long_kernel's rescale chain, [n_seq * S, heads * 64] float64:
    2.1 chain (p @ |v|) / l (derivation in long_attention_contract_ref)."""
    q, k, v = _heads_view(qkv, n_seq, S, heads)
    s = q @ k.transpose(-1, -2)
    _, m_last, chain = running_block_max(s)
    p = torch.exp(s - m_last)
    return _rows(2.1 * chain * (p @ v.abs()) / p.sum(-1, keepdim=True), n_seq, S, heads)


def probs_contract_ref(qkv, n_seq, S, heads, causal, mask):
    """What attention_probs_kernel writes, in float64: P = softmax(q k^T) over the visible keys ([n_seq, heads, S, S];
    masked entries and rows without a visible key are 0), and the relative bound `rel` of the same shape its fp32
    arithmetic is entitled to, per element:
         4 x 2^-23 (|q| |k_j| + max_k |q| |k_k|)    the fp32 score of the entry and those that dominate the row sum
         1.5 x 2^-24 |s_j - m|                       the rounding of the exp2 argument
         2 x 2 x 2^-23                               ex2.approx of the entry and of the row sum's terms
         chain                                       the rescale chain of l (running_block_max; the entry is taken
                                                     against the final maximum, every block of l through its factors)
         (16 n_kb + 4) x 2^-24                       l summed in fp32: 16 terms per block and thread, two shuffle adds,
                                                     the reciprocal and the product
    The kernel flushes exps below 2^-126 to zero; callers add an absolute slack far below anything that matters."""
    q, k, _ = _heads_view(qkv, n_seq, S, heads)
    s = q @ k.transpose(-1, -2)
    if causal:
        s = s + torch.full((S, S), float("-inf"), device=qkv.device, dtype=torch.float64).triu(1)
    if mask is not None:
        s = s.masked_fill((mask == 0)[:, None, None, :], float("-inf"))
    vis = torch.isfinite(s)
    _, m_last, chain = running_block_max(s)
    m_safe = torch.where(torch.isfinite(m_last), m_last, torch.zeros_like(m_last))
    p = torch.where(vis, torch.exp(s - m_safe), torch.zeros_like(s))
    rowsum = p.sum(-1, keepdim=True)
    probs = torch.where(rowsum > 0, p / rowsum.clamp_min(1e-300), torch.zeros_like(p))
    mag = q.abs() @ k.abs().transpose(-1, -2)
    n_kb = (S + KEY_BLOCK - 1) // KEY_BLOCK
    rel = (4 * U32 * (mag + mag.amax(-1, keepdim=True)) + 1.5 * 2.0 ** -24 * torch.where(vis, s - m_safe, 0.0).abs()
           + 4 * U32 + chain + (16 * n_kb + 4) * 2.0 ** -24)
    return probs, torch.where(vis, rel, torch.zeros_like(rel))


def _first_bad(bad, err, tol, out, ref, what, where=None):
    r, c = bad.nonzero()[0].tolist()
    msg = (f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bound; first at row {r} col {c}: "
           f"out {out[r, c].item():.9g} ref {ref[r, c].item():.9g} err {err[r, c].item():.3g} tol {tol[r, c].item():.3g}")
    if where is not None:
        msg += " (" + where(r, c) + ")"
    return msg


def assert_within(out, ref, slack, rel, key, what, where=None):
    out64 = out.double()
    err = (out64 - ref).abs()
    tol = rel * ref.abs() + slack
    bad = ~(err <= tol)                                       # NaN counts as bad
    assert not bad.any(), _first_bad(bad, err, tol, out64, ref, what, where)
    _note(key, (err / tol).max().item())
