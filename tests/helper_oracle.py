"""float64 references of the helper kernels around the towers' GEMMs (elementwise.cu), with the per-element slack each
kernel's fp32 arithmetic is entitled to.

  layernorm_kernel       layernorm_ref (+ layernorm_slack), layernorm_emulate (the kernel's op order in fp32)
  rowstats_cast_kernel   rowstats_ref
  im2col_kernel          im2col_ref, u8_table
  text_embed_kernel      text_embed_ref
  eos_row_kernel         pooled_rows_ref
  mask_to_i32_kernel     mask_ref
  cls_rows_kernel        cls_rows_ref
  gather_rows_kernel     gather_rows_ref
  pos_interp_kernel      cubic_taps32, pos_interp_ref

Everything here runs on the CPU; tests/test_helper_oracle.py holds the references to torch's own operators and
checks that they reject planted mistakes, tests/test_gpu_helper_contract.py holds the kernels to them.

Notation: u = 2^-24 is the unit roundoff of fp32 (round to nearest), gamma(n) = n u / (1 - n u) bounds the relative
error of n successive roundings, and an fp32 sum whose every term passes through at most n additions is within
gamma(n) sum |x_i| of the exact sum (Higham, Accuracy and Stability of Numerical Algorithms, §4.2).  These are worst-case
bounds, not random-walk estimates.
"""
from fractions import Fraction
from functools import lru_cache

import numpy as np
import torch

U = 2.0 ** -24
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
EOS_ID = 49407
VOCAB = 49408
LN_EPS = 1e-5
GRID = 7                                  # the stored vision position table is 7 x 7 patches (+ the class row)


def gamma(n):
    return n * U / (1 - n * U)


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------------------------
def layernorm_ref(x, g, b, eps=LN_EPS):
    """(x - mean) / sqrt(var + eps) * g + b per row in float64, var the biased (1/D) variance.  [rows, D]."""
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    var = (d * d).mean(-1, keepdim=True)
    return d / torch.sqrt(var + eps) * g.double() + b.double()


def layernorm_slack(x, g, b, eps=LN_EPS):
    """Per-element bound on |kernel - layernorm_ref| for layernorm_kernel<D> (D = 128 V), [rows, D] float64.

    The kernel's op order (one warp per row, each lane holding V float4):
      s    = butterfly sum over 5 levels of the lane sums  sum_j (x0 + x1) + (x2 + x3): every x passes through at most
             2 + V additions in its lane and 5 in the butterfly, so |s - S| <= gamma(V + 7) sum|x|.
      d    = FFMA(-s, fl(1/D), x): the subtracted value differs from mean = S / D by at most
             e_mu = gamma(V + 7) sum|x| / D + 2 u |mean|  (fl(1/D) is off by u relative, and a build that rounds the
             mean before subtracting adds another u |mean|), and the FFMA rounds once: e_d = e_mu + u (|d| + e_mu).
      q    = the same sum tree over the products d*d: |q - sum d^2| <= sum e_d (2|d| + e_d) + gamma(V + 8) sum (|d| + e_d)^2.
      v    = FFMA(q, fl(1/D), eps): e_v = (e_q + u q) / D + u (v + (e_q + u q) / D).
      rstd = rsqrtf(v): 2 ulp (2^-22 relative) of rsqrt of the computed v, which is itself off by e_v, so
             |rstd - 1/sqrt(v)| <= (e_v / (2 (v - e_v)) + 2^-22) / sqrt(v)  (rsqrt's derivative, taken at the lower end).
      y    = FFMA(g, fl(d * rstd), b): e_t = e_d r (1 + rel_r) + |d| r rel_r + u (|d| r + ...), e_y = |g| e_t + u (|y| + |g| e_t).
    A factor 1 + 2^-20 on the result covers the float64 evaluation of the bound itself."""
    x = x.double()
    D = x.shape[-1]
    V = D // 128
    g, b = g.double(), b.double()
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    A = x.abs().sum(-1, keepdim=True)
    e_mu = gamma(V + 7) * A / D + 2 * U * mu.abs()
    e_d = e_mu + U * (d.abs() + e_mu)
    Q = (d * d).sum(-1, keepdim=True)
    e_q = (e_d * (2 * d.abs() + e_d)).sum(-1, keepdim=True) + gamma(V + 8) * ((d.abs() + e_d) ** 2).sum(-1, keepdim=True)
    v = Q / D + eps
    e_v0 = (e_q + U * Q) / D
    e_v = e_v0 + U * (v + e_v0)
    r = 1.0 / torch.sqrt(v)
    rel_r = e_v / (2 * (v - e_v)) + 2.0 ** -22
    rel_r = rel_r * (1 + rel_r)                       # second-order term of the perturbed square root
    t = d.abs() * r
    e_t = e_d * r * (1 + rel_r) + t * rel_r
    e_t = e_t + U * (t + e_t)
    y = (d * r * g + b).abs()
    e_y = g.abs() * e_t
    e_y = e_y + U * (y + e_y)
    return e_y * (1 + 2.0 ** -20)


def layernorm_emulate(x, g, b, eps=LN_EPS, *, one_pass=False, eps_outside=False, unbiased=False):
    """layernorm_kernel's op order in fp32 on the CPU (sums in the kernel's tree; products and the centring rounded
    separately, which layernorm_slack also covers).  The keyword arguments plant the mistakes a LayerNorm kernel makes:
    one_pass = var from E[x^2] - mean^2, eps_outside = 1 / (sqrt(var) + eps), unbiased = var / (D - 1)."""
    x = x.float()
    R, D = x.shape
    V = D // 128

    def tree_sum(t):                     # [R, D] -> [R], lane sums over V float4 then 5 butterfly levels
        t4 = t.view(R, V, 32, 4)                                   # element (j, lane, k) = t[:, 128 j + 4 lane + k]
        lane = torch.zeros(R, 32, dtype=torch.float32)
        for j in range(V):
            q = t4[:, j]
            lane = lane + ((q[..., 0] + q[..., 1]) + (q[..., 2] + q[..., 3]))
        for o in (16, 8, 4, 2, 1):
            lane = lane + lane[:, torch.arange(32) ^ o]
        return lane[:, 0]

    inv_d = torch.tensor(1.0 / D, dtype=torch.float32)
    s = tree_sum(x)
    mean = (s * inv_d)[:, None]
    d = x - mean
    if one_pass:
        var = tree_sum(x * x)[:, None] * inv_d - mean * mean
    else:
        var = tree_sum(d * d)[:, None] * (1.0 / (D - 1) if unbiased else inv_d)
    var = var.float()
    eps32 = torch.tensor(eps, dtype=torch.float32)
    rstd = 1.0 / (torch.sqrt(var) + eps32) if eps_outside else torch.rsqrt(var + eps32)
    return (d * rstd) * g.float() + b.float()


# ------------------------------------------------------------------------------------------------------------------
# Row statistics
# ------------------------------------------------------------------------------------------------------------------
def rowstats_ref(x):
    """(sum x, sum x^2) per row in float64 and their slack for rowstats_cast_kernel<D>: the same lane / butterfly sum
    tree as the LayerNorm's, so |s1 - sum x| <= gamma(V + 7) sum |x| and, with one more rounding for the product (or
    the FFMA that absorbs it), |s2 - sum x^2| <= gamma(V + 8) sum x^2.  Returns (s1, s2, tol1, tol2), [rows] each."""
    x = x.double()
    V = x.shape[-1] // 128
    return (x.sum(-1), (x * x).sum(-1), gamma(V + 7) * x.abs().sum(-1), gamma(V + 8) * (x * x).sum(-1))


# ------------------------------------------------------------------------------------------------------------------
# im2col
# ------------------------------------------------------------------------------------------------------------------
def _f32(v):
    return np.float32(v)


def u8_table(*, swap_means=False):
    """The 3 x 256 values im2col_kernel<U8> can produce before the 16-bit cast, float32 [3, 256]:
    fl(fl(FFMA(byte, fl(1/255), -fl(mean_c))) * fl(1 / fl(std_c))).  byte * fl(1/255) - fl(mean_c) is exact in float64
    (a 32-bit integer times 2^-31 plus a 24-bit mantissa at 2^-25), so one float64 -> float32 rounding is the FFMA's,
    and the product of two floats is exact in float64 as well.  swap_means plants swapped means of channels 0 and 1."""
    c255 = np.float64(_f32(1.0) / _f32(255.0))
    mean = [np.float64(_f32(m)) for m in CLIP_MEAN]
    if swap_means:
        mean[0], mean[1] = mean[1], mean[0]
    istd = [np.float64(_f32(1.0) / _f32(s)) for s in CLIP_STD]
    byte = np.arange(256, dtype=np.float64)
    out = np.empty((3, 256), np.float32)
    for c in range(3):
        t = (byte * c255 - mean[c]).astype(np.float32).astype(np.float64)
        out[c] = (t * istd[c]).astype(np.float32)
    return torch.from_numpy(out)


def im2col_ref(pixels, fmt, dt, *, swap_k=False):
    """What im2col_kernel<fmt> writes for pixels (f32 / bf16 [n, 3, H, W], or uint8 [n, H, W, 3]) in the 16-bit
    operand type dt: [n * gh * gw, 3072], row b * gh * gw + py * gw + px, column c * 1024 + ky * 32 + kx from pixel
    (py * 32 + ky, px * 32 + kx); the last H % 32 rows and W % 32 columns are not read.  Bit exact:
      f32   the RNE cast to dt;
      bf16  a copy, or bf16 -> fp32 -> fp16 (RNE) for fp16 operands;
      u8    u8_table, then the RNE cast.
    swap_k plants swapped ky / kx."""
    if fmt == 2:
        n, H, W, _ = pixels.shape
        vals = u8_table().to(pixels.device)                                # [3, 256]
        chw = pixels.permute(0, 3, 1, 2).long()
        x = torch.stack([vals[c][chw[:, c]] for c in range(3)], 1)         # float32 [n, 3, H, W]
    else:
        n, _, H, W = pixels.shape
        x = pixels.float()
    gh, gw = H // 32, W // 32
    x = x[:, :, :gh * 32, :gw * 32].reshape(n, 3, gh, 32, gw, 32)
    x = x.permute(0, 2, 4, 1, 5, 3) if swap_k else x.permute(0, 2, 4, 1, 3, 5)
    return x.reshape(n * gh * gw, 3072).to(dt)


# ------------------------------------------------------------------------------------------------------------------
# Text embeddings, pooled rows, key mask
# ------------------------------------------------------------------------------------------------------------------
def text_embed_ref(ids, seq_len, tok, pos):
    """x[b * seq_len + t] = fl32(tok[clamp(ids[b, t], 0, 49407)] + pos[t]) for the first seq_len ids of each row,
    bit exact (one fp32 addition).  [n * seq_len, 512] float32."""
    idx = ids[:, :seq_len].long().clamp(0, VOCAB - 1)
    return (tok[idx] + pos[:seq_len][None]).reshape(-1, tok.shape[1])


def pooled_rows_ref(ids, seq_len, argmax_mode, *, last_eos=False, later_tie=False):
    """The pooled row b * seq_len + t of each caption, looking at the first seq_len ids only (HF CLIPTextTransformer):
      t = the first position of eos (49407) if there is one;
      else 0 in mode 0 ((ids == eos).int().argmax(-1) of all zeros) and, in mode 1 (legacy configs, OpenAI CLIP),
      the first position of the largest id (ids.argmax(-1); torch.argmax returns the first maximal index).
    Raw ids are compared, before the clamp the embedding applies.  last_eos / later_tie plant the last eos and ties
    resolved to the later position.  int64 [n]."""
    ids = ids[:, :seq_len].long()
    n = ids.shape[0]
    out = torch.empty(n, dtype=torch.int64)
    for b in range(n):
        row = ids[b].tolist()
        hits = [t for t, v in enumerate(row) if v == EOS_ID]
        if hits:
            t = hits[-1] if last_eos else hits[0]
        elif argmax_mode:
            m = max(row)
            ties = [t for t, v in enumerate(row) if v == m]
            t = ties[-1] if later_tie else ties[0]
        else:
            t = 0
        out[b] = b * seq_len + t
    return out


def mask_ref(mask, seq_len, *, truncate_i32=False):
    """mask[:, :seq_len] != 0 as int32, flattened: transformers turns the attention mask into a boolean with
    .to(torch.bool), so any nonzero value attends, including an int64 value whose low 32 bits are zero.
    truncate_i32 plants a cast to int32 before the test."""
    m = mask[:, :seq_len]
    if truncate_i32:
        m = m.to(torch.int32)
    return (m != 0).to(torch.int32).reshape(-1)


def cls_rows_ref(cls, pos0):
    """The class row cls + pos[0] in fp32, bit exact (one addition)."""
    return cls.float() + pos0.float()


def gather_rows_ref(src, n, row_index=None, row_stride=0):
    """Rows row_index[i] (or i * row_stride) of src, i < n: exact copies."""
    idx = row_index.long() if row_index is not None else torch.arange(n) * row_stride
    return src[idx]


# ------------------------------------------------------------------------------------------------------------------
# Position table
# ------------------------------------------------------------------------------------------------------------------
def _round32(q):
    """A rational rounded to the nearest float32 (ties to even), exactly; normal range only (all this module needs)."""
    if q == 0:
        return 0.0
    s = -1 if q < 0 else 1
    q = abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1                                              # now 2^e <= q < 2^(e + 1)
    m = round(q * Fraction(2) ** (23 - e))                   # Fraction rounds half to even
    return s * float(m) * 2.0 ** (e - 23)


def _fma32(a, b, c):
    return _round32(Fraction(a) * Fraction(b) + Fraction(c))


def _add32(a, b):
    return _round32(Fraction(a) + Fraction(b))


def _mul32(a, b):
    return _round32(Fraction(a) * Fraction(b))


@lru_cache(maxsize=None)
def cubic_taps32(g, i, align_corners=False, clamp_hi=GRID - 1):
    """cubic_taps(g, i) of pos_interp_kernel as the sm_90a build computes it, every operation an fp32 rounding:
      scale = fl(7 / g); real = FFMA(fl(i + 0.5), scale, -0.5); t = fl(real - floor(real)) (exact unless real < 0);
      t1 = fl(t + 1), t2 = fl(1 - t), t3 = fl(2 - t);
      w0 = FFMA(t1, FFMA(t1, FFMA(t1, -0.75, 3.75), -6), 3)          (((A t1 - 5A) t1 + 8A) t1 - 4A, A = -0.75)
      w1 = FFMA(t, fl(t * FFMA(t, 1.25, -2.25)), 1)                   (((A + 2) t - (A + 3)) t t + 1)
      w2 = the same in t2, w3 = w0's polynomial in t3;  taps clamp(floor(real) - 1 + k, 0, 6).
    Returns (taps, weights) as tuples.  align_corners / clamp_hi plant the source coordinate of align_corners=True
    and taps clamped to [0, clamp_hi]."""
    if align_corners:
        real = 0.0 if g == 1 else _mul32(_round32(Fraction(GRID - 1) / Fraction(g - 1)), float(i))
    else:
        scale = _round32(Fraction(GRID) / Fraction(g))
        real = _fma32(float(i) + 0.5, scale, -0.5)
    fl = float(np.floor(real))
    t = _add32(real, -fl)                                   # rounds when real < 0 (i = 0 of an upscale)
    t1, t2, t3 = _add32(t, 1.0), _add32(1.0, -t), _add32(2.0, -t)

    def outer(s):
        return _fma32(s, _fma32(s, _fma32(s, -0.75, 3.75), -6.0), 3.0)

    def inner(s):
        return _fma32(s, _mul32(s, _fma32(s, 1.25, -2.25)), 1.0)

    w = (outer(t1), inner(t), inner(t2), outer(t3))
    taps = tuple(min(max(int(fl) - 1 + k, 0), clamp_hi) for k in range(4))
    return taps, w


def _interp_matrix(g, weights, **kw):
    """[g, 7] float64 resampling matrix of one axis (clamped taps accumulate), with |w| alongside; a planted tap past
    the grid (clamp_hi = 7) lands in an 8th column that reads zeros."""
    M = torch.zeros(g, GRID + 1, dtype=torch.float64)
    Ma = torch.zeros_like(M)
    for i in range(g):
        if weights == "fp32":
            taps, w = cubic_taps32(g, i, **kw)
        else:
            taps, w = cubic_taps64(g, i)
        for k in range(4):
            M[i, taps[k]] += w[k]
            Ma[i, taps[k]] += abs(w[k])
    return M, Ma


def cubic_taps64(g, i):
    """The same taps with float64 weights of the exact source coordinate: what F.interpolate computes in float64."""
    A = -0.75
    real = GRID / g * (i + 0.5) - 0.5
    fl = np.floor(real)
    t = real - fl

    def c1(s):
        return ((A + 2) * s - (A + 3)) * s * s + 1

    def c2(s):
        return ((A * s - 5 * A) * s + 8 * A) * s - 4 * A

    w = (c2(t + 1), c1(t), c1(1 - t), c2(2 - t))
    return tuple(min(max(int(fl) - 1 + k, 0), GRID - 1) for k in range(4)), w


def pos_interp_ref(pos, gh, gw, weights="fp32", **kw):
    """The [1 + gh * gw, 768] table pos_interp_kernel writes, in float64 from the fp32 weights of cubic_taps32, and
    its per-element slack.  Row 0 is pos[0] (an exact copy).  Row 1 + y * gw + x is sum_a wy_a sum_b wx_b p[iy_a, ix_b]:
    the kernel accumulates the four x taps with FFMAs into t, then the four t with FFMAs into acc, so every product
    passes through at most 4 + 4 roundings and |kernel - ref| <= gamma(8) sum_a |wy_a| sum_b |wx_b| |p[iy_a, ix_b]|.
    weights = "fp64" gives F.interpolate's float64 weights instead (and the slack between the two weight sets as the
    third value: sum |wy wx - wy64 wx64| |p|).  Returns (ref, slack) [or (ref, slack, weight_gap) for fp64]."""
    D = pos.shape[-1]
    p = pos[1:].double().reshape(GRID, GRID, D)
    p = torch.nn.functional.pad(p.permute(2, 0, 1), (0, 1, 0, 1)).permute(1, 2, 0)          # [8, 8, D], zero row/col 7
    My, May = _interp_matrix(gh, weights, **kw)
    Mx, Max = _interp_matrix(gw, weights, **kw)
    ref = torch.einsum("ya,xb,abd->yxd", My, Mx, p).reshape(gh * gw, D)
    slack = gamma(8) * torch.einsum("ya,xb,abd->yxd", May, Max, p.abs()).reshape(gh * gw, D)
    ref = torch.cat([pos[:1].double(), ref], 0)
    slack = torch.cat([torch.zeros(1, D, dtype=torch.float64), slack], 0) * (1 + 2.0 ** -20)
    if weights == "fp64":
        My32, _ = _interp_matrix(gh, "fp32")
        Mx32, _ = _interp_matrix(gw, "fp32")
        wy, wx = (My32 - My), (Mx32 - Mx)
        gap = (torch.einsum("ya,xb,abd->yxd", (My32.abs() + My.abs()), wx.abs(), p.abs())
               + torch.einsum("ya,xb,abd->yxd", wy.abs(), Mx.abs(), p.abs())).reshape(gh * gw, D)
        return ref, slack, torch.cat([torch.zeros(1, D, dtype=torch.float64), gap], 0)
    return ref, slack
