"""float64 contracts of the DenseNet-121 kernels (densenet.cu) and the per-element slack each is entitled to.

Each reference starts from the operands the kernel reads and restates what it is specified to compute, following the
module comment of densenet.cu:

  A operand (bit-exact, no slack): formed in torch fp32 in the kernel's order and rounded to bf16 once.
    stem_a     bf16(((u8 / 255) - mean) / std), K = (ky, kx, c) = 147; out-of-image taps and K-pad columns 147..159 are 0
    preact_a   bf16(relu((x * s) + b)), two fp32 roundings before the ReLU
    pool_a     bf16((((r00 + r01) + r10) + r11) * 0.25), r = relu((x * s) + b) in fp32
    tap3_a     the stored bottleneck, K = (ky, kx, c) = 1152, zeros outside the image
  Accumulator: acc = A W^T in float64; slack 2 x 2^-23 sqrt(K / 16) sum_k |a_k| |w_k| (acc_ref).
  Epilogues:   kEpiBnRelu relu(fl(fl(acc s) + b)) (bn_relu_ref), kEpiStore acc; then one rounding to bf16, checked
               per element by attention_oracle.assert_within with REL[0] = 2^-8.
  Max pool:    exact (maxpool_ref).
  Tail:        exact against a sequential fp32 restatement (tail_ref).

Everything works on CPU and CUDA tensors alike.  Divisions go through tensor divisors, never a Python scalar: on the
GPU torch turns `t / 255.0` into a multiplication by the reciprocal, which is not the kernel's __fdiv_rn.
"""
import math

import torch

from attention_oracle import REL, U32, _bits, assert_within

BF = torch.bfloat16
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
STEM_K, STEM_KPAD = 147, 160


def _full(t, v):
    return torch.full_like(t, v)


# ---- A operands ---------------------------------------------------------------------------------------------------
def stem_a(tiles):
    """uint8 [n, H, W, 3] -> bf16 [n (H / 2) (W / 2), 160]: conv0's 7x7 / s2 / p3 A operand, K order (ky, kx, c)."""
    n, H, W, _ = tiles.shape
    x = tiles.float()
    x = x / _full(x, 255.0)
    mean = torch.tensor(MEAN, dtype=torch.float32, device=x.device)
    std = torch.tensor(STD, dtype=torch.float32, device=x.device)
    x = ((x - mean) / std).to(BF)
    xp = torch.zeros(n, H + 6, W + 6, 3, dtype=BF, device=x.device)   # zero padding after the normalisation
    xp[:, 3:H + 3, 3:W + 3] = x
    cols = xp.unfold(1, 7, 2).unfold(2, 7, 2)                        # [n, H / 2, W / 2, 3, ky, kx]
    cols = cols.permute(0, 1, 2, 4, 5, 3).reshape(-1, STEM_K)
    return torch.cat([cols, torch.zeros(cols.shape[0], STEM_KPAD - STEM_K, dtype=BF, device=x.device)], 1)


def preact_a(x, c_in, s, b):
    """bf16 rows [M, lda] -> bf16 [M, c_in]: conv1's A operand, relu(x s + b) per K column."""
    return torch.relu(x[:, :c_in].float() * s + b).to(BF)


def pool_r(x, c_in, s, b):
    """fp32 (((r00 + r01) + r10) + r11) * 0.25 of bf16 [n, 2 side, 2 side, lda], r = relu(x s + b): [n, side, side, c_in]."""
    r = torch.relu(x[..., :c_in].float() * s + b)
    return (((r[:, 0::2, 0::2] + r[:, 0::2, 1::2]) + r[:, 1::2, 0::2]) + r[:, 1::2, 1::2]) * 0.25


def pool_a(x, c_in, s, b):
    """The transition's A operand: bf16 [n side^2, c_in]."""
    return pool_r(x, c_in, s, b).to(BF).reshape(-1, c_in)


def tap3_a(neck):
    """bf16 [n, side, side, 128] -> bf16 [n side^2, 1152]: conv2's 3x3 / p1 A operand, K order (ky, kx, c)."""
    n, side, _, c = neck.shape
    xp = torch.zeros(n, side + 2, side + 2, c, dtype=neck.dtype, device=neck.device)
    xp[:, 1:side + 1, 1:side + 1] = neck
    cols = xp.unfold(1, 3, 1).unfold(2, 3, 1)                        # [n, side, side, c, ky, kx]
    return cols.permute(0, 1, 2, 4, 5, 3).reshape(-1, 9 * c)


def conv_weight_k(w4):
    """[N, C, kh, kw] -> [N, kh kw C]: the kernels' (ky, kx, c) K order."""
    return w4.permute(0, 2, 3, 1).reshape(w4.shape[0], -1)


# ---- accumulator and epilogues ------------------------------------------------------------------------------------
def acc_ref(A, W):
    """acc = A W^T in float64 and its slack, both [M, N].

    mma.sync m16n8k16 adds the 16 exact products of a k16 step to the fp32 accumulator with one rounding (or
    truncation: 2^-23 relative to the running sum) per step, K / 16 steps.  For operands with random signs the errors
    add like a random walk and the running sum stays far below sum_k |a_k w_k|, so
        |acc_kernel - acc| <= 2 x 2^-23 sqrt(K / 16) sum_k |a_k| |w_k|
    (the model of the wgmma GEMM's tests, gemm_ref in test_gpu_kernel_edges.py)."""
    A64, W64 = A.double(), W.double()
    K = A.shape[1]
    return A64 @ W64.t(), 2 * U32 * math.sqrt(K / 16) * (A64.abs() @ W64.abs().t())


def bn_relu_ref(acc, slack, s, b):
    """kEpiBnRelu: relu(fl(fl(acc s) + b)) per output column.  Returns (ref, slack, pre): pre is the float64
    pre-activation, where pre <= -slack the kernel's output must be exactly +0."""
    s64, b64 = s.double(), b.double()
    t = acc * s64
    pre = t + b64
    sl = s64.abs() * slack + U32 * (t.abs() + pre.abs())
    return pre.clamp_min(0.0), sl, pre


def check_out(out, ref, slack, key, what, pre=None, where=None):
    """bf16 kernel output [M, N] against the float64 contract: |out - ref| <= 2^-8 |ref| + slack per element, and
    exactly +0 wherever the float64 pre-activation of a ReLU is at or below -slack."""
    assert_within(out, ref, slack, REL[0], key, what, where)
    if pre is not None:
        dead = pre <= -slack
        nz = dead & (_bits(out) != 0)
        assert not nz.any(), f"{what}: {int(nz.sum())} outputs with pre-activation <= -slack are not +0"


# ---- max pool and tail --------------------------------------------------------------------------------------------
def maxpool_ref(x):
    """3x3 / s2 / p1 max pool of [n, H, W, C] (NHWC, any float type), taps taken one by one; the window's centre is
    always inside the image, padding never wins."""
    n, H, W, C = x.shape
    xp = torch.full((n, H + 2, W + 2, C), float("-inf"), dtype=x.dtype, device=x.device)
    xp[:, 1:H + 1, 1:W + 1] = x
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out = None
    for ky in range(3):
        for kx in range(3):
            t = xp[:, ky:ky + 2 * Ho - 1:2, kx:kx + 2 * Wo - 1:2]
            out = t if out is None else torch.maximum(out, t)
    return out


def tail_ref(x, s, b):
    """bf16 [n, 49, C] -> fp32 [n, C]: s = fl(s + x_q) for q = 0..48 in order, fl(s / 49), fl(fl(mean scale) + shift)."""
    xf = x.float()
    acc = torch.zeros_like(xf[:, 0])
    for q in range(xf.shape[1]):
        acc = acc + xf[:, q]
    mean = acc / _full(acc, float(xf.shape[1]))
    return mean * s + b
