"""The long-sequence attention kernel (attention_long_kernel, 128 < S <= 1025) and the attention-probabilities kernel
(attention_probs_kernel, any S <= 1025) held to float64 contracts element by element: the S edges of their 64-key
blocks and 128-query blocks, flat and peaked softmax, a row maximum that moves in every key block, guard rows behind
the output and the arguments they refuse.

Everything goes through the C ABI test hooks plip_dbg_attention / plip_dbg_attention_probs.  References
(attention_oracle) are float64 from the 16-bit inputs the kernels read.

Constants of the kernels the cases below are derived from (attention.cu; revisit the cases when one of them changes):
  long kernel    one CTA per (sequence, head, block of 128 queries), two warpgroups of 64 query rows each; keys in
                 blocks of 64, the last block zero-filled by TMA past S and masked to -inf; online softmax (running
                 row max m, l *= alpha and O *= alpha with alpha = 2^(m_old - m_new) per block)
  probs kernel   one CTA per (sequence, head, block of 64 queries); pass 1 runs the same online max / sum over 64-key
                 blocks, pass 2 writes exp2(s - m) / l
"""
import json
import os

import pytest
import torch

from attention_oracle import (ATT_ABS, DT, KEY_BLOCK, OBSERVED, REL, SENT, U32, _bits, _round_to, assert_within,
                              long_attention_contract_ref, long_chain_slack, probs_contract_ref, running_block_max)
from plip_b200._lib import check, last_error, lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    yield lib()
    path = os.environ.get("PLIP_EDGE_REPORT")
    if path and OBSERVED:
        with open(path, "w") as f:
            json.dump(OBSERVED, f, indent=1, sort_keys=True)


@pytest.fixture
def fmt_guard(L):
    """Lets a test switch the handle-free hooks to fp16 operands; bf16 is restored whatever happens."""
    def set_fmt(fmt):
        check(L.plip_dbg_set_operand_format(fmt), "set_operand_format")
    try:
        yield set_fmt
    finally:
        L.plip_dbg_set_operand_format(0)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _fmt_name(fmt):
    return "bf16" if fmt == 0 else "fp16"


GUARD_ROWS = 8


def run_long(L, qkv, n_seq, S, heads, fmt):
    """One launch of the long kernel into [n_seq S + 8, D] rows of SENT; the guard rows must keep their bits."""
    D = heads * 64
    out = torch.full((n_seq * S + GUARD_ROWS, D), SENT, device=qkv.device, dtype=DT[fmt])
    check(L.plip_dbg_attention(qkv.data_ptr(), n_seq, S, heads, 0, None, out.data_ptr(), _stream()), "attention")
    torch.cuda.synchronize()
    guard = _bits(out[n_seq * S:])
    changed = guard != _bits(torch.full_like(out[n_seq * S:], SENT))
    assert not changed.any(), f"long attention S={S} n_seq={n_seq}: guard row write at {changed.nonzero()[0].tolist()}"
    return out[:n_seq * S]


def run_probs(L, qkv, n_seq, S, heads, causal, mask):
    """plip_dbg_attention_probs into [n_seq, heads, S, S] with 37 rows of SENT on each side, which keep their bits."""
    G = 37 * S
    n = n_seq * heads * S * S
    buf = torch.full((n + 2 * G,), SENT, device=qkv.device, dtype=torch.float32)
    check(L.plip_dbg_attention_probs(qkv.data_ptr(), n_seq, S, heads, int(causal),
                                     mask.data_ptr() if mask is not None else None, buf[G:].data_ptr(), _stream()),
          "attention_probs")
    torch.cuda.synchronize()
    guard = _bits(torch.cat([buf[:G], buf[G + n:]]))
    assert torch.equal(guard, _bits(torch.full((2 * G,), SENT, device=qkv.device))), "a write left the probabilities"
    return buf[G:G + n].view(n_seq, heads, S, S)


def long_reference(qkv, n_seq, S, heads, fmt):
    """(contract, slack) of the long kernel, slack = ATT_ABS + flip + the rescale chain's, over chunks of
    sequences that keep each float64 [n, heads, S, S] temporary near 256 MB."""
    per = max(1, (1 << 25) // (heads * S * S))
    parts = []
    for s0 in range(0, n_seq, per):
        n = min(per, n_seq - s0)
        x = qkv[s0 * S:(s0 + n) * S]
        contract, _, flip = long_attention_contract_ref(x, n, S, heads, fmt)
        parts.append((contract, ATT_ABS + flip + long_chain_slack(x, n, S, heads)))
    return [torch.cat(t) for t in zip(*parts)]


def _where_long(S):
    def where(r, c):
        seq, row = divmod(r, S)
        return (f"sequence {seq} row {row}: query block {row // 128} warpgroup {(row % 128) // 64} "
                f"{'second' if row % 16 >= 8 else 'first'} row of its thread; head {c // 64} dim {c % 64}")
    return where


def check_long(L, qkv, n_seq, S, heads, fmt, key, what):
    out = run_long(L, qkv, n_seq, S, heads, fmt)
    contract, slack = long_reference(qkv, n_seq, S, heads, fmt)
    assert_within(out, contract, slack, REL[fmt], key, what, _where_long(S))
    return out


def _prefix_holes_mask(n_seq, S, g, dev):
    """Key padding mask [n_seq, S] int32: a visible prefix of 1..S keys with holes; key 0 always visible."""
    lens = torch.randint(1, S + 1, (n_seq,), generator=g, device=dev)
    lens[-1] = S
    mask = torch.arange(S, device=dev)[None] < lens[:, None]
    mask &= torch.rand(n_seq, S, generator=g, device=dev) > 0.3
    mask[:, 0] = True
    return mask.to(torch.int32).contiguous()


# ------------------------------------------------------------------------------------------------------------------
# Long kernel against its contract
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f16", [0, 1])
@pytest.mark.parametrize("S", [129, 145, 197, 257, 600, 1025])
@pytest.mark.parametrize("n_seq", [1, 3, 37])
def test_long_attention(L, fmt_guard, S, n_seq, f16):
    """Vision-sized sequences with N(0,1) q, k, v: per element against the contract, bitwise reproducible (key
    blocks in a fixed order), and independent of the neighbouring sequences."""
    heads, D = 12, 768
    dt = DT[f16]
    fmt_guard(f16)
    g = torch.Generator().manual_seed(S * 7 + n_seq)
    qkv = torch.randn(n_seq * S, 3 * D, generator=g).to(dt).cuda()
    out = check_long(L, qkv, n_seq, S, heads, f16, f"long attention vs contract ({_fmt_name(f16)})",
                     f"long attention n_seq={n_seq} S={S} fmt={f16}")
    assert torch.equal(run_long(L, qkv, n_seq, S, heads, f16), out)        # fixed key-block order: reproducible
    if n_seq > 1:
        # every other sequence overwritten with +-3e4: the 3-D tensor maps never read (or write) across sequences
        j = n_seq // 2
        big = qkv.clone().view(n_seq, S, 3 * D)
        keep = big[j].clone()
        big.copy_(torch.where(torch.rand(big.shape, device="cuda") < 0.5, -3e4, 3e4).to(dt))
        big[j] = keep
        out2 = run_long(L, big.view(n_seq * S, 3 * D), n_seq, S, heads, f16).view(n_seq, S, D)
        assert torch.equal(out2[j], out.view(n_seq, S, D)[j])


# S mod 64 in {1, 63, 0}: a last key block of one key, of 63 keys, or full (no masked key at all).  S mod 128 in
# [1, 64] (129, 191, 192, 257, 319, 320, 575, 576, 1025): the last query block's second warpgroup has no row to store.
# An image of gh x gw patches (gh, gw <= 32) gives S = 1 + gh gw: 129, 191, 193, 256, 257, 320, 576 and 1025 occur
# in vision encodes; 192, 255, 319, 575, 1023 and 1024 only through the hook.  (n_seq, heads) cycle through
# {1, 2, 5} x {1, 12, 16}.
LONG_S = [129, 191, 192, 193, 255, 256, 257, 319, 320, 575, 576, 1023, 1024, 1025]
SHAPES = [(n, h) for n in (1, 2, 5) for h in (1, 12, 16)]
LONG_CASES = [(S, *SHAPES[(2 * i + fmt) % len(SHAPES)], fmt) for i, S in enumerate(LONG_S) for fmt in (0, 1)]


@pytest.mark.parametrize("S,n_seq,heads,fmt", LONG_CASES)
def test_long_contract_edges(L, fmt_guard, S, n_seq, heads, fmt):
    fmt_guard(fmt)
    dev = "cuda"
    g = _gen(dev, S * 131 + n_seq * 7 + heads + fmt)
    qkv = torch.randn(n_seq * S, 3 * heads * 64, generator=g, device=dev).to(DT[fmt])
    check_long(L, qkv, n_seq, S, heads, fmt, f"long attention vs contract ({_fmt_name(fmt)})",
               f"long attention edges n_seq={n_seq} S={S} heads={heads} fmt={fmt}")


# ------------------------------------------------------------------------------------------------------------------
# Flat softmax: q = 0, every score is 0
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("S", [129, 191, 192, 193, 1024, 1025])
def test_long_flat_softmax(L, fmt_guard, S, fmt):
    """Every key weighs 1 / S: the output is the mean of the sequence's V rows.  A padded key of the last block that
    escaped the mask would score 0 like the real ones and scale the output by S / (S + padding)."""
    fmt_guard(fmt)
    dev, n_seq, heads = "cuda", 3, 4
    D = heads * 64
    qkv = torch.randn(n_seq * S, 3 * D, generator=_gen(dev, S + fmt), device=dev).to(DT[fmt])
    qkv[:, :D] = 0
    out = run_long(L, qkv, n_seq, S, heads, fmt)
    v = qkv[:, 2 * D:].double().view(n_seq, S, D)
    mean_v = v.mean(1, keepdim=True).expand(n_seq, S, D).reshape(n_seq * S, D)
    # P = 1 exactly and alpha = 1 exactly: O is an fp32 sum of S products, one rounding per k16 step of the tensor
    # core (<= 2^-23 of sum |v| each), then O * (1 / l) with l = S exact
    slack = U32 * (S / 16 + 4) * v.abs().mean(1, keepdim=True).expand(n_seq, S, D).reshape(n_seq * S, D)
    assert_within(out, mean_v, slack, REL[fmt], "long attention flat softmax (mean of V)",
                  f"long flat S={S} fmt={fmt}", _where_long(S))


@pytest.mark.parametrize("kind", ["none", "key_mask", "causal", "causal_key_mask"])
@pytest.mark.parametrize("S", [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 1024, 1025])
def test_probs_flat_softmax(L, S, kind):
    """Every visible entry is float32(1 / count) bit for bit: the scores are 0, ex2(0) = 1, l counts the visible keys
    exactly in fp32 and 1.0f / l is an IEEE division (no fast math).  Masked entries are +0; keys past S may not
    count, and nothing is written outside [n_seq, heads, S, S]."""
    dev, n_seq, heads = "cuda", 3, 2
    D = heads * 64
    g = _gen(dev, 5 * S + len(kind))
    qkv = torch.randn(n_seq * S, 3 * D, generator=g, device=dev).to(torch.bfloat16)
    qkv[:, :D] = 0
    causal = kind.startswith("causal")
    mask = _prefix_holes_mask(n_seq, S, g, dev) if kind.endswith("key_mask") else None
    got = run_probs(L, qkv, n_seq, S, heads, causal, mask).cpu()
    vis = torch.ones(n_seq, 1, S, S, dtype=torch.bool)
    if causal:
        vis &= torch.ones(S, S, dtype=torch.bool).tril()
    if mask is not None:
        vis &= (mask.cpu() != 0)[:, None, None, :]
    count = vis.sum(-1, keepdim=True).to(torch.float32)
    want = torch.where(vis, torch.ones(()) / count, torch.zeros(())).expand(n_seq, heads, S, S).contiguous()
    bad = _bits(got) != _bits(want)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"probs flat S={S} {kind}: {int(bad.sum())} entries differ; first at (seq, head, row, "
                             f"key) {i}: got {got[tuple(i)].item()!r} want {want[tuple(i)].item()!r} "
                             f"(count {int(count[i[0], 0, i[2], 0])})")


# ------------------------------------------------------------------------------------------------------------------
# Peaked softmax: one key dominates every row
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("S", [129, 191, 576, 1025])
def test_long_peaked_softmax(L, fmt_guard, S, fmt):
    """Unit-norm keys, q = 80 k_target: the target scores 80 and every other key far less, so the output is v_target.
    Targets sit in block 0 (the maximum is found first and never moves), in the last key block (it moves last, by
    ~50) and at key S - 1."""
    fmt_guard(fmt)
    dev, n_seq, heads = "cuda", 2, 4
    D = heads * 64
    g = _gen(dev, 3 * S + fmt)
    k = torch.randn((n_seq, S, heads, 64), generator=g, device=dev).double()
    k = _round_to(k / k.norm(dim=-1, keepdim=True), DT[fmt])
    last0 = (S - 1) // KEY_BLOCK * KEY_BLOCK
    first = torch.randint(0, min(KEY_BLOCK, S), (n_seq, S), generator=g, device=dev)
    last = torch.randint(last0, S, (n_seq, S), generator=g, device=dev)
    row = torch.arange(S, device=dev)[None].expand(n_seq, S)
    tgt = torch.where(row % 3 == 0, first, torch.where(row % 3 == 1, last, torch.full_like(row, S - 1)))
    q = 80.0 * torch.gather(k, 1, tgt[:, :, None, None].expand(n_seq, S, heads, 64))
    vv = torch.randn((n_seq, S, heads, 64), generator=g, device=dev)
    qkv = torch.stack([q.float(), k.float(), vv], 2).reshape(n_seq * S, 3 * D).to(DT[fmt])
    out = check_long(L, qkv, n_seq, S, heads, fmt, "long attention peaked softmax vs contract",
                     f"long peaked S={S} fmt={fmt}")
    qs = qkv[:, :D].double().view(n_seq, S, heads, 64)
    ks = qkv[:, D:2 * D].double().view(n_seq, S, heads, 64)
    sc = torch.einsum("nihd,njhd->nhij", qs, ks)
    t_score = sc.gather(-1, tgt[:, None, :, None].expand(n_seq, heads, S, 1))[..., 0]
    assert (sc.amax(-1) - t_score).abs().max().item() < 1e-9                  # the target is each row's maximum
    second = sc.masked_fill(torch.nn.functional.one_hot(tgt, S).bool()[:, None], float("-inf")).amax(-1)
    gap = t_score - second
    v =qkv[:, 2 * D:].double().view(n_seq, S, heads, 64)
    v_t = torch.gather(v, 1, tgt[:, :, None, None].expand(n_seq, S, heads, 64))
    leak = (S * torch.exp(-gap) * v.abs().amax()).permute(0, 2, 1)[..., None].expand(n_seq, S, heads, 64)
    assert_within(out, v_t.reshape(n_seq * S, D), (1e-6 + leak).reshape(n_seq * S, D), REL[fmt],
                  "long attention peaked softmax vs v_target", f"long peaked closed form S={S} fmt={fmt}", _where_long(S))


# ------------------------------------------------------------------------------------------------------------------
# A row maximum that moves in every key block (rising) or never after block 0 (falling)
# ------------------------------------------------------------------------------------------------------------------
def _moving_max_qkv(n_seq, S, heads, rising, fmt, g, dev):
    """Scores s_ij = gamma_i (1 + 2 j' / 64) + small noise, j' = j (rising) or S - 1 - j (falling), gamma_i in
    [0.75, 1.25]: the row maximum climbs by 2 gamma per 64-key block (every rescale factor ~ e^-2 gamma) or is found
    in block 0 (every factor 1)."""
    u = torch.randn(heads, 64, generator=g, device=dev)
    u = u / u.norm(dim=-1, keepdim=True)

    def ortho(x):                                             # the part of x orthogonal to u
        return x - (x * u).sum(-1, keepdim=True) * u
    j = torch.arange(S, device=dev, dtype=torch.float32)
    ramp = 2.0 * (j if rising else S - 1 - j) / KEY_BLOCK
    k = (1.0 + ramp)[None, :, None, None] * u + ortho(torch.randn(n_seq, S, heads, 64, generator=g, device=dev) / 8)
    gamma = 0.75 + 0.5 * torch.rand(n_seq, S, heads, 1, generator=g, device=dev)
    q = gamma * u + ortho(torch.randn(n_seq, S, heads, 64, generator=g, device=dev) / 16)
    v = torch.randn(n_seq, S, heads, 64, generator=g, device=dev)
    return torch.stack([q, k, v], 2).reshape(n_seq * S, 3 * heads * 64).to(DT[fmt])


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("S", [257, 1025])
@pytest.mark.parametrize("direction", ["rising", "falling"])
@pytest.mark.parametrize("kernel", ["long", "probs"])
def test_moving_maximum(L, fmt_guard, kernel, direction, S, fmt):
    """The online softmax's rescale, row by row: l *= alpha in both kernels, O *= alpha (each row pair of a thread
    with its own alpha) in the long one."""
    fmt_guard(fmt)
    dev, n_seq, heads = "cuda", 2, 3
    g = _gen(dev, S + 2 * fmt + (direction == "rising"))
    qkv = _moving_max_qkv(n_seq, S, heads, direction == "rising", fmt, g, dev)
    q, k = (qkv.double().view(n_seq, S, 3, heads, 64)[:, :, i].transpose(1, 2) for i in (0, 1))
    m_key, _, _ = running_block_max(q @ k.transpose(-1, -2))
    m_blocks = m_key[..., ::KEY_BLOCK]                        # [n_seq, heads, S, n_kb]
    full = S // KEY_BLOCK
    if direction == "rising":                                 # the precondition: every full block raises the maximum
        assert (m_blocks[..., 1:full] - m_blocks[..., :full - 1]).min().item() > 1.0
    else:                                                     # ... or none after block 0 does
        assert torch.equal(m_blocks, m_blocks[..., :1].expand_as(m_blocks))
    what = f"{kernel} moving maximum ({direction}) S={S} fmt={fmt}"
    if kernel == "long":
        check_long(L, qkv, n_seq, S, heads, fmt, "long attention moving maximum vs contract", what)
        return
    got = run_probs(L, qkv, n_seq, S, heads, False, None)
    probs, rel = probs_contract_ref(qkv, n_seq, S, heads, False, None)
    assert_within(got.reshape(-1, S), probs.reshape(-1, S), 1e-30, rel.reshape(-1, S),
                  "attention probabilities moving maximum vs contract", what,
                  lambda r, c: f"sequence {r // (heads * S)} head {(r // S) % heads} row {r % S} key {c}")


# ------------------------------------------------------------------------------------------------------------------
# Arguments the kernels refuse: an error naming the reason, and no launch
# ------------------------------------------------------------------------------------------------------------------
def test_rejections_launch_nothing(L):
    dev, n_seq = "cuda", 2
    qkv = torch.zeros(n_seq * 1026, 3 * 17 * 64, device=dev, dtype=torch.bfloat16)
    out = torch.full((n_seq * 1026 + GUARD_ROWS, 17 * 64), SENT, device=dev, dtype=torch.bfloat16)
    probs = torch.full((n_seq * 17 * 1026 * 1026,), SENT, device=dev)
    mask = torch.ones(n_seq, 1026, device=dev, dtype=torch.int32)

    def long_call(S, heads, causal=0, km=None):
        return L.plip_dbg_attention(qkv.data_ptr(), n_seq, S, heads, causal, km, out.data_ptr(), _stream())

    def probs_call(S, heads):
        return L.plip_dbg_attention_probs(qkv.data_ptr(), n_seq, S, heads, 0, None, probs.data_ptr(), _stream())

    launches = int(L.plip_launch_count())
    for call, fragment in ((lambda: long_call(200, 12, causal=1), "attention: seq_len 200 > 128 is supported without causal or key mask"),
                           (lambda: long_call(129, 12, km=mask.data_ptr()), "attention: seq_len 129 > 128 is supported without causal or key mask"),
                           (lambda: long_call(1026, 12), "attention: bad shape n_seq=2 seq_len=1026"),
                           (lambda: long_call(200, 17), "attention: bad head count 17"),
                           (lambda: probs_call(1026, 12), "attention_probs: bad shape n_seq=2 seq_len=1026"),
                           (lambda: probs_call(200, 17), "attention_probs: bad head count 17")):
        assert call() != 0, fragment
        assert fragment in last_error(), (fragment, last_error())
    torch.cuda.synchronize()
    assert int(L.plip_launch_count()) == launches
    for t in (out, probs):
        assert torch.equal(_bits(t), _bits(torch.full_like(t, SENT))), "a refused call wrote its output"
