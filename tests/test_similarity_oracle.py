"""The similarity-head references (similarity_oracle.py) on the CPU: they agree with the CPU oracle and torch.topk, an
fp32 emulation of the tensor-core path stays inside them for every input family, and each of a list of small
mistakes in that emulation is rejected."""
import math

import pytest
import torch

from similarity_oracle import (FAMILIES, SUB16, assert_within, l2_ref, make_pair, similarity_refs, split_rows,
                               topk_check, f32)


def emulate_split(a, b, scale, norm_a, norm_b, ftz=False, rs_shift=0, ss_hi=False, drop_hilo=False):
    """fp32 emulation of split_embed_kernel + the EPI_SIM_F32 GEMM: the exact products of each k16 step added to an
    fp32 running sum with one rounding, fp32 row norms and rsqrt, (acc * rs) * cs in fp32.  The keywords plant the
    mistakes the contract must catch:
      ftz        fp16-subnormal lo parts flushed to zero (an ftz build)
      rs_shift   rows from rs_shift on take the row scale of the row rs_shift earlier (a stale scale vector in the
                 second A chunk)
      ss_hi      the norms taken from the hi parts only
      drop_hilo  the hi_a . lo_b term left out"""
    s = torch.tensor(f32(scale), dtype=torch.float32)

    def operand(x, norm, lo_first):
        p, f, hi, lo = split_rows(x)
        if ftz:
            lo = torch.where(lo.float().abs() < SUB16, torch.zeros_like(lo), lo)
        src = (hi.float() / p[:, None].float()) if ss_hi else x.float()
        ss = (src * src).sum(-1)
        undo = (1.0 / p).float()
        vs = undo * (torch.rsqrt(ss) if norm else torch.ones_like(ss))
        ops = [hi, lo, hi] if lo_first else [hi, hi, lo]
        return torch.cat(ops, 1).double(), vs

    A, rs = operand(a, norm_a, True)
    B, cs = operand(b, norm_b, False)
    rs = rs * s
    if drop_hilo:
        A[:, 1024:] = 0
    if rs_shift:
        rs = torch.cat([rs[:rs_shift], rs[:-rs_shift]])
    acc = torch.zeros(a.shape[0], b.shape[0], dtype=torch.float32)
    for k0 in range(0, A.shape[1], 16):
        acc = (acc.double() + A[:, k0:k0 + 16] @ B[:, k0:k0 + 16].t()).float()
    return (acc * rs[:, None]) * cs[None]


FLAGS = [(1, 1), (0, 0), (1, 0), (0, 1)]


def test_references_against_clip_oracle():
    from oracle import clip_oracle as O
    g = torch.Generator().manual_seed(3)
    a, b = torch.randn(6, 512, generator=g), torch.randn(9, 512, generator=g)
    r = similarity_refs(a, b, 14.3, 1, 1)
    want = O.similarity(O.l2_normalize(a.double()), O.l2_normalize(b.double()), f32(14.3))
    assert torch.allclose(r["plain"], want, rtol=1e-13, atol=1e-13)
    assert torch.allclose(r["contract"], want, rtol=0, atol=1e-5)      # the split: ~2^-22 relative
    x = torch.randn(5, 33, generator=g)
    ref, rel = l2_ref(x)
    assert torch.allclose(ref, O.l2_normalize(x.double()), rtol=1e-14, atol=0) and rel < 4e-7
    assert torch.isnan(l2_ref(torch.zeros(1, 8))[0]).all()
    # top-k: torch.topk of the reference is accepted with zero slack, named mistakes are not
    zero = torch.zeros_like(r["plain"])
    v, i = r["plain"].topk(4, dim=-1)
    topk_check(i.int(), v.float(), r["plain"], zero + 1e-6, 4, "torch.topk")
    bad_lists = {"order": (i.flip(-1), v.flip(-1)),
                 "repeat": (torch.cat([i[:, :1], i[:, :3]], 1), torch.cat([v[:, :1], v[:, :3]], 1)),
                 "range": (i.masked_fill(i == i[0, 0], 9), v),
                 "left out": (torch.cat([i[:, :3], r["plain"].topk(5, dim=-1).indices[:, 4:]], 1),
                              torch.cat([v[:, :3], r["plain"].topk(5, dim=-1).values[:, 4:]], 1)),
                 "pad": (torch.cat([i[:, :3], torch.full_like(i[:, :1], -1)], 1),
                         torch.cat([v[:, :3], torch.full_like(v[:, :1], float("-inf"))], 1))}
    for name, (bi, bv) in bad_lists.items():
        with pytest.raises(AssertionError):
            topk_check(bi.int(), bv.float(), r["plain"], zero + 1e-6, 4, name)
    # NaN scores (a zero row): never chosen, the list runs out into -1 / -inf
    ref = r["plain"].clone()
    ref[0] = float("nan")
    ref[1, 2:] = float("nan")
    i2, v2 = i.clone(), v.clone()
    i2[0], v2[0] = -1, float("-inf")
    v2[1, :2], i2[1, :2] = ref[1, :2].sort(descending=True)
    i2[1, 2:], v2[1, 2:] = -1, float("-inf")
    topk_check(i2.int(), v2.float(), ref, zero + 1e-6, 4, "NaN rows")
    with pytest.raises(AssertionError):
        topk_check(i.int(), v.float(), ref, zero + 1e-6, 4, "NaN chosen")


@pytest.mark.parametrize("family", FAMILIES)
def test_split_emulation_within_bounds(family):
    """The split residual stays within plain_ref's bound, and the fp32 emulation of the kernel within the contract
    and the plain bound, for every input family and normalisation pair."""
    a, b = make_pair(family, 24, 40, 11, "cpu")
    for na, nb in FLAGS:
        for scale in (1.0, 100.0):
            r = similarity_refs(a, b, scale, na, nb)
            what = f"{family} norm=({na},{nb}) scale={scale}"
            assert_within(r["contract"], r["plain"], r["resid"], 0.0, "cpu split residual / resid bound", what)
            out = emulate_split(a, b, scale, na, nb)
            assert_within(out, r["contract"], r["contract_slack"], 0.0, "cpu fp32 emulation / contract", what)
            assert_within(out, r["plain"], r["plain_slack"], 0.0, "cpu fp32 emulation / plain", what)


# mistake -> (family, emulate_split keywords); each must leave the contract
MUTATIONS = {
    "lo subnormals flushed": ("spike", dict(ftz=True)),
    "rs of the wrong row in the second A chunk": ("randn", dict(rs_shift=8)),
    "ss from the hi parts": ("parallel", dict(ss_hi=True)),
    "hi.lo term dropped": ("randn", dict(drop_hilo=True)),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS) + ["near-zero logit moved by 1e-4 max"])
def test_contract_rejects_mistakes(mutation):
    if mutation in MUTATIONS:
        family, kw = MUTATIONS[mutation]
        a, b = make_pair(family, 24, 40, 11, "cpu")
        out = emulate_split(a, b, 100.0, 1, 1, **kw)
    else:
        a, b = make_pair("orthogonal", 24, 40, 11, "cpu")
        out = emulate_split(a, b, 100.0, 1, 1)
        r = similarity_refs(a, b, 100.0, 1, 1)
        rr, cc = divmod(r["contract"].abs().argmin().item(), 40)
        assert abs(r["contract"][rr, cc].item()) < 1e-3 * r["contract"].abs().max().item()
        out[rr, cc] += 1e-4 * r["contract"].abs().max().item()
    r = similarity_refs(a, b, 100.0, 1, 1)
    with pytest.raises(AssertionError):
        assert_within(out, r["contract"], r["contract_slack"], 0.0, "mutation", mutation)


def test_l2_bound_rejects_a_dropped_lane():
    g = torch.Generator().manual_seed(4)
    for dim in (1, 31, 32, 33, 512, 768, 1024):
        x = torch.randn(40, dim, generator=g)
        ref, rel = l2_ref(x)
        ss = (x * x).sum(-1, keepdim=True)
        out = x * (1.0 / torch.sqrt(ss))
        assert_within(out, ref, 0.0, rel, "cpu l2 emulation / l2 bound", f"dim={dim}")
        if dim > 1:
            lane = x.clone()
            lane[:, 1::32] = 0                                     # lane 1's terms left out of the sum
            wrong = x * (1.0 / torch.sqrt((lane * lane).sum(-1, keepdim=True)))
            with pytest.raises(AssertionError):
                assert_within(wrong, ref, 0.0, rel, "l2 dropped lane", f"dim={dim}")
    assert math.isclose(l2_ref(torch.ones(1, 512))[1], (21 / 2 + 3) * 2.0 ** -24 * (1 + 2.0 ** -10))
