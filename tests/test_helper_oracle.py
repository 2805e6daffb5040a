"""The helper-kernel references of helper_oracle.py against torch's own operators, and the planted mistakes they must
reject.  CPU only."""
import pytest
import torch
import torch.nn.functional as F

import helper_oracle as H
from oracle import clip_oracle as O


def _ln_rows(D, seed):
    """Rows of the kinds the GPU suite uses: N(0.5, 3), near-constant (variance below eps), mean 1e3 with std 1e-2,
    one channel at +-300 (make_state_dict(mode="outlier")), all equal."""
    g = torch.Generator().manual_seed(seed)
    rows = [torch.randn(8, D, generator=g) * 3 + 0.5,
            0.25 + 1e-4 * torch.randn(4, D, generator=g),
            1e3 + 1e-2 * torch.randn(4, D, generator=g),
            torch.randn(4, D, generator=g),
            torch.full((2, D), -7.125)]
    rows[3][0, 5], rows[3][1, D - 1], rows[3][2, 0], rows[3][3, 127] = 300.0, -300.0, 300.0, -300.0
    x = torch.cat(rows)
    gam = 1 + 0.1 * torch.randn(D, generator=g)
    bet = 0.1 * torch.randn(D, generator=g)
    return x, gam, bet


@pytest.mark.parametrize("D", [768, 512])
def test_layernorm_ref_matches_torch_and_bounds_emulation(D):
    x, g, b = _ln_rows(D, D)
    ref = H.layernorm_ref(x, g, b)
    # float64 against float64: the mean-1e3 rows cancel 5 digits, so 1e-9 is still 2^-53 x 1e5 x |y| with a margin
    d64 = (ref - F.layer_norm(x.double(), (D,), g.double(), b.double(), 1e-5)).abs().max().item()
    assert d64 < 1e-9, d64
    slack = H.layernorm_slack(x, g, b)
    err = (H.layernorm_emulate(x, g, b).double() - ref).abs()
    assert (err <= slack).all(), (err / slack).max().item()
    # torch's own fp32 LayerNorm on the ordinary rows (its sum order differs, its error is of the same size)
    e32 = (F.layer_norm(x[:8], (D,), g, b, 1e-5).double() - ref[:8]).abs()
    assert (e32 <= slack[:8]).all(), (e32 / slack[:8]).max().item()


@pytest.mark.parametrize("D", [768, 512])
@pytest.mark.parametrize("mistake,rows", [("one_pass", slice(12, 16)), ("eps_outside", slice(0, 8)),
                                          ("unbiased", slice(0, 8))])
def test_layernorm_ref_rejects_planted_mistakes(D, mistake, rows):
    x, g, b = _ln_rows(D, D + 1)
    if mistake == "eps_outside":
        x = x * 0.01                                    # std ~0.03: eps / sqrt(var) ~ 3e-4 relative
    x = x[rows]
    ref, slack = H.layernorm_ref(x, g, b), H.layernorm_slack(x, g, b)
    assert ((H.layernorm_emulate(x, g, b).double() - ref).abs() <= slack).all()
    bad = H.layernorm_emulate(x, g, b, **{mistake: True}).double()
    ratio = torch.nan_to_num((bad - ref).abs() / slack, nan=float("inf")).max().item()
    assert ratio > 2, (mistake, ratio)


@pytest.mark.parametrize("D", [768, 512])
def test_rowstats_ref_bounds_fp32_sums(D):
    x, _, _ = _ln_rows(D, 3)
    s1, s2, t1, t2 = H.rowstats_ref(x)
    assert torch.allclose(s1, x.double().sum(-1), rtol=1e-15, atol=0)
    e1 = (x.sum(-1).double() - s1).abs()
    e2 = ((x * x).sum(-1).double() - s2).abs()
    assert (e1 <= t1).all() and (e2 <= t2).all()


def test_u8_table_matches_clip_preprocessing():
    """The 768 values agree with CLIPImageProcessor's rescale + normalise (oracle/clip_oracle.preprocess_u8, divisions
    in fp32) to one fp32 ulp of the operands of the subtraction, scaled by 1/std: the two differ only in where they
    round (1/255 and 1/std as constants, the FFMA)."""
    t = H.u8_table().double()
    img = torch.arange(256, dtype=torch.uint8).view(1, 1, 256, 1).expand(1, 1, 256, 3).contiguous()
    pre = O.preprocess_u8(img)[0, :, 0, :].double()                       # [3, 256]
    byte = torch.arange(256, dtype=torch.float64)
    ulp = torch.stack([(byte / 255 + m) / s for m, s in zip(H.CLIP_MEAN, H.CLIP_STD)]) * 2.0 ** -23
    assert ((t - pre).abs() <= ulp).all(), ((t - pre).abs() / ulp).max().item()
    assert not torch.equal(H.u8_table(swap_means=True), H.u8_table())
    assert ((H.u8_table(swap_means=True).double() - pre).abs() > ulp).any()


@pytest.mark.parametrize("h,w", [(224, 224), (266, 250), (63, 95)])
def test_im2col_ref_is_the_stride_32_conv_gather(h, w):
    """im2col_ref . W^T equals nn.Conv2d(3, 768, 32, 32, bias=False) (unfold), and swapped ky / kx is rejected."""
    g = torch.Generator().manual_seed(h + w)
    px = torch.randn(2, 3, h, w, generator=g)
    cols = F.unfold(px, 32, stride=32)                                     # [n, 3072, L], column c * 1024 + ky * 32 + kx
    ref = cols.transpose(1, 2).reshape(-1, 3072)
    assert torch.equal(H.im2col_ref(px, 0, torch.float32), ref)
    assert not torch.equal(H.im2col_ref(px, 0, torch.float32, swap_k=True), ref)
    u8 = torch.randint(0, 256, (2, h, w, 3), generator=g, dtype=torch.uint8)
    vals = H.u8_table()
    pre = torch.stack([vals[c][u8[..., c].long()] for c in range(3)], 1)
    assert torch.equal(H.im2col_ref(u8, 2, torch.bfloat16), F.unfold(pre, 32, stride=32).transpose(1, 2)
                       .reshape(-1, 3072).to(torch.bfloat16))


def test_pooled_rows_ref_is_hf_semantics():
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, 49406, (64, 77), generator=g)
    ids[::2, 40] = H.EOS_ID
    ids[::4, 60] = H.EOS_ID
    ids[1::4, 3] = ids[1::4].max(1).values                                 # ties of the largest id
    for S in (77, 41, 1):
        got = H.pooled_rows_ref(ids, S, 0) - torch.arange(64) * S
        assert torch.equal(got, (ids[:, :S] == H.EOS_ID).int().argmax(-1))
        got1 = H.pooled_rows_ref(ids, S, 1) - torch.arange(64) * S
        has = (ids[:, :S] == H.EOS_ID).any(1)
        want = torch.where(has, (ids[:, :S] == H.EOS_ID).int().argmax(-1), ids[:, :S].argmax(-1))
        assert torch.equal(got1, want)
    assert not torch.equal(H.pooled_rows_ref(ids, 77, 0, last_eos=True), H.pooled_rows_ref(ids, 77, 0))
    assert not torch.equal(H.pooled_rows_ref(ids, 77, 1, later_tie=True), H.pooled_rows_ref(ids, 77, 1))


def test_mask_ref_is_to_bool():
    m = torch.tensor([[0, 1, 2, -1, 2 ** 33, 2 ** 32, 0]], dtype=torch.int64)
    assert torch.equal(H.mask_ref(m, 7), m.to(torch.bool).to(torch.int32).reshape(-1))
    assert not torch.equal(H.mask_ref(m, 7, truncate_i32=True), H.mask_ref(m, 7))


def test_text_embed_ref_clamps_ids():
    g = torch.Generator().manual_seed(2)
    tok, pos = torch.randn(H.VOCAB, 512, generator=g), torch.randn(77, 512, generator=g)
    ids = torch.tensor([[-1, 49408, 2 ** 40, 5]])
    x = H.text_embed_ref(ids, 4, tok, pos)
    assert torch.equal(x, torch.stack([tok[0] + pos[0], tok[-1] + pos[1], tok[-1] + pos[2], tok[5] + pos[3]]))


GRIDS = [(g, g) for g in range(1, 33)] + [(1, 32), (32, 1), (7, 8), (10, 15), (31, 17)]


@pytest.mark.parametrize("gh,gw", GRIDS)
def test_pos_interp_ref_matches_torch_bicubic(gh, gw):
    """The fp32-weight reference agrees with F.interpolate(bicubic, align_corners=False) in float64 within the gap of
    the two weight sets; the 7 x 7 table is the stored one; align_corners=True and taps clamped to [0, 7] are rejected."""
    g = torch.Generator().manual_seed(gh * 33 + gw)
    pos = torch.randn(50, 768, generator=g) * 0.02
    ref, slack = H.pos_interp_ref(pos, gh, gw)
    grid = pos[1:].double().reshape(1, 7, 7, 768).permute(0, 3, 1, 2)
    ti = F.interpolate(grid, size=(gh, gw), mode="bicubic", align_corners=False).permute(0, 2, 3, 1).reshape(-1, 768)
    ref64, _, gap = H.pos_interp_ref(pos, gh, gw, weights="fp64")
    assert torch.allclose(ref64[1:], ti, rtol=0, atol=1e-15)
    assert ((ref - ref64).abs() <= gap + 1e-15).all()
    assert torch.equal(ref[0], pos[0].double())
    if (gh, gw) == (7, 7):
        assert torch.equal(ref, pos.double())
    for plant in ({"align_corners": True}, {"clamp_hi": 7}):
        bad, _ = H.pos_interp_ref(pos, gh, gw, **plant)
        differs = ((bad - ref).abs() > slack + 1e-30).any()
        # align_corners gives the same coordinates on the 7 x 7 grid, and a tap clamped to 7 instead of 6 only matters
        # where its weight is nonzero
        if plant.get("align_corners") and (gh, gw) == (7, 7):
            continue
        if "clamp_hi" in plant and not any(
                a != b_ and w != 0 for g_ in (gh, gw) for i in range(g_)
                for a, b_, w in zip(H.cubic_taps32(g_, i)[0], H.cubic_taps32(g_, i, clamp_hi=7)[0],
                                    H.cubic_taps32(g_, i)[1])):
            continue
        assert differs, plant
