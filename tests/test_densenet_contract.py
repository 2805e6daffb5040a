"""The float64 DenseNet-121 contracts of densenet_contract.py, without a GPU: they restate torch.nn.functional and the
bf16 emulation of densenet_oracle, and they reject the small mistakes a kernel could make (a near-zero output moved,
a border tap or the last k-tile dropped, two BN scales swapped)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import attention_oracle as AO
import densenet_contract as C
import densenet_oracle as O

BF = torch.bfloat16


@pytest.fixture(autouse=True)
def _keep_report():
    """The passing controls below go through assert_within, which records err / tol; keep those out of the report the
    GPU suites write."""
    saved = dict(AO.OBSERVED)
    yield
    AO.OBSERVED.clear()
    AO.OBSERVED.update(saved)


def _bf(shape, g, scale=1.0):
    return (scale * torch.randn(shape, generator=g)).to(BF)


def _store(ref):
    """What a kernel that meets the contract exactly writes: the float64 value rounded to fp32, then to bf16."""
    return ref.float().to(BF)


def test_stem_operand_matches_numpy_fp32_and_conv2d():
    g = torch.Generator().manual_seed(0)
    tiles = torch.randint(0, 256, (2, 20, 20, 3), generator=g, dtype=torch.uint8)
    a = C.stem_a(tiles)
    assert a.shape == (2 * 10 * 10, 160) and not a[:, 147:].float().any()
    # the normalised pixel, IEEE fp32 step by step, against numpy
    u = tiles.numpy().astype(np.float32)
    x = ((u / np.float32(255)) - np.array(C.MEAN, np.float32)) / np.array(C.STD, np.float32)
    x = torch.from_numpy(x).to(BF)
    assert torch.equal(O._bf(O.normalize_u8(tiles)).to(BF), x.permute(0, 3, 1, 2))   # the emulation's input rounding
    xp = torch.zeros(2, 26, 26, 3, dtype=BF)
    xp[:, 3:23, 3:23] = x
    assert torch.equal(a[11, :3], xp[0, 2, 2])          # output (1, 1): taps start at input (-1, -1) + 3
    assert not a[0, :21].float().any()                  # output (0, 0), ky = 0: the whole tap row is padding
    w4 = _bf((5, 3, 7, 7), g, 0.1)
    acc, slack = C.acc_ref(a, torch.cat([C.conv_weight_k(w4), torch.zeros(5, 13, dtype=BF)], 1))
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w4.double(), stride=2, padding=3).permute(0, 2, 3, 1).reshape(-1, 5)
    assert torch.allclose(acc, ref, rtol=0, atol=1e-12)
    assert (slack > 0).all()


def test_conv_operands_agree_with_functional():
    g = torch.Generator().manual_seed(1)
    n, side, c_in, lda = 2, 6, 64, 72
    x = _bf((n, side, side, lda), g, 3.0)
    s, b = torch.randn(c_in, generator=g), torch.randn(c_in, generator=g)
    # conv1: 1x1 over bf16(relu(x s + b))
    a = C.preact_a(x.view(-1, lda), c_in, s, b)
    assert torch.equal(a, O._bf(F.relu(x[..., :c_in].float() * s + b)).to(BF).view(-1, c_in))
    w = _bf((128, c_in), g, c_in ** -0.5)
    acc, _ = C.acc_ref(a, w)
    ref = F.conv2d(a.view(n, side, side, c_in).permute(0, 3, 1, 2).double(), w.double()[:, :, None, None])
    assert torch.allclose(acc, ref.permute(0, 2, 3, 1).reshape(-1, 128), rtol=0, atol=1e-12)
    # conv2: 3x3 / p1 over the bottleneck
    neck = torch.relu(_bf((n, side, side, 128), g))
    w4 = _bf((32, 128, 3, 3), g, 1152 ** -0.5)
    acc, _ = C.acc_ref(C.tap3_a(neck), C.conv_weight_k(w4))
    ref = F.conv2d(neck.permute(0, 3, 1, 2).double(), w4.double(), padding=1).permute(0, 2, 3, 1).reshape(-1, 32)
    assert torch.allclose(acc, ref, rtol=0, atol=1e-12)
    # transition: the fp32 pool-first operand is avg_pool2d of relu(bn(x)) up to fp32 rounding, and pooling before
    # the 1x1 conv equals pooling after it
    r = C.pool_r(x, c_in, s, b).double()
    xs = x[..., :c_in].double() * s.double()
    h = torch.relu(xs + b.double()).permute(0, 3, 1, 2)
    avg = F.avg_pool2d(h, 2).permute(0, 2, 3, 1)
    mag = F.avg_pool2d(xs.abs().permute(0, 3, 1, 2) + h, 2).permute(0, 2, 3, 1)   # x s and x s + b, rounded each
    assert ((r - avg).abs() <= AO.U32 * (mag + 3 * avg)).all()
    wt = _bf((c_in // 2, c_in), g, c_in ** -0.5).double()
    after = F.avg_pool2d(F.conv2d(h, wt[:, :, None, None]), 2).permute(0, 2, 3, 1).reshape(-1, c_in // 2)
    assert torch.allclose(avg.reshape(-1, c_in) @ wt.t(), after, rtol=0, atol=1e-12)
    assert torch.equal(C.pool_a(x, c_in, s, b), r.float().to(BF).reshape(-1, c_in))


def test_maxpool_and_tail_agree_with_functional():
    g = torch.Generator().manual_seed(2)
    x = _bf((2, 12, 10, 16), g)
    mp = C.maxpool_ref(x)
    ref = F.max_pool2d(x.permute(0, 3, 1, 2).float(), 3, 2, 1).permute(0, 2, 3, 1)
    assert mp.dtype == BF and torch.equal(mp.float(), ref)
    t = _bf((3, 49, 64), g, 50.0)
    s, b = 30 * torch.randn(64, generator=g), 20 * torch.randn(64, generator=g)
    out = C.tail_ref(t, s, b)
    assert out.dtype == torch.float32
    ref = F.adaptive_avg_pool2d(t.double().view(3, 7, 7, 64).permute(0, 3, 1, 2), 1).flatten(1) * s.double() + b.double()
    assert ((out.double() - ref).abs() <= 1e-5 * (t.double().abs().mean(1) * s.double().abs() + b.double().abs())).all()


def _contract_features(sd, tiles):
    """DenseNet-121 features + tail built only from the contracts, each conv's output stored as a kernel that meets
    its contract exactly would store it."""
    n, H = tiles.shape[0], tiles.shape[1]
    wk = lambda k: C.conv_weight_k(sd[k]).to(BF)  # noqa: E731
    w0 = torch.cat([wk("features.conv0.weight"), torch.zeros(64, 13, dtype=BF)], 1)
    acc, sl = C.acc_ref(C.stem_a(tiles), w0)
    x = _store(C.bn_relu_ref(acc, sl, *O.fold(sd, "features.norm0"))[0]).view(n, H // 2, H // 2, 64)
    x = C.maxpool_ref(x)
    side = H // 4
    for kind, pre, c in O.layer_names():
        if kind == "layer":
            acc, sl = C.acc_ref(C.preact_a(x.reshape(-1, c), c, *O.fold(sd, f"{pre}.norm1")), wk(f"{pre}.conv1.weight"))
            h = _store(C.bn_relu_ref(acc, sl, *O.fold(sd, f"{pre}.norm2"))[0]).view(n, side, side, 128)
            acc, _ = C.acc_ref(C.tap3_a(h), wk(f"{pre}.conv2.weight"))
            x = torch.cat([x, _store(acc).view(n, side, side, 32)], -1)
        else:
            side //= 2
            acc, _ = C.acc_ref(C.pool_a(x, c, *O.fold(sd, f"{pre}.norm")), wk(f"{pre}.conv.weight"))
            x = _store(acc).view(n, side, side, c // 2)
    return C.tail_ref(x.reshape(n, side * side, -1), *O.fold(sd, "features.norm5"))


def test_contracts_compose_to_the_bf16_emulation():
    """Chained through the whole network (64 x 64 tiles, so block 4 runs at 2 x 2), the contracts give the emulation's
    result up to its fp32 summation order.  A bf16 rounding that flips early is carried through 120 layers, so two
    bf16 evaluations that only sum in different orders end up a fraction of the bf16-vs-fp32 gap apart (0.2 of it
    here); a wrong layout, K order or pooling order would put them as far apart as unrelated features."""
    sd = O.make_state_dict(0)
    g = torch.Generator().manual_seed(3)
    tiles = torch.randint(0, 256, (2, 64, 64, 3), generator=g, dtype=torch.uint8)
    with torch.no_grad():
        got = _contract_features(sd, tiles)
        emu = O.forward_u8(sd, tiles, emulate=True)
        ref = O.forward_u8(sd, tiles)
    gap, bf16_gap = O.cosine_gap(got, emu).max().item(), O.cosine_gap(emu, ref).max().item()
    assert gap <= 0.5 * bf16_gap, (gap, bf16_gap)


# ---- teeth: each mistake must be rejected -------------------------------------------------------------------------
def _passes(out, ref, slack, pre=None):
    try:
        C.check_out(out, ref, slack, "teeth", "teeth", pre)
    except AssertionError:
        return False
    return True


def _hard_bn(c, g):
    s = (0.5 + torch.rand(c, generator=g)) * torch.where(torch.rand(c, generator=g) < 0.5, -1.0, 1.0)
    s[::4] = 30.0
    s[1::7] = 1e-3
    return s, 2 * torch.randn(c, generator=g)


def test_teeth_conv2_near_zero_output_moved():
    g = torch.Generator().manual_seed(4)
    neck = torch.relu(_bf((2, 7, 7, 128), g))
    w = C.conv_weight_k(_bf((32, 128, 3, 3), g, 1152 ** -0.5))
    acc, slack = C.acc_ref(C.tap3_a(neck), w)
    out = _store(acc)
    assert _passes(out, acc, slack)
    i = int(acc.abs().argmin())
    r, c = divmod(i, acc.shape[1])
    bad = out.clone()
    bad[r, c] = (acc[r, c] + 1e-4 * acc.abs().max()).float().to(BF)
    assert not _passes(bad, acc, slack)


def test_teeth_border_tap_dropped():
    g = torch.Generator().manual_seed(5)
    side = 7
    neck = torch.relu(_bf((1, side, side, 128), g))
    w = C.conv_weight_k(_bf((32, 128, 3, 3), g, 1152 ** -0.5))
    A = C.tap3_a(neck)
    acc, slack = C.acc_ref(A, w)
    assert _passes(_store(acc), acc, slack)
    row, tap = 3, 5                                      # output (0, 3), tap (ky, kx) = (1, 2): input (0, 4)
    k = slice(tap * 128, (tap + 1) * 128)
    assert A[row, k].float().any()
    dropped = acc.clone()
    dropped[row] -= A[row, k].double() @ w[:, k].double().t()
    assert not _passes(_store(dropped), acc, slack)


def test_teeth_conv1_last_k_tile_dropped():
    g = torch.Generator().manual_seed(6)
    c_in = 96
    x = _bf((64, 104), g, 3.0)
    a_s, a_b = _hard_bn(c_in, g)
    e_s, e_b = _hard_bn(128, g)
    A = C.preact_a(x, c_in, a_s, a_b)
    w = _bf((128, c_in), g, c_in ** -0.5)
    acc, slack = C.acc_ref(A, w)
    ref, sl, pre = C.bn_relu_ref(acc, slack, e_s, e_b)
    assert _passes(_store(ref), ref, sl, pre)
    short, _ = C.acc_ref(A[:, :c_in - 32], w[:, :c_in - 32])
    assert not _passes(_store(C.bn_relu_ref(short, slack, e_s, e_b)[0]), ref, sl, pre)


def test_teeth_bn_scale_of_neighbour_column():
    g = torch.Generator().manual_seed(7)
    c_in, col = 64, 6
    A = C.preact_a(_bf((64, c_in), g, 3.0), c_in, *_hard_bn(c_in, g))
    w = _bf((128, c_in), g, c_in ** -0.5)
    e_s, e_b = _hard_bn(128, g)
    e_s[col], e_s[col + 1] = 1.25, -0.75
    acc, slack = C.acc_ref(A, w)
    ref, sl, pre = C.bn_relu_ref(acc, slack, e_s, e_b)
    assert _passes(_store(ref), ref, sl, pre)
    swapped = e_s.clone()
    swapped[col], swapped[col + 1] = e_s[col + 1], e_s[col]
    assert not _passes(_store(C.bn_relu_ref(acc, slack, swapped, e_b)[0]), ref, sl, pre)
