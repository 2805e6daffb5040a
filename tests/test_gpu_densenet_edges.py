"""DenseNet-121 kernels (densenet.cu) at every layer shape of the network, held per element to the float64 contracts of
densenet_contract.py, with guard bands around every output and poison around every input; and the network's
invariance to where an image sits in a batch and to what earlier passes left in the workspace.

Everything per kernel goes through plip_dbg_densenet_op.  Constants of the kernels the cases are derived from
(revisit the cases when one of them changes):
  densenet.cu   kBM = 128 rows per CTA tile, kBK = 32 (K is a whole number of k-tiles); BN = 64 (stem), 128 (conv1,
                transition), 32 (conv2).  Rows m >= M load zero A and are not stored.
  row tiles     M = n side^2:  side 56: n = 1 -> 3136 = 24 x 128 + 64;   n = 2 -> 6272 = 49 x 128
                               side 28: n = 1 ->  784 =  6 x 128 + 16;   n = 8 -> 6272
                               side 14: n = 1 ->  196 =  1 x 128 + 68;   n = 32 -> 6272
                               side  7: n = 1 ->   49 (one partial tile); n = 3 -> 147 = 128 + 19;  n = 128 -> 6272
                the stem's M = 112^2 n = 98 x 128 n is always whole tiles.
  network       block inputs 64 / 128 / 256 / 512 channels, buffers 256 / 512 / 1024 / 1024, sides 56 / 28 / 14 / 7;
                conv2 writes its 32 channels at column c_in of the block buffer (ldo = C_block), the transition
                channels [0, C / 2) of the next block's buffer.

Poison.  Out-of-range reads must land inside allocations the test owns, so every input sits in a larger buffer whose
guard rows and pad channels hold values that cannot go unnoticed once read:
  - conv2 and the tail read raw bf16: their guard rows hold NaN.
  - conv1 and the transition pass what they read through relu(x s + b), and fmaxf(NaN, 0) is 0, so NaN would vanish:
    their pad channels and guard rows hold +-2^64 (alternating by channel, so one of each pair survives the ReLU
    whatever the sign of the scale).  Their BN vectors are allocated to lda, pad entries (1, 0).
  - the max pool's input is post-ReLU and __hmax2 returns the other operand of a NaN: its guard rows hold +inf.
Outputs are written into buffers with 8 rows past M (and, where the hook takes ldo > N, pad columns) that hold
SENT or live data; every one of those elements must keep its bits.
"""
import json
import os

import pytest
import torch
import torch.nn.functional as F

import densenet_contract as C
import densenet_oracle as O
from attention_oracle import OBSERVED, SENT, _bits, _note

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
GUARD = 8                       # sentinel rows past M of every output, poison rows on both sides of every input
POISON = 2.0 ** 64
BLOCK_IN = (64, 128, 256, 512)
BLOCK_C = (256, 512, 1024, 1024)
LAYERS = (6, 12, 24, 16)
SIDES = (56, 28, 14, 7)
RAGGED = {56: 1, 28: 1, 14: 1, 7: 3}
WHOLE = {56: 2, 28: 8, 14: 32, 7: 128}

CONV1 = [(BLOCK_IN[b] + 32 * j, SIDES[b], BLOCK_C[b], RAGGED[SIDES[b]]) for b in range(4) for j in range(LAYERS[b])]
CONV1 += [(BLOCK_IN[b] + 32 * j, SIDES[b], BLOCK_C[b], WHOLE[SIDES[b]]) for b in range(4) for j in (0, LAYERS[b] - 1)]


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from plip_b200._lib import lib
    yield lib()
    path = os.environ.get("PLIP_EDGE_REPORT")
    if path and OBSERVED:
        with open(path, "w") as f:
            json.dump(OBSERVED, f, indent=1, sort_keys=True)


def _op(L, op, x, lda, n, side, c_in, w, a_s, a_b, e_s, e_b, out, ldo):
    from plip_b200._lib import check
    p = lambda t: 0 if t is None else t.data_ptr()  # noqa: E731
    check(L.plip_dbg_densenet_op(op, p(x), lda, n, side, c_in, p(w), p(a_s), p(a_b), p(e_s), p(e_b), p(out), ldo,
                                 torch.cuda.current_stream().cuda_stream), f"plip_dbg_densenet_op({op})")
    torch.cuda.synchronize()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(shape, g, scale=1.0):
    return scale * torch.randn(shape, generator=g, device="cuda")


def _activations(shape, g):
    """bf16 activations of ordinary size with one element in 16 scaled up to a few hundred."""
    x = _randn(shape, g, 2.0)
    big = torch.rand(shape, generator=g, device="cuda") < 1 / 16
    return torch.where(big, 100 * x, x).clamp(-400, 400).to(BF)


def _hard_bn(c, g, pad_to=None):
    """Folded BN as real checkpoints have it: negative scales, scales near 1e-3 and near 30, shifts up to +-20.
    With pad_to, the vectors are allocated that long and hold (1, 0) past c."""
    kind = torch.randint(0, 4, (c,), generator=g, device="cuda")
    mag = 0.5 + torch.rand(c, generator=g, device="cuda")
    s = torch.where(kind == 0, -mag, torch.where(kind == 1, 1e-3 * mag, torch.where(kind == 2, 30 * mag, mag)))
    s = s * torch.where(torch.rand(c, generator=g, device="cuda") < 0.2, -1.0, 1.0)
    wide = torch.rand(c, generator=g, device="cuda") < 0.25
    b = torch.where(wide, 40 * torch.rand(c, generator=g, device="cuda") - 20, _randn(c, g, 0.5))
    if pad_to is None:
        return s, b
    sp, bp = torch.ones(pad_to, device="cuda"), torch.zeros(pad_to, device="cuda")
    sp[:c], bp[:c] = s, b
    return sp, bp


def _relu_poison(rows, lda):
    """[rows, lda] bf16 of +-2^64, the sign alternating by channel."""
    sign = torch.where(torch.arange(lda, device="cuda") % 2 == 0, 1.0, -1.0)
    return (POISON * sign).to(BF).expand(rows, lda).contiguous()


def _inside(data, fill):
    """data [rows, ...] placed between GUARD rows of `fill` (a tensor of one row's shape, or a scalar).  Returns the
    whole allocation and the view of the data in it."""
    whole = torch.empty((data.shape[0] + 2 * GUARD,) + tuple(data.shape[1:]), dtype=data.dtype, device=data.device)
    whole[:] = fill
    whole[GUARD:GUARD + data.shape[0]] = data
    return whole, whole[GUARD:GUARD + data.shape[0]]


def _guarded_out(M, ldo):
    """[M + GUARD, ldo] bf16 output buffer of SENT."""
    return torch.full((M + GUARD, ldo), SENT, dtype=BF, device="cuda")


def _kept(out, before, rows, cols, what):
    """Every element of `out` outside [rows, cols] has the bits it had in `before`."""
    mask = torch.ones(out.shape, dtype=torch.bool, device=out.device)
    mask[rows, cols] = False
    changed = mask & (_bits(out) != _bits(before))
    assert not changed.any(), f"{what}: {int(changed.sum())} elements outside the output changed, first at " \
                              f"{changed.nonzero()[0].tolist()}"


def _where_rows(side):
    return lambda r, c: f"image {r // (side * side)}, pixel {r % (side * side)}, channel {c}, row tile {r // 128}"


# ---- stem ---------------------------------------------------------------------------------------------------------
def _stem_tiles(g):
    """[random with extreme corners, all 0, all 255, one-pixel checkerboard of 0 and 255]."""
    t = torch.randint(0, 256, (4, 224, 224, 3), generator=g, device="cuda", dtype=torch.uint8)
    t[0, :8, :8] = 255
    t[0, -8:, -8:] = 0
    t[1] = 0
    t[2] = 255
    yy, xx = torch.meshgrid(torch.arange(224, device="cuda"), torch.arange(224, device="cuda"), indexing="ij")
    t[3] = (((yy + xx) % 2) * 255).to(torch.uint8)[..., None]
    return t


@pytest.mark.parametrize("n", [1, 4])
def test_stem_contract(L, n):
    g = _gen(100 + n)
    if n == 1:
        tiles = torch.randint(0, 256, (1, 224, 224, 3), generator=g, device="cuda", dtype=torch.uint8)
    else:
        tiles = _stem_tiles(g)
    _, tiles = _inside(tiles, 255)                      # whole images of 255 on both sides
    w = _randn((64, 160), g, 0.1)
    w[:, 147:] = 2.0 ** 20                              # A's K pad must be exactly 0 for these to drop out
    w = w.to(BF)
    e_s, e_b = _hard_bn(64, g)
    M, ldo = n * 112 * 112, 72
    out = _guarded_out(M, ldo)
    before = out.clone()
    _op(L, 0, tiles, 0, n, 112, 3, w, None, None, e_s, e_b, out, ldo)
    acc, slack = C.acc_ref(C.stem_a(tiles), w)
    ref, sl, pre = C.bn_relu_ref(acc, slack, e_s, e_b)
    C.check_out(out[:M, :64], ref, sl, "densenet stem (kAStem, kEpiBnRelu)", f"stem n={n}", pre, _where_rows(112))
    _kept(out, before, slice(0, M), slice(0, 64), f"stem n={n}")


# ---- max pool -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 64])
def test_maxpool_exact(L, n):
    g = _gen(200 + n)
    x = _randn((n * 112 * 112, 64), g, 10.0).abs()
    x = torch.where(torch.rand(x.shape, generator=g, device="cuda") < 0.1, torch.zeros_like(x), x).to(BF)
    _, x = _inside(x, float("inf"))
    M, ldo = n * 56 * 56, 256
    out = _guarded_out(M, ldo)
    before = out.clone()
    _op(L, 1, x, 64, n, 112, 64, None, None, None, None, None, out, ldo)
    ref = C.maxpool_ref(x.view(n, 112, 112, 64)).reshape(M, 64)
    bad = _bits(out[:M, :64]) != _bits(ref)
    assert not bad.any(), f"max pool n={n}: {int(bad.sum())} outputs differ, first at {bad.nonzero()[0].tolist()}"
    _kept(out, before, slice(0, M), slice(0, 64), f"max pool n={n}")


# ---- conv1: every (c_in, side, lda) of the network ----------------------------------------------------------------
@pytest.mark.parametrize("c_in,side,lda,n", CONV1)
def test_conv1_contract(L, c_in, side, lda, n):
    g = _gen(c_in * 1000 + side * 10 + n)
    M = n * side * side
    data = _relu_poison(M, lda).clone()
    data[:, :c_in] = _activations((M, c_in), g)
    _, x = _inside(data, _relu_poison(1, lda)[0])
    a_s, a_b = _hard_bn(c_in, g, pad_to=lda)
    e_s, e_b = _hard_bn(128, g)
    w = _randn((128, c_in), g, c_in ** -0.5).to(BF)
    ldo = 136
    out = _guarded_out(M, ldo)
    before = out.clone()
    _op(L, 2, x, lda, n, side, c_in, w, a_s, a_b, e_s, e_b, out, ldo)
    acc, slack = C.acc_ref(C.preact_a(x, c_in, a_s[:c_in], a_b[:c_in]), w)
    ref, sl, pre = C.bn_relu_ref(acc, slack, e_s, e_b)
    what = f"conv1 c_in={c_in} side={side} lda={lda} n={n}"
    C.check_out(out[:M, :128], ref, sl, "densenet conv1 (kAPreact, kEpiBnRelu)", what, pre, _where_rows(side))
    _kept(out, before, slice(0, M), slice(0, 128), what)


# ---- conv2: into the middle of a block buffer ---------------------------------------------------------------------
CONV2 = [(b, n) for b in range(4) for n in sorted({RAGGED[SIDES[b]], WHOLE[SIDES[b]], 1})]


@pytest.mark.parametrize("block,n", CONV2)
def test_conv2_contract_in_block_buffer(L, block, n):
    side, c_blk = SIDES[block], BLOCK_C[block]
    cin = BLOCK_IN[block] + 32 * (LAYERS[block] // 2)       # live channels on both sides of the slice
    g = _gen(300 + 10 * block + n)
    M = n * side * side
    neck = torch.relu(_activations((M, 128), g).float()).to(BF)
    _, neck = _inside(neck, float("nan"))
    w = _randn((32, 1152), g, 1152 ** -0.5).to(BF)
    blk = _activations((M + GUARD, c_blk), g)
    before = blk.clone()
    _op(L, 3, neck, 128, n, side, 128, w, None, None, None, None, blk[:, cin:], c_blk)
    acc, slack = C.acc_ref(C.tap3_a(neck.view(n, side, side, 128)), w)
    what = f"conv2 side={side} n={n} at channel {cin} of {c_blk}"
    C.check_out(blk[:M, cin:cin + 32], acc, slack, "densenet conv2 (kATap3, kEpiStore)", what, None, _where_rows(side))
    _kept(blk, before, slice(0, M), slice(cin, cin + 32), what)


# ---- transition: into channels [0, C / 2) of the next block buffer ------------------------------------------------
TRANSITION = [(b, n) for b in range(3) for n in sorted({1, RAGGED[SIDES[b + 1]], WHOLE[SIDES[b + 1]]})]


@pytest.mark.parametrize("block,n", TRANSITION)
def test_transition_contract(L, block, n):
    c_in, side, ldo = BLOCK_C[block], SIDES[block + 1], BLOCK_C[block + 1]
    lda = c_in + 16
    g = _gen(400 + 10 * block + n)
    rows = n * 4 * side * side
    data = _relu_poison(rows, lda).clone()
    data[:, :c_in] = _activations((rows, c_in), g)
    _, x = _inside(data, _relu_poison(1, lda)[0])
    a_s, a_b = _hard_bn(c_in, g, pad_to=lda)
    w = _randn((c_in // 2, c_in), g, c_in ** -0.5).to(BF)
    M = n * side * side
    out = _activations((M + GUARD, ldo), g)
    before = out.clone()
    _op(L, 4, x, lda, n, side, c_in, w, a_s, a_b, None, None, out, ldo)
    acc, slack = C.acc_ref(C.pool_a(x.view(n, 2 * side, 2 * side, lda), c_in, a_s[:c_in], a_b[:c_in]), w)
    what = f"transition c_in={c_in} side={side} n={n}"
    C.check_out(out[:M, :c_in // 2], acc, slack, "densenet transition (kAPool, kEpiStore)", what, None,
                _where_rows(side))
    _kept(out, before, slice(0, M), slice(0, c_in // 2), what)


@pytest.mark.parametrize("block", [0, 1, 2])
def test_accumulator_on_cancelling_sums(L, block):
    """The accumulator model measured alone: the transition's K halves carry the same A and opposite weights, so the
    exact sum is 0 and what the kernel stores is its fp32 accumulation error, rounded to bf16 at 2^-8 of itself."""
    c_in, side, ldo = BLOCK_C[block], SIDES[block + 1], BLOCK_C[block + 1]
    g = _gen(500 + block)
    n = WHOLE[side]
    rows, h = n * 4 * side * side, c_in // 2
    half = _activations((rows, h), g)
    x = torch.cat([half, half], 1)
    s, b = _hard_bn(h, g)
    s, b = torch.cat([s, s]), torch.cat([b, b])
    wh = _randn((h, h), g, c_in ** -0.5).to(BF)
    w = torch.cat([wh, -wh], 1)
    M = n * side * side
    out = torch.full((M, ldo), SENT, dtype=BF, device="cuda")
    _op(L, 4, x, c_in, n, side, c_in, w, s, b, None, None, out, ldo)
    acc, slack = C.acc_ref(C.pool_a(x.view(n, 2 * side, 2 * side, c_in), c_in, s, b), w)
    ratio = ((out[:, :h].double() - acc).abs() / slack).max().item()
    _note("densenet accumulator, cancelling sums (|acc| / 2 x 2^-23 sqrt(K/16) sum|a||w|, mma.sync)", ratio)
    assert ratio <= 1.0, f"transition c_in={c_in}: accumulation error {ratio:.3f} of the slack"


# ---- tail ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 300])
def test_tail_exact(L, n):
    g = _gen(600 + n)
    x = _activations((n, 49, 1024), g)
    _, x = _inside(x, float("nan"))
    s, b = _hard_bn(1024, g)
    out = torch.full((n + 2, 1024), SENT, dtype=torch.float32, device="cuda")
    _op(L, 5, x, 1024, n, 7, 1024, None, None, None, s, b, out, 1024)
    ref = C.tail_ref(x.cpu(), s.cpu(), b.cpu())
    bad = _bits(out[:n].cpu()) != _bits(ref)
    assert not bad.any(), f"tail n={n}: {int(bad.sum())} outputs differ, first at {bad.nonzero()[0].tolist()}"
    assert (out[n:] == SENT).all()


# ---- the network: position in the batch and the workspace's history ----------------------------------------------
@pytest.fixture(scope="module")
def sd():
    return O.make_state_dict(0)


def _tiles(n, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.randint(0, 256, (n, 28, 28, 3), generator=g, dtype=torch.uint8).float()
    t = F.interpolate(base.permute(0, 3, 1, 2), size=(224, 224), mode="bilinear", align_corners=False)
    t = t + 12 * torch.randn(t.shape, generator=g)
    return t.clamp(0, 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous().cuda()


def _extreme_tiles(n):
    g = _gen(700)
    t = torch.randint(0, 256, (n, 224, 224, 3), generator=g, device="cuda", dtype=torch.uint8)
    t[0] = 255
    yy, xx = torch.meshgrid(torch.arange(224, device="cuda"), torch.arange(224, device="cuda"), indexing="ij")
    t[1] = (((yy + xx) % 2) * 255).to(torch.uint8)[..., None]
    t[2] = ((((yy // 8) + (xx // 8)) % 2) * 255).to(torch.uint8)[..., None]
    return t


def test_network_position_and_workspace_invariance(L, sd):
    """n = 19 at a micro-batch of 8 (passes of 8, 8 and 3).  Every output element has a fixed K order whatever its
    row, so an image's embedding must not depend, bit for bit, on where it sits in the batch, on the batch it comes
    with, or on what earlier calls left in the workspace (block-buffer channels at or past c_in hold the previous
    pass's data until this pass writes them)."""
    from plip_b200.densenet import DenseNetEngine
    tiles = _tiles(19, seed=21)
    fresh = DenseNetEngine(sd, device="cuda:0", max_micro_batch=8)
    ref = fresh.encode_images(tiles).clone()
    for k in range(19):
        assert torch.equal(fresh.encode_images(tiles[k:k + 1]), ref[k:k + 1]), f"image {k} alone"
    perm = torch.randperm(19, generator=torch.Generator().manual_seed(5)).cuda()
    assert torch.equal(fresh.encode_images(tiles[perm]), ref[perm])
    fresh.close()
    dirty = DenseNetEngine(sd, device="cuda:0", max_micro_batch=8)
    dirty.encode_images(_extreme_tiles(8))
    assert torch.equal(dirty.encode_images(tiles), ref)
    dirty.encode_images(_extreme_tiles(8))
    assert torch.equal(dirty.encode_images(tiles[16:]), ref[16:])
    dirty.close()
