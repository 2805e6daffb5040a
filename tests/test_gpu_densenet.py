"""MuDiPath DenseNet-121 on the GPU: every kernel against its float64 contract (densenet_contract.py), the whole
network against the fp32 oracle (bound from the bf16 emulation) and the torchvision golden outputs, and the
``mudipath`` branch of ``EmbedderFactory``."""
import os
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import densenet_contract as C
import densenet_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "densenet_golden.npz")


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from plip_b200._lib import lib
    return lib()


@pytest.fixture(scope="module")
def sd():
    return O.make_state_dict(0)


@pytest.fixture(scope="module")
def engine(sd, L):
    from plip_b200.densenet import DenseNetEngine
    return DenseNetEngine(sd, device="cuda:0", max_micro_batch=4)


@pytest.fixture
def no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _op(L, op, x, lda, n, side, c_in, w, a_s, a_b, e_s, e_b, out, ldo):
    from plip_b200._lib import check
    p = lambda t: 0 if t is None else t.data_ptr()  # noqa: E731
    check(L.plip_dbg_densenet_op(op, p(x), lda, n, side, c_in, p(w), p(a_s), p(a_b), p(e_s), p(e_b), p(out), ldo,
                                 torch.cuda.current_stream().cuda_stream), f"plip_dbg_densenet_op({op})")
    torch.cuda.synchronize()


def _bn(c, g):
    s = (0.5 + torch.rand(c, generator=g)).cuda()
    b = (0.5 * torch.randn(c, generator=g)).cuda()
    return s, b


def _bf_rand(shape, g, scale=1.0):
    return (scale * torch.randn(shape, generator=g)).to(torch.bfloat16).cuda()


def test_stem_with_padded_corners(L):
    g = torch.Generator().manual_seed(1)
    n = 2
    tiles = torch.randint(0, 256, (n, 224, 224, 3), generator=g, dtype=torch.uint8)
    tiles[:, :8, :8] = 255          # extreme values at the padded corners
    tiles[:, -8:, -8:] = 0
    w4 = (0.1 * torch.randn(64, 3, 7, 7, generator=g)).to(torch.bfloat16)
    wk = torch.zeros(64, 160, dtype=torch.bfloat16)
    wk[:, :147] = C.conv_weight_k(w4)
    s, b = _bn(64, g)
    out = torch.empty(n * 112 * 112, 64, dtype=torch.bfloat16, device="cuda")
    _op(L, 0, tiles.cuda(), 0, n, 112, 3, wk.cuda(), None, None, s, b, out, 64)
    acc, slack = C.acc_ref(C.stem_a(tiles.cuda()), wk.cuda())
    ref, sl, pre = C.bn_relu_ref(acc, slack, s, b)
    C.check_out(out, ref, sl, "densenet stem (kAStem, kEpiBnRelu)", "stem, padded corners", pre)
    # the contract's operand is the emulation's normalised input, and its accumulator F.conv2d's
    y = F.conv2d(O.normalize_u8(tiles).to(torch.bfloat16).double().cuda(), w4.double().cuda(), stride=2, padding=3)
    assert torch.allclose(acc, y.permute(0, 2, 3, 1).reshape(-1, 64), rtol=0, atol=1e-12)


def test_maxpool_exact(L):
    g = torch.Generator().manual_seed(2)
    n = 2
    x = torch.relu(_bf_rand((n, 112, 112, 64), g))
    out = torch.zeros(n * 56 * 56, 256, dtype=torch.bfloat16, device="cuda")
    _op(L, 1, x, 64, n, 112, 64, None, None, None, None, None, out, 256)
    ref = F.max_pool2d(x.permute(0, 3, 1, 2).float(), 3, 2, 1).permute(0, 2, 3, 1).reshape(-1, 64)
    assert torch.equal(out[:, :64].float(), ref)
    assert not out[:, 64:].any()


@pytest.mark.parametrize("c_in,side,lda", [(64, 56, 256), (224, 56, 256), (128, 28, 512), (480, 28, 512),
                                           (256, 14, 1024), (992, 14, 1024), (512, 7, 1024), (992, 7, 1024)])
def test_conv1_preactivation(L, c_in, side, lda):
    g = torch.Generator().manual_seed(c_in + side)
    n = 3
    x = _bf_rand((n, side, side, lda), g)
    w = _bf_rand((128, c_in), g, c_in ** -0.5)
    a_s, a_b = _bn(c_in, g)
    e_s, e_b = _bn(128, g)
    out = torch.empty(n * side * side, 128, dtype=torch.bfloat16, device="cuda")
    _op(L, 2, x, lda, n, side, c_in, w, a_s, a_b, e_s, e_b, out, 128)
    acc, slack = C.acc_ref(C.preact_a(x.view(-1, lda), c_in, a_s, a_b), w)
    ref, sl, pre = C.bn_relu_ref(acc, slack, e_s, e_b)
    C.check_out(out, ref, sl, "densenet conv1 (kAPreact, kEpiBnRelu)", f"conv1 c_in={c_in} side={side}", pre)


@pytest.mark.parametrize("side", [56, 28, 14, 7])
def test_conv2_3x3_borders(L, side):
    g = torch.Generator().manual_seed(side)
    n = 3
    x = torch.relu(_bf_rand((n, side, side, 128), g))
    w4 = _bf_rand((32, 128, 3, 3), g, 1152 ** -0.5)
    wk = C.conv_weight_k(w4).contiguous()
    ldo = 64
    out = torch.zeros(n * side * side, ldo, dtype=torch.bfloat16, device="cuda")
    _op(L, 3, x, 128, n, side, 128, wk, None, None, None, None, out, ldo)
    acc, slack = C.acc_ref(C.tap3_a(x), wk)
    C.check_out(out[:, :32], acc, slack, "densenet conv2 (kATap3, kEpiStore)", f"conv2 side={side}")
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w4.double(), padding=1).permute(0, 2, 3, 1).reshape(-1, 32)
    assert torch.allclose(acc, ref, rtol=0, atol=1e-12)
    assert not out[:, 32:].any()


@pytest.mark.parametrize("c_in,side", [(256, 28), (512, 14), (1024, 7)])
def test_transition_pool_first(L, c_in, side):
    g = torch.Generator().manual_seed(c_in)
    n = 3
    x = _bf_rand((n, 2 * side, 2 * side, c_in), g)
    w = _bf_rand((c_in // 2, c_in), g, c_in ** -0.5)
    a_s, a_b = _bn(c_in, g)
    out = torch.empty(n * side * side, c_in // 2, dtype=torch.bfloat16, device="cuda")
    _op(L, 4, x, c_in, n, side, c_in, w, a_s, a_b, None, None, out, c_in // 2)
    acc, slack = C.acc_ref(C.pool_a(x, c_in, a_s, a_b), w)
    C.check_out(out, acc, slack, "densenet transition (kAPool, kEpiStore)", f"transition c_in={c_in}")


def test_tail(L):
    g = torch.Generator().manual_seed(5)
    n = 3
    x = _bf_rand((n, 49, 1024), g)
    s, b = _bn(1024, g)
    out = torch.empty(n, 1024, dtype=torch.float32, device="cuda")
    _op(L, 5, x, 1024, n, 7, 1024, None, None, None, s, b, out, 1024)
    assert torch.equal(out.cpu(), C.tail_ref(x.cpu(), s.cpu(), b.cpu()))   # the kernel's fp32 order, bit for bit


def _network_tiles(n, seed=11):
    g = torch.Generator().manual_seed(seed)
    base = torch.randint(0, 256, (n, 28, 28, 3), generator=g, dtype=torch.uint8).float()
    # smooth, image-like tiles: upsampled noise plus fine noise
    t = F.interpolate(base.permute(0, 3, 1, 2), size=(224, 224), mode="bilinear", align_corners=False)
    t = t + 12 * torch.randn(t.shape, generator=g)
    return t.clamp(0, 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def test_network_against_oracle_and_emulation(engine, sd, no_tf32):
    n = 9                                  # more than the micro-batch of 4: three passes, the last one of 1
    tiles = _network_tiles(n)
    out = engine.encode_images(tiles.cuda())
    again = engine.encode_images(tiles.cuda())
    torch.cuda.synchronize()
    assert torch.equal(out, again)         # two runs bit-identical
    sdc = {k: v.cuda() for k, v in sd.items()}
    ref = O.forward_u8(sdc, tiles.cuda())
    emu = O.forward_u8(sdc, tiles.cuda(), emulate=True)
    bound = O.cosine_gap(emu, ref).max().item()
    gap = O.cosine_gap(out, ref)
    gap_emu = O.cosine_gap(out, emu)
    print(f"\n1-cos vs fp32: max {gap.max().item():.2e}; emulation vs fp32 {bound:.2e}; vs emulation "
          f"{gap_emu.max().item():.2e}")
    assert gap.max().item() <= 2 * bound + 1e-6
    assert gap_emu.max().item() <= bound + 1e-6
    for m in (1, 3):                       # a lone image and an odd batch give the same rows
        part = engine.encode_images(tiles[:m].cuda())
        assert torch.equal(part, out[:m])


def test_network_against_torchvision_golden(engine, sd, no_tf32):
    z = np.load(GOLDEN)
    assert str(z["weights_sha256"]) == O.checksum(sd)
    tiles = torch.from_numpy(z["tiles"])
    out = engine.encode_images(tiles.cuda()).cpu()
    emu = O.forward_u8({k: v.cuda() for k, v in sd.items()}, tiles.cuda(), emulate=True).cpu()
    ref = torch.from_numpy(z["outputs"])
    bound = O.cosine_gap(emu, ref).max().item()
    gap = O.cosine_gap(out, ref)
    assert gap.max().item() <= 2 * bound + 1e-6, (gap, bound)


def test_host_variant_and_empty(engine):
    tiles = _network_tiles(5, seed=3)
    dev = engine.encode_images(tiles.cuda()).cpu().numpy()
    host = engine.encode_images_host(tiles.numpy())
    assert np.array_equal(dev, host)
    assert engine.encode_images(tiles[:0].cuda()).shape == (0, 1024)


def test_factory_mudipath(sd, tmp_path, monkeypatch, L):
    import PIL.Image
    from plip_b200.embedders import DenseNetEmbedder, EmbedderFactory
    from plip_b200.preprocess import to_uint8_tiles_bilinear
    ckpt = tmp_path / "densenet121-mh-best-191205-141200.pth"
    raw = {"features." + k: v for k, v in sd.items() if not k.startswith("classifier.")}
    raw["heads.0.weight"] = torch.zeros(3, 1024)      # the multi-task heads the reference's cleaning drops
    torch.save(raw, ckpt)
    monkeypatch.setenv("PLIP_B200_MTDP", str(ckpt))
    emb = EmbedderFactory().factory(Namespace(model_name="mudipath", backbone="default"))
    assert isinstance(emb, DenseNetEmbedder)
    rng = np.random.default_rng(0)
    arrays = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in [(224, 224), (300, 260), (180, 410)]]
    paths = []
    for i, a in enumerate(arrays):
        p = tmp_path / f"img{i}.png"
        PIL.Image.fromarray(a).save(p)
        paths.append(str(p))
    pils = [PIL.Image.fromarray(a) for a in arrays]
    e_paths = emb.embed_images(paths, batch_size=2)
    e_pil = emb.embed_images(pils)
    assert e_paths.shape == (3, 1024) and e_paths.dtype == np.float32
    assert np.array_equal(e_paths, e_pil)
    direct = emb.model.encode_images(torch.from_numpy(to_uint8_tiles_bilinear(pils)).cuda()).cpu().numpy()
    assert np.array_equal(e_pil, direct)
    assert emb.embed_images(paths[:1]).shape == (1, 1024)
