"""Images of any size (``interpolate_pos_encoding``) on the GPU: the interpolated position table, vision hidden states
and image features against the oracle and the live-transformers golden vectors, token-budget micro-batching,
last-layer pruning and ``PlipCLIPModel.forward``.  The long-sequence attention kernel itself is held to its float64
contract in test_gpu_attention_long.py."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import hires_oracle as HO
from oracle import clip_oracle as O
from oracle import synth
from plip_b200._lib import check, lib
from plip_b200.engine import Engine
from plip_b200.modeling import PlipCLIPModel
from plip_b200.synthetic import pixel_values_hw

pytestmark = pytest.mark.gpu
COS_TOL = 1e-4
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hires_golden.npz")


@pytest.fixture(scope="module")
def hires_golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


@pytest.fixture(scope="module")
def engine16(state_dict):
    eng = Engine(state_dict, max_micro_batch=64, operand_dtype="fp16")
    yield eng
    eng.close()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _cos_err(a, b):
    return (1 - O.cosine(a.cpu(), b.cpu())).max().item()


# ---- 1. position table -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("gh,gw", [(8, 8), (14, 14), (10, 15), (8, 7), (32, 32), (7, 7), (1, 3)])
def test_pos_interp_matches_torch_bicubic(state_dict, gh, gw):
    L = lib()
    pos = state_dict["vision_model.embeddings.position_embedding.weight"]
    ref = HO.interpolate_pos(pos, gh, gw)
    pd = pos.cuda().contiguous()
    out = torch.full((1 + gh * gw, 768), float("nan"), device="cuda")
    check(L.plip_dbg_pos_interp(pd.data_ptr(), gh, gw, out.data_ptr(), _stream()), "pos_interp")
    got = out.cpu()
    if (gh, gw) == (7, 7):
        assert torch.equal(got, pos)
    assert (got - ref).abs().max().item() <= 1e-6 * pos.abs().max().item()
    from helper_oracle import pos_interp_ref
    cref, slack = pos_interp_ref(pos, gh, gw)               # the kernel's fp32 weights, gamma(8) sum |w||p| per element
    assert ((got.double() - cref).abs() <= slack).all()


# ---- 2. vision hidden states -------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(448, 448), (320, 480), (266, 250), (256, 256)])
def test_vision_hidden_states_hires(engine, state_dict, hires_golden, h, w):
    px = pixel_values_hw(2, h, w)
    hid = []
    HO.vision_transformer(state_dict, px, hidden=hid, interpolate_pos_encoding=True)
    k = HO.size_key(h, w)
    for nl in (0, 1, 6, 12):
        got = engine.hidden_states("vision", px.cuda(), nl, interpolate_pos_encoding=True).cpu()
        assert got.shape == hid[nl].shape
        d = (got - hid[nl]).abs()
        assert d.max().item() < 0.05 and d.mean().item() < 6e-3, (nl, d.max().item(), d.mean().item())
        if nl in (0, 1, 12):
            gs = torch.cat([got[:1, :5], got[:1, -5:]], dim=1)
            dg = (gs - torch.from_numpy(hires_golden[f"vision_hidden_{nl}_{k}"])).abs()
            assert dg.max().item() < 0.05 and dg.mean().item() < 6e-3, (nl, dg.max().item())


# ---- 3. image features against the golden ---------------------------------------------------------------------
@pytest.mark.parametrize("h,w", HO.HIRES_SIZES)
def test_image_features_hires_vs_golden(engine, engine16, hires_golden, h, w):
    px = pixel_values_hw(2, h, w)
    ref = torch.from_numpy(hires_golden[f"image_features_{HO.size_key(h, w)}"])
    worst = {}
    for name, eng in (("bf16", engine), ("fp16", engine16)):
        out = eng.encode_images(px.cuda(), interpolate_pos_encoding=True)
        assert out.shape == (2, 512)
        worst[f"{name}/f32"] = _cos_err(out, ref)
        worst[f"{name}/bf16px"] = _cos_err(eng.encode_images(px.cuda().to(torch.bfloat16), interpolate_pos_encoding=True), ref)
        # uint8 tiles: the fused (x / 255 - mean) / std against the same engine on the fp32 preprocessed pixels
        u8 = torch.from_numpy(np.random.default_rng(h * w).integers(0, 256, (2, h, w, 3), dtype=np.uint8))
        o8 = eng.encode_images(u8.cuda(), interpolate_pos_encoding=True)
        worst[f"{name}/u8"] = _cos_err(o8, eng.encode_images(O.preprocess_u8(u8).cuda(), interpolate_pos_encoding=True))
    print(f"hires 1-cos {h}x{w}: " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))
    assert max(worst.values()) <= COS_TOL, worst


def test_u8_hires_vs_oracle(engine, state_dict):
    u8 = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (2, 266, 250, 3), dtype=np.uint8))
    ref = HO.get_image_features(state_dict, O.preprocess_u8(u8), interpolate_pos_encoding=True)
    assert _cos_err(engine.encode_images(u8.cuda(), interpolate_pos_encoding=True), ref) < COS_TOL


# ---- 4. a 7 x 7 grid is the 224 path -------------------------------------------------------------------------------
def test_7x7_grid_equals_224_bitwise(engine):
    px = pixel_values_hw(3, 240, 230)
    crop = px[:, :, :224, :224].contiguous().cuda()
    base = engine.encode_images(crop)
    assert torch.equal(engine.encode_images(crop, interpolate_pos_encoding=True), base)
    assert torch.equal(engine.encode_images(px.cuda(), interpolate_pos_encoding=True), base)
    u8 = torch.from_numpy(np.random.default_rng(9).integers(0, 256, (2, 240, 230, 3), dtype=np.uint8))
    assert torch.equal(engine.encode_images(u8.cuda(), interpolate_pos_encoding=True),
                       engine.encode_images(u8[:, :224, :224].contiguous().cuda()))


# ---- 5. micro-batching by tokens -----------------------------------------------------------------------------------
def test_token_budget_micro_batches(engine, state_dict):
    # max_micro_batch 64 -> 3200 token rows -> 16 images of 197 tokens per pass: 37 images take 3 passes
    px = pixel_values_hw(37, 448, 448, seed=11).cuda()
    whole = engine.encode_images(px, interpolate_pos_encoding=True)
    single = torch.cat([engine.encode_images(px[i:i + 1], interpolate_pos_encoding=True) for i in range(37)])
    assert torch.equal(whole, single)
    engine.profile(True)
    try:
        engine.encode_images(px[:2], interpolate_pos_encoding=True)
        names = {r["name"]: r["launches"] for r in engine.profile_read()}
    finally:
        engine.profile(False)
    assert names.get("vision/attention[long]") == 12 and "vision/attention" not in names
    small = Engine(state_dict, max_micro_batch=8)   # 400 token rows
    try:
        assert small.encode_images(px[:3], interpolate_pos_encoding=True).shape == (3, 512)
        with pytest.raises(RuntimeError, match=r"1025 tokens.*max_micro_batch >= 21"):
            small.encode_images(pixel_values_hw(1, 1024, 1024).cuda(), interpolate_pos_encoding=True)
    finally:
        small.close()


# ---- 6. last-layer pruning -------------------------------------------------------------------------------------------
def test_last_layer_pruning_hires(engine):
    px = pixel_values_hw(5, 448, 448, seed=5).cuda()
    assert not engine.last_layer_pruning
    full = engine.encode_images(px, interpolate_pos_encoding=True)
    engine.set_last_layer_pruning(True)
    try:
        pruned = engine.encode_images(px, interpolate_pos_encoding=True)
    finally:
        engine.set_last_layer_pruning(False)
    assert torch.equal(pruned, full)


# ---- 7. PlipCLIPModel.forward ------------------------------------------------------------------------------------------
def test_model_forward_hires_device_and_host(state_dict):
    model = PlipCLIPModel(state_dict, max_micro_batch=16)   # 800 token rows: 4 images of 197 tokens per pass
    try:
        px = pixel_values_hw(6, 448, 448, seed=8)
        ids, mask = synth.token_ids(3)
        dev = model(input_ids=ids.cuda(), pixel_values=px.cuda(), attention_mask=mask.cuda(), interpolate_pos_encoding=True)
        host = model(input_ids=ids, pixel_values=px, attention_mask=mask, interpolate_pos_encoding=True)
        assert torch.equal(dev.logits_per_image, host.logits_per_image)
        img = model.engine.encode_images(px.cuda(), normalize=True, interpolate_pos_encoding=True)
        txt = model.engine.encode_text(ids.cuda(), mask.cuda(), normalize=True)
        assert torch.equal(model.engine.similarity(img, txt, normalize_image=False, normalize_text=False),
                           dev.logits_per_image)
        feats = model.get_image_features(pixel_values=px.cuda(), interpolate_pos_encoding=True)
        assert _cos_err(feats, img) < 1e-10                   # get_image_features is the un-normalised tower output
        ref = HO.get_image_features(state_dict, px, interpolate_pos_encoding=True)
        ref_t = O.get_text_features(state_dict, ids, mask)
        lpi = O.similarity(O.l2_normalize(ref), O.l2_normalize(ref_t), float(state_dict["logit_scale"].exp()))
        dl = (dev.logits_per_image.cpu() - lpi).abs().max().item()
        print(f"hires forward |dlogits| {dl:.2e}")
        assert dl < 1e-2       # the end-to-end bound smoke() holds the 224 path to
        with pytest.raises(ValueError, match=r"doesn't match model \(224\*224\)"):
            model(input_ids=ids.cuda(), pixel_values=px.cuda())
    finally:
        model.engine.close()
