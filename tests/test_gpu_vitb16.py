"""CLIP ViT-B/16 on the GPU: the patch-16 im2col (tiles and windows) bit for bit, the 197-row position table against its
float64 reference, both towers' embeddings, hidden states and attentions against the fp32 oracle (pinned to transformers
by vitb16_golden.npz), micro-batching, the forward / pair / host / pruning paths against separate calls bit for bit,
determinism, an unchanged ViT-B/32 engine, and the ``ViT-B/16`` arm of ``EmbedderFactory``."""
import ctypes as C
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

import vitb16_oracle as V
from oracle import clip_oracle as O
from oracle import synth
from plip_b200._lib import check, lib
from plip_b200.engine import Engine
from plip_b200.modeling import PlipCLIPModel
from plip_b200.synthetic import make_state_dict, pixel_values_hw
from plip_b200.weights import pack_state_dict
from test_weights import _to_openai

pytestmark = pytest.mark.gpu
COS_TOL = 1e-4
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vitb16_golden.npz")
DT = {0: torch.bfloat16, 1: torch.float16}


@pytest.fixture(scope="module")
def sd16():
    torch.set_grad_enabled(False)
    return make_state_dict(0, "rich", patch=16)


@pytest.fixture(scope="module")
def golden16():
    return dict(np.load(GOLDEN, allow_pickle=False))


@pytest.fixture(scope="module")
def eng16(sd16):
    eng = Engine(sd16, max_micro_batch=64)          # 3200 token rows: 16 images of 197 tokens per pass
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def eng16h(sd16):
    eng = Engine(sd16, max_micro_batch=64, operand_dtype="fp16")
    yield eng
    eng.close()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _cos_err(a, b):
    return (1 - O.cosine(a.cpu(), b.cpu())).max().item()


def _u8(n, h, w, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8))


def test_engine_reports_its_patch(eng16, engine):
    assert eng16.vision_patch == 16 and engine.vision_patch == 32
    assert eng16.vision_seq_len() == 197 and eng16.vision_seq_len(512, 512) == 1025
    with pytest.raises(ValueError, match=r"at most 32 patches of 16 per side \(<= 527 px\)"):
        eng16.encode_images(pixel_values_hw(1, 528, 224).cuda(), interpolate_pos_encoding=True)


# ---- 1. im2col ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("pix", [0, 1, 2])
@pytest.mark.parametrize("h,w", [(224, 224), (266, 250)])
def test_im2col_patch16_bitexact(h, w, pix, fmt):
    L = lib()
    check(L.plip_dbg_set_operand_format(fmt), "operand format")
    try:
        n = 3
        g = torch.Generator(device="cuda").manual_seed(h + w + pix)
        if pix == 2:
            px = torch.randint(0, 256, (n, h, w, 3), generator=g, device="cuda", dtype=torch.uint8)
        else:
            px = (torch.randn(n, 3, h, w, generator=g, device="cuda") * 2).to(torch.float32 if pix == 0 else torch.bfloat16)
        P = (h // 16) * (w // 16)
        out = torch.full((n * P + 4, 768), float("nan"), device="cuda", dtype=DT[fmt])
        check(L.plip_dbg_im2col_patch(px.data_ptr(), pix, n, h, w, 16, out.data_ptr(), _stream()), "im2col_patch")
        torch.cuda.synchronize()
        ref = V.im2col_ref(px, pix, DT[fmt])
        assert torch.equal(out[:n * P].view(torch.int16), ref.view(torch.int16))
        assert out[n * P:].isnan().all()                                        # nothing past the patch rows
        if pix == 0:                                                            # torch's unfold restatement
            uf = torch.nn.functional.unfold(px[:, :, :h // 16 * 16, :w // 16 * 16], 16, stride=16)
            assert torch.equal(out[:n * P], uf.transpose(1, 2).reshape(n * P, 768).to(DT[fmt]))
        same32 = torch.empty(n * (h // 32) * (w // 32), 3072, device="cuda", dtype=DT[fmt])
        b32 = torch.empty_like(same32)
        check(L.plip_dbg_im2col_patch(px.data_ptr(), pix, n, h, w, 32, same32.data_ptr(), _stream()), "patch 32")
        check(L.plip_dbg_im2col_hw(px.data_ptr(), pix, n, h, w, b32.data_ptr(), _stream()), "im2col_hw")
        torch.cuda.synchronize()
        assert torch.equal(same32.view(torch.int16), b32.view(torch.int16))
    finally:
        check(L.plip_dbg_set_operand_format(0), "operand format")


def test_im2col_rejects_other_patch_sizes():
    L = lib()
    x = torch.zeros(1, 3, 224, 224, device="cuda")
    out = torch.zeros(196, 768, device="cuda", dtype=torch.bfloat16)
    assert L.plip_dbg_im2col_patch(x.data_ptr(), 0, 1, 224, 224, 14, out.data_ptr(), _stream()) != 0


# ---- 2. windows -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [0, 1])
def test_window_im2col_equals_tile_im2col(fmt):
    L = lib()
    check(L.plip_dbg_set_operand_format(fmt), "operand format")
    try:
        region = torch.from_numpy(np.random.default_rng(4).integers(0, 256, (600, 731, 3), dtype=np.uint8)).cuda()
        origins = torch.tensor([[0, 0], [1, 3], [376, 507], [201, 402], [17, 5]], dtype=torch.int32)
        crops = torch.stack([region[r:r + 224, c:c + 224] for r, c in origins.tolist()]).contiguous()
        n = origins.shape[0]
        a = torch.empty(n * 196, 768, device="cuda", dtype=DT[fmt])
        b = torch.empty_like(a)
        od = origins.cuda()
        check(L.plip_dbg_window_im2col_patch(region.data_ptr(), region.stride(0), od.data_ptr(), n, 16, a.data_ptr(),
                                             _stream()), "window_im2col_patch")
        check(L.plip_dbg_im2col_patch(crops.data_ptr(), 2, n, 224, 224, 16, b.data_ptr(), _stream()), "im2col_patch")
        torch.cuda.synchronize()
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    finally:
        check(L.plip_dbg_set_operand_format(0), "operand format")


def test_encode_region_equals_cut_out_crops(sd16):
    from plip_b200.plip import PLIP
    plip = PLIP.from_state_dict(sd16, max_micro_batch=32)           # 8 windows per pass
    try:
        img = np.random.default_rng(7).integers(0, 256, (900, 1100, 3), dtype=np.uint8)
        emb, origins, _ = plip.encode_region(torch.from_numpy(img).cuda())
        assert emb.shape == (len(origins), 512) and len(origins) > 8
        crops = torch.from_numpy(np.stack([img[r:r + 224, c:c + 224] for r, c in origins])).cuda()
        assert np.array_equal(emb, plip.model.engine.encode_images(crops).cpu().numpy())
    finally:
        plip.model.engine.close()


# ---- 3. position table ------------------------------------------------------------------------------------------------
def test_pos_interp_from_14x14(sd16):
    L = lib()
    pos = sd16["vision_model.embeddings.position_embedding.weight"].clone()
    pos[3, 5], pos[150, 700] = 3.0, -2.5
    pd = pos.cuda()
    for gh, gw in [(14, 14), (20, 28), (32, 32), (1, 1), (7, 9), (15, 14), (31, 17)]:
        rows = 1 + gh * gw
        out = torch.full((rows + 2, 768), float("nan"), device="cuda")
        check(L.plip_dbg_pos_interp_patch(pd.data_ptr(), 16, gh, gw, out.data_ptr(), _stream()), "pos_interp_patch")
        torch.cuda.synchronize()
        got = out.cpu()
        ref, slack = V.pos_interp_ref(pos, gh, gw)
        assert torch.equal(got[0], pos[0])
        if (gh, gw) == (14, 14):
            assert torch.equal(got[:rows], pos)
        assert ((got[1:rows].double() - ref[1:]).abs() <= slack[1:]).all(), (gh, gw)
        assert got[rows:].isnan().all()
    assert L.plip_dbg_pos_interp_patch(pd.data_ptr(), 8, 4, 4, out.data_ptr(), _stream()) != 0


def test_224_to_239_equal_224_bitwise(eng16):
    px = pixel_values_hw(2, 239, 239, seed=3)
    base = eng16.encode_images(px[:, :, :224, :224].contiguous().cuda())
    for s in (224, 231, 239):
        crop = px[:, :, :s, :s].contiguous().cuda()
        assert torch.equal(eng16.encode_images(crop, interpolate_pos_encoding=True), base), s
    u8 = _u8(2, 239, 230, 9)
    assert torch.equal(eng16.encode_images(u8.cuda(), interpolate_pos_encoding=True),
                       eng16.encode_images(u8[:, :224, :224].contiguous().cuda()))


# ---- 4. towers against the oracle ------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", V.SIZES)
def test_image_features_vs_oracle(eng16, eng16h, sd16, golden16, h, w):
    ipe = (h, w) != (224, 224)
    px = pixel_values_hw(2, h, w)
    ref = V.get_image_features(sd16, px, interpolate_pos_encoding=ipe)
    gold = torch.from_numpy(golden16[f"image_features_{V.size_key(h, w)}"])
    assert _cos_err(ref, gold) < 1e-9
    worst = {}
    for name, eng in (("bf16", eng16), ("fp16", eng16h)):
        out = eng.encode_images(px.cuda(), interpolate_pos_encoding=ipe)
        assert out.shape == (2, 512)
        worst[f"{name}/f32"] = _cos_err(out, ref)
        worst[f"{name}/bf16px"] = _cos_err(eng.encode_images(px.cuda().to(torch.bfloat16), interpolate_pos_encoding=ipe),
                                           ref)
        u8 = _u8(2, h, w, h * w)
        worst[f"{name}/u8"] = _cos_err(eng.encode_images(u8.cuda(), interpolate_pos_encoding=ipe),
                                       V.get_image_features(sd16, O.preprocess_u8(u8), interpolate_pos_encoding=ipe))
    print(f"ViT-B/16 1-cos {h}x{w}: " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))
    assert max(worst.values()) <= COS_TOL, worst


def test_text_tower_unchanged_by_patch(eng16, sd16, state_dict):
    """A ViT-B/32 engine with the same text weights (make_state_dict draws the text tower first, text_projection last)
    returns the same text embeddings, bit for bit."""
    mixed = dict(state_dict)
    mixed.update({k: v for k, v in sd16.items() if k.startswith("text") or k == "logit_scale"})
    eng32 = Engine(mixed, max_micro_batch=64)
    try:
        ids, mask = synth.token_ids(5)
        assert torch.equal(eng16.encode_text(ids.cuda(), mask.cuda()), eng32.encode_text(ids.cuda(), mask.cuda()))
    finally:
        eng32.close()


# ---- 5. micro-batches -------------------------------------------------------------------------------------------------
def test_micro_batches(eng16, sd16):
    px = pixel_values_hw(37, 224, 224, seed=11).cuda()         # 16 images per pass: 3 passes
    whole = eng16.encode_images(px)
    single = torch.cat([eng16.encode_images(px[i:i + 1]) for i in range(37)])
    assert torch.equal(whole, single)
    host = eng16.encode_images_host(px.cpu())
    assert torch.equal(host, whole.cpu())
    eng16.profile(True)
    try:
        eng16.encode_images(px[:2])
        names = {r["name"]: r for r in eng16.profile_read()}
    finally:
        eng16.profile(False)
    assert names["vision/attention[long]"]["launches"] == 12 and "vision/attention" not in names
    assert names["vision/gemm[patch_embed]"]["flops"] == 2 * 2 * 196 * 768 * 768
    small = Engine(sd16, max_micro_batch=4)                    # 200 token rows: one 197-token image per pass
    try:
        assert torch.equal(small.encode_images(px[:3]), whole[:3])
    finally:
        small.close()
    with pytest.raises(RuntimeError, match=r"max_micro_batch must be >= 4"):
        Engine(sd16, max_micro_batch=3)


# ---- 6. per-token outputs -----------------------------------------------------------------------------------------------
def test_vision_outputs_vs_oracle(eng16, sd16, golden16):
    model = PlipCLIPModel(sd16, max_micro_batch=16)
    px = pixel_values_hw(2, 224, 224)
    try:
        out = model.vision_model(pixel_values=px.cuda(), output_hidden_states=True, output_attentions=True)
    finally:
        model.engine.close()
    assert len(out.hidden_states) == 13 and all(h.shape == (2, 197, 768) for h in out.hidden_states)
    assert len(out.attentions) == 12 and all(a.shape == (2, 12, 197, 197) for a in out.attentions)
    ref32 = V.vision_outputs(sd16, px)
    ref16 = V.vision_outputs(sd16, px, dt=torch.bfloat16)
    for l in range(13):
        d = (out.hidden_states[l].cpu() - ref32["hidden_states"][l]).abs()
        assert d.max().item() < 0.05 and d.mean().item() < 6e-3, (l, d.max().item(), d.mean().item())
        assert torch.equal(out.hidden_states[l], eng16.hidden_states("vision", px.cuda(), l)), l
    worst = 0.0
    for l in range(12):
        bound = max(4 * (ref32["attentions"][l] - ref16["attentions"][l]).abs().max().item(), 2e-3)
        e = (out.attentions[l].cpu() - ref32["attentions"][l]).abs().max().item()
        worst = max(worst, e / bound)
        assert e <= bound, (l, e, bound)
    print(f"ViT-B/16 attentions: worst err / bound {worst:.2f}")
    assert ((torch.stack(out.attentions).sum(-1) - 1).abs() < 1e-4).all()
    g = torch.from_numpy(golden16["vision_attn_11_224x224"])
    assert (out.attentions[11][:1, :, :4].cpu() - g).abs().max().item() < 2e-2
    d = (out.pooler_output.cpu() - ref32["pooler_output"]).abs()
    assert d.max().item() < 0.05
    assert torch.equal(eng16.vision_outputs(px.cuda())["embeds"], eng16.encode_images(px.cuda()))


# ---- 7. forward, pair, host input, pruning -----------------------------------------------------------------------------
# n = 6 without graph replay runs both towers of encode_pair side by side; with it, and for n = 40 (more than the 16
# images of one pass), encode_pair is the two calls
@pytest.mark.parametrize("n,graphs", [(6, False), (6, True), (40, True)])
def test_forward_equals_separate_calls(sd16, n, graphs, monkeypatch):
    if not graphs:
        monkeypatch.setenv("PLIP_GRAPH_MAX", "0")
    model = PlipCLIPModel(sd16, max_micro_batch=64)
    eng = model.engine
    try:
        px = pixel_values_hw(n, 224, 224, seed=n).cuda()
        ids, mask = synth.token_ids(n, seed=n)
        ids, mask = ids.cuda(), mask.cuda()
        img = eng.encode_images(px, normalize=True)
        txt = eng.encode_text(ids, mask, normalize=True)
        lpi = eng.similarity(img, txt, normalize_image=False, normalize_text=False)
        for _ in range(2):                                       # a second call replays whatever the first set up
            out = model(input_ids=ids, pixel_values=px, attention_mask=mask, return_loss=True)
            assert torch.equal(out.image_embeds, img) and torch.equal(out.text_embeds, txt)
            assert torch.equal(out.logits_per_image, lpi) and torch.equal(out.logits_per_text, lpi.t())
        tgt = torch.arange(n, device="cuda")
        loss = (torch.nn.functional.cross_entropy(lpi.t(), tgt) + torch.nn.functional.cross_entropy(lpi, tgt)) / 2
        assert torch.equal(out.loss, loss)
        pi, pt = eng.encode_pair(px, ids, mask)
        assert torch.equal(pi, img) and torch.equal(pt, txt)
        host = model(input_ids=ids.cpu(), pixel_values=px.cpu(), attention_mask=mask.cpu())
        assert torch.equal(host.logits_per_image, lpi)
        eng.set_last_layer_pruning(True)
        try:
            assert torch.equal(eng.encode_images(px, normalize=True), img)
            p2i, p2t = eng.encode_pair(px, ids, mask)
            assert torch.equal(p2i, img) and torch.equal(p2t, txt)
        finally:
            eng.set_last_layer_pruning(False)
        ref = O.l2_normalize(V.get_image_features(sd16, px.cpu()))
        ref_t = O.l2_normalize(O.get_text_features(sd16, ids.cpu(), mask.cpu()))
        dl = (lpi.cpu() - O.similarity(ref, ref_t, float(sd16["logit_scale"].exp()))).abs().max().item()
        print(f"ViT-B/16 forward |dlogits| {dl:.2e}")
        assert dl < 1e-2
    finally:
        eng.close()


def test_hires_forward_and_pruning(eng16):
    px = pixel_values_hw(5, 320, 448, seed=5).cuda()
    full = eng16.encode_images(px, interpolate_pos_encoding=True)
    eng16.set_last_layer_pruning(True)
    try:
        assert torch.equal(eng16.encode_images(px, interpolate_pos_encoding=True), full)
    finally:
        eng16.set_last_layer_pruning(False)


# ---- 8. determinism ---------------------------------------------------------------------------------------------------------
def test_deterministic(eng16):
    px = _u8(33, 224, 224, 2).cuda()
    assert torch.equal(eng16.encode_images(px), eng16.encode_images(px))
    q = pixel_values_hw(3, 512, 512).cuda()
    assert torch.equal(eng16.encode_images(q, interpolate_pos_encoding=True),
                       eng16.encode_images(q, interpolate_pos_encoding=True))


# ---- 9. a ViT-B/32 engine is unchanged ----------------------------------------------------------------------------------------
def test_b32_create_patch_equals_create_ex(state_dict, engine):
    L = lib()
    blob, scale = pack_state_dict(state_dict)
    hs = []
    try:
        for fn, args in (("plip_create_ex", (0,)), ("plip_create_patch", (0, 32))):
            h = C.c_void_p()
            check(getattr(L, fn)(blob.data_ptr(), blob.numel(), C.c_float(scale), 0, 16, *args, C.byref(h)), fn)
            hs.append(h)
        assert [L.plip_vision_patch(h) for h in hs] == [32, 32]
        px = _u8(20, 224, 224, 5).cuda()
        outs = []
        for h in hs:
            o = torch.empty(20, 512, device="cuda")
            check(L.plip_encode_images(h, px.data_ptr(), 2, 20, o.data_ptr(), 0, _stream()), "encode_images")
            outs.append(o)
        assert torch.equal(outs[0], outs[1])
        b16, _ = pack_state_dict(make_state_dict(1, "hf_init", patch=16))
        h = C.c_void_p()
        assert L.plip_create_patch(b16.data_ptr(), b16.numel(), C.c_float(1.0), 0, 16, 0, 32, C.byref(h)) != 0
        assert L.plip_create_patch(blob.data_ptr(), blob.numel(), C.c_float(1.0), 0, 16, 0, 8, C.byref(h)) != 0
    finally:
        for h in hs:
            L.plip_destroy(h)


# ---- 10. EmbedderFactory ------------------------------------------------------------------------------------------------------
def test_factory_vitb16(sd16, tmp_path, monkeypatch):
    from plip_b200.embedders import EmbedderFactory
    path = tmp_path / "ViT-B-16.pt"
    torch.save(_to_openai(sd16), path)
    monkeypatch.setenv("PC_CLIP_ARCH", "ViT-B/16")
    monkeypatch.setenv("PLIP_B200_OPENAI_CLIP", str(path))
    import sys
    monkeypatch.setitem(sys.modules, "clip", None)
    imgs = [np.random.default_rng(i).integers(0, 256, (224, 224, 3), dtype=np.uint8) for i in range(5)]
    ref = O.l2_normalize(V.get_image_features(sd16, O.preprocess_u8(torch.from_numpy(np.stack(imgs))))).numpy()
    for name, backbone in (("clip", "unused.pt"), ("plip", str(path))):
        emb = EmbedderFactory().factory(Namespace(model_name=name, backbone=backbone))
        try:
            assert emb.model.engine.vision_patch == 16
            rows = emb.image_embedder(imgs, batch_size=4)
            assert rows.shape == (5, 512) and rows.dtype == np.float32
            assert np.allclose(np.linalg.norm(rows, axis=1), 1, atol=1e-6)
            assert (1 - (rows.astype(np.float64) * ref).sum(1)).max() < COS_TOL
        finally:
            emb.model.engine.close()
