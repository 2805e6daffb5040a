"""Whole-path parity on the GPU: CUDA engine vs the oracle and the committed golden vectors.

Tolerances (stated by BASELINE.json's north_star / SURVEY.md §7): per-vector embedding cosine >= 1 - 1e-4
vs the fp32 reference; |dlogits| <= 1e-3 for the similarity head on identical embeddings; end-to-end
logits (bf16 GEMM operands upstream) are reported against a looser, explicitly stated bound."""
import numpy as np
import PIL.Image
import pytest
import torch

from oracle import clip_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu
COS_TOL = 1e-4


def _t(a):
    return torch.from_numpy(np.asarray(a))


def test_vision_hidden_states_layerwise(engine, state_dict):
    px = synth.pixel_values(4)
    hid = []
    O.vision_transformer(state_dict, px, hidden=hid)
    for nl in (0, 1, 6, 12):
        h = engine.hidden_states("vision", px.cuda(), nl).cpu()
        d = (h - hid[nl]).abs()
        assert d.max().item() < 0.05 and d.mean().item() < 6e-3, (nl, d.max().item(), d.mean().item())


def test_text_hidden_states_layerwise(engine, state_dict):
    ids, mask = synth.token_ids(4)
    hid = []
    O.text_transformer(state_dict, ids, mask, hidden=hid)
    h0 = engine.hidden_states("text", ids.cuda(), 0, attention_mask=mask.cuda()).cpu()
    assert torch.equal(h0, hid[0])                     # embedding gather + add is exact fp32
    for nl in (1, 12):
        h = engine.hidden_states("text", ids.cuda(), nl, attention_mask=mask.cuda()).cpu()
        d = (h - hid[nl]).abs()
        assert d.max().item() < 0.08 and d.mean().item() < 8e-3, (nl, d.max().item(), d.mean().item())


def test_image_embeddings_vs_golden_and_oracle(engine, state_dict, golden):
    px = synth.pixel_values(8)
    out = engine.encode_images(px.cuda()).cpu()
    assert out.shape == (8, 512) and out.dtype == torch.float32
    assert (1 - O.cosine(out, _t(golden["image_features"]))).max().item() < COS_TOL
    assert (1 - O.cosine(out, O.get_image_features(state_dict, px))).max().item() < COS_TOL
    outb = engine.encode_images(px.cuda().to(torch.bfloat16)).cpu()
    assert (1 - O.cosine(outb, _t(golden["image_features"]))).max().item() < COS_TOL
    outn = engine.encode_images(px.cuda(), normalize=True).cpu()
    assert (outn - _t(golden["image_embeds"])).abs().max().item() < 2e-3
    assert (outn.norm(dim=-1) - 1).abs().max().item() < 1e-5


def test_text_embeddings_vs_golden(engine, golden):
    ids, mask = synth.token_ids(8)
    out = engine.encode_text(ids.cuda(), mask.cuda()).cpu()
    assert (1 - O.cosine(out, _t(golden["text_features"]))).max().item() < COS_TOL
    out32 = engine.encode_text(ids.to(torch.int32).cuda()).cpu()          # int32 ids, no mask
    assert torch.equal(out32, out)                                       # eos padding + causality: mask is a no-op
    idf, mf = synth.token_ids(4, seed=77, full_length=True)
    outf = engine.encode_text(idf.cuda(), mf.cuda()).cpu()
    assert (1 - O.cosine(outf, _t(golden["text_features_full77"]))).max().item() < COS_TOL


def test_text_real_padding_mask_and_short_sequences(engine, state_dict):
    """Masks that actually change the result (zeros before the eos) and seq_len < 77."""
    ids, mask = synth.token_ids(6, seed=5, min_len=20)
    mask2 = mask.clone()
    mask2[:, 3:6] = 0
    ref = O.get_text_features(state_dict, ids, mask2)
    out = engine.encode_text(ids.cuda(), mask2.cuda()).cpu()
    assert (1 - O.cosine(out, ref)).max().item() < COS_TOL
    short = ids[:, :24].clone()
    short[:, 23] = 49407
    ref_s = O.get_text_features(state_dict, short, None)
    out_s = engine.encode_text(short.cuda()).cpu()
    assert (1 - O.cosine(out_s, ref_s)).max().item() < COS_TOL


def test_text_prefix_processing_is_exact(engine, state_dict):
    """Short prompts (the common case: ~12 of 77 tokens): only the prefix up to the longest first-eos is
    processed.  Causality makes that exact; compare with the full-length run and with the oracle."""
    ids, mask = synth.token_ids(40, seed=21, min_len=5)
    lens = mask.sum(1)
    keep = lens <= 20
    ids, mask = ids[keep][:12], mask[keep][:12]
    assert ids.shape[0] >= 4
    longest = int(mask.sum(1).max())
    full = engine.encode_text(ids.cuda(), mask.cuda()).cpu()
    pre = engine.encode_text(ids.cuda(), mask.cuda(), prefix_len=longest).cpu()
    host = engine.encode_text_host(ids, mask)                          # scans the ids, picks the prefix itself
    ref = O.get_text_features(state_dict, ids, mask)
    assert (1 - O.cosine(pre, full)).max().item() < 1e-5
    assert torch.equal(host, pre)
    assert (1 - O.cosine(pre, ref)).max().item() < COS_TOL
    with pytest.raises(ValueError):
        engine.encode_text(ids.cuda(), prefix_len=78)


def test_uint8_tiles_and_reference_plip_cfg1(engine, golden):
    """cfg1 through the device u8 path: matches the reference PLIP.encode_images golden."""
    tiles = torch.from_numpy(synth.tiles_u8(32, seed=0))
    out = engine.encode_images(tiles.cuda()).cpu()
    assert (1 - O.cosine(out, _t(golden["ref_plip_encode_images_bs8"]))).max().item() < COS_TOL


def test_similarity_head_and_clip_forward(state_dict, golden):
    from plip_b200.modeling import PlipCLIPModel
    model = PlipCLIPModel(state_dict, max_micro_batch=16)
    eng = model.engine
    # (b) similarity head alone on identical (golden) embeddings: fp32 FMA -> far inside 1e-3
    lg = eng.similarity(_t(golden["image_embeds"]).cuda(), _t(golden["text_embeds"]).cuda()).cpu()
    assert (lg - _t(golden["logits_per_image"])).abs().max().item() < 1e-4
    # (c) end to end: bounded by the bf16-operand towers (SURVEY.md §7: ~1e-2 at exp(logit_scale)=14.3)
    px = synth.pixel_values(8)
    ids, mask = synth.token_ids(8)
    out = model(input_ids=ids.cuda(), pixel_values=px.cuda(), attention_mask=mask.cuda())
    assert out.logits_per_image.shape == (8, 8)
    # measured bound of the bf16-operand contract on this 8 x 8 block (DESIGN.md §2; emulated max 8e-3, GPU r1 3.3e-3 on 4 x 4)
    assert (out.logits_per_image.cpu() - _t(golden["logits_per_image"])).abs().max().item() < 1.0e-2
    assert torch.equal(out.logits_per_text, out.logits_per_image.t())
    assert (1 - O.cosine(out.image_embeds.cpu(), _t(golden["image_embeds"]))).max().item() < COS_TOL
    assert (1 - O.cosine(out.text_embeds.cpu(), _t(golden["text_embeds"]))).max().item() < COS_TOL
    f = model.get_image_features(pixel_values=px.cuda())
    assert torch.is_tensor(f) and f.shape == (8, 512)            # v4-style return: the tensor itself
    assert torch.equal(model.encode_image(px.cuda()), f)
    with pytest.raises(ValueError, match="doesn't match model"):
        model.get_image_features(pixel_values=torch.zeros(1, 3, 256, 256))
    with pytest.raises(ValueError, match="Sequence length"):
        model.get_text_features(input_ids=torch.zeros(1, 78, dtype=torch.long))
    with pytest.raises(ValueError, match="specify input_ids"):
        model(pixel_values=px.cuda())


def test_microbatching_host_path_and_determinism(engine):
    """Size-independent properties: an image's embedding does not depend on its batch neighbours or on the
    micro-batch split; host path == device path; run-to-run bitwise reproducible."""
    tiles = torch.from_numpy(synth.tiles_u8(150, seed=3))          # max_micro_batch = 64 -> 3 passes, ragged tail
    full = engine.encode_images(tiles.cuda()).cpu()
    again = engine.encode_images(tiles.cuda()).cpu()
    assert torch.equal(full, again)
    # Batch composition only changes fp32 summation order inside the PV product (an image sits in the upper or
    # lower half of a packed attention tile): ~1e-7 relative, occasionally amplified to a bf16 ulp by the next
    # rounding.  The embedding must stay far inside the parity bar (1e-4).
    part = engine.encode_images(tiles[37:38].cuda()).cpu()
    d = (1 - O.cosine(part, full[37:38])).max().item()
    assert d < 1e-5, d
    assert torch.equal(engine.encode_images_host(tiles.numpy()), full)
    assert torch.equal(engine.encode_images_host(tiles.pin_memory()), full)
    ids, mask = synth.token_ids(100, seed=9)
    t_full = engine.encode_text(ids.cuda(), mask.cuda()).cpu()
    assert (1 - O.cosine(engine.encode_text_host(ids, mask), t_full)).max().item() < 1e-5   # host path = prefix run
    assert engine.encode_images(torch.zeros(0, 3, 224, 224)).shape == (0, 512)


def test_small_batch_graph_replay_is_bit_identical(engine, state_dict):
    """n <= 128: the first call of a shape runs the launches eagerly and records them as a CUDA graph, later calls
    replay the graph on staged inputs (engine.cu).  Replays must reproduce the eager result bit for bit, for both
    towers, with and without a mask, and must not leak one call's inputs into the next."""
    px = synth.pixel_values(8, seed=51).cuda()
    px2 = synth.pixel_values(8, seed=52).cuda()
    ids, mask = synth.token_ids(8, seed=53)
    ids2, mask2 = synth.token_ids(8, seed=54)
    e1 = engine.encode_images(px).clone()                      # eager + capture
    o2 = engine.encode_images(px2).clone()                     # replay, other input
    e1b = engine.encode_images(px).clone()                     # replay, first input again
    assert torch.equal(e1, e1b) and not torch.equal(e1, o2)
    assert (1 - O.cosine(o2.cpu(), O.get_image_features(state_dict, px2.cpu()))).max().item() < COS_TOL
    t1 = engine.encode_text(ids.cuda(), mask.cuda()).clone()
    t2 = engine.encode_text(ids2.cuda(), mask2.cuda()).clone()
    t1b = engine.encode_text(ids.cuda(), mask.cuda()).clone()
    assert torch.equal(t1, t1b) and not torch.equal(t1, t2)
    assert (1 - O.cosine(t2.cpu(), O.get_text_features(state_dict, ids2, mask2))).max().item() < COS_TOL
    n1 = engine.encode_images(px, normalize=True)              # a different graph key (normalize)
    assert torch.allclose(n1, e1 / e1.norm(dim=1, keepdim=True), atol=1e-6)
    assert (1 - O.cosine(engine.encode_images(px[:3]).cpu(), e1[:3].cpu())).max().item() < 1e-6   # another n / graph


def test_last_layer_pruning_gives_the_same_embeddings(engine, state_dict):
    """plip_set_last_layer_pruning: the last layer's out_proj / LN2 / MLP on the pooled rows only.  Per-row arithmetic is
    unchanged (only the grouping of the LayerNorm-statistics partials can differ with the tile shape), so the
    embeddings must agree with the full run to fp32 rounding — eager (n > 128, several micro-batches), graph replay
    (n <= 128), ragged eos positions, masks, short sequences, no-eos rows — and hidden states must not change."""
    px = synth.pixel_values(8, seed=61).cuda()
    pxl = synth.pixel_values(150, seed=62).cuda()
    ids, mask = synth.token_ids(8, seed=63, min_len=4)
    idl, maskl = synth.token_ids(150, seed=64, min_len=3)
    mask2 = maskl.clone(); mask2[:, 1:3] = 0
    noeos = ids.clone(); noeos[noeos == 49407] = 17; noeos[:, 0] = 1234
    short = ids[:, :24].clone(); short[:, 23] = 49407
    assert not engine.last_layer_pruning
    def run():
        return [engine.encode_images(px).clone(), engine.encode_images(px).clone(), engine.encode_images(pxl).clone(),
                engine.encode_images(pxl, normalize=True).clone(),
                engine.encode_text(ids.cuda(), mask.cuda()).clone(), engine.encode_text(ids.cuda(), mask.cuda()).clone(),
                engine.encode_text(idl.cuda(), mask2.cuda()).clone(), engine.encode_text(idl.cuda()).clone(),
                engine.encode_text(noeos.cuda()).clone(), engine.encode_text(short.cuda()).clone(),
                engine.encode_text(idl.cuda(), maskl.cuda(), prefix_len=int(maskl.sum(1).max())).clone(),
                engine.encode_text_host(idl, maskl).clone(), engine.encode_images_host(pxl.cpu()).clone()]
    full = run()
    hv = engine.hidden_states("vision", px, 12).clone()
    engine.set_last_layer_pruning(True)
    try:
        assert engine.last_layer_pruning
        pruned = run()
        assert torch.equal(engine.hidden_states("vision", px, 12), hv)
    finally:
        engine.set_last_layer_pruning(False)
    for i, (a, b) in enumerate(zip(full, pruned)):
        assert a.shape == b.shape
        rel = ((a - b).abs().max() / a.abs().max()).item()
        assert rel < 2e-5, (i, rel)
    assert (1 - O.cosine(pruned[2].cpu(), O.get_image_features(state_dict, pxl.cpu()))).max().item() < COS_TOL
    assert (1 - O.cosine(pruned[6].cpu(), O.get_text_features(state_dict, idl, mask2))).max().item() < COS_TOL
    assert torch.equal(run()[0], full[0])                       # switched off again: the unpruned graph is replayed


def test_forward_on_host_inputs_equals_device_inputs(state_dict):
    """`model(**inputs)` with HOST tensors (the e2e path of bench.py): pixels are uploaded micro-batch by micro-batch on
    the engine's copy stream while the text tower / the previous micro-batch computes — same logits, bit for bit."""
    from plip_b200.modeling import PlipCLIPModel
    model = PlipCLIPModel(state_dict, max_micro_batch=64)
    tiles = torch.from_numpy(synth.tiles_u8(150, seed=61))
    ids = synth.token_ids(20, seed=62)[0]
    dev = model(input_ids=ids.cuda(), pixel_values=tiles.cuda())
    host = model(input_ids=ids, pixel_values=tiles.pin_memory())
    host2 = model(input_ids=ids, pixel_values=tiles)                      # pageable source
    assert host.logits_per_image.is_cuda and host.logits_per_image.shape == (150, 20)
    assert torch.equal(dev.logits_per_image, host.logits_per_image) and torch.equal(dev.logits_per_image, host2.logits_per_image)
    model.engine.close()


def test_calls_on_different_streams_are_serialised(engine):
    """One handle = one workspace: back-to-back calls on different streams (and the host path right after a
    device call) must not corrupt each other."""
    tiles = torch.from_numpy(synth.tiles_u8(64, seed=11)).cuda()
    ids = synth.token_ids(64, seed=12)[0].cuda()
    ref_i = engine.encode_images(tiles).clone()
    ref_t = engine.encode_text(ids).clone()
    ref_h = engine.hidden_states("vision", tiles, 12).clone()
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for _ in range(3):
        with torch.cuda.stream(s1):
            a = engine.encode_images(tiles)
        with torch.cuda.stream(s2):
            h = engine.hidden_states("vision", tiles, 12)   # right behind the image call on the other stream
            b = engine.encode_text(ids)
        c = engine.encode_images_host(tiles.cpu())          # engine's own streams, right behind the two above
        torch.cuda.synchronize()
        assert torch.equal(a, ref_i) and torch.equal(b, ref_t) and torch.equal(c, ref_i.cpu())
        assert torch.equal(h, ref_h)


def test_plip_class_drop_in(state_dict, golden):
    """The reference-facing class: same call, same return type/shape/order as plip.PLIP (plip.py:31-53)."""
    from plip_b200.plip import PLIP
    p = PLIP.from_state_dict(state_dict, max_micro_batch=16)
    tiles = synth.tiles_u8(32, seed=0)
    pil = [PIL.Image.fromarray(t) for t in tiles]
    for bs in (8, 32):
        emb = p.encode_images(pil, batch_size=bs)
        assert isinstance(emb, np.ndarray) and emb.shape == (32, 512) and emb.dtype == np.float32
        assert (1 - O.cosine(_t(emb), _t(golden["ref_plip_encode_images_bs8"]))).max().item() < COS_TOL
    ids, mask = synth.token_ids(8)
    temb = p.encode_token_ids(ids, mask)
    assert (1 - O.cosine(_t(temb), _t(golden["text_features"]))).max().item() < COS_TOL
    sim = p._cosine_similarity(golden["heads_key"], golden["heads_space"])
    assert np.abs(sim - golden["ref_cosine_similarity"]).max() < 1e-5
    nn = p._nearest_neighbours(5, golden["heads_key"], golden["heads_space"])
    assert np.array_equal(nn, golden["ref_nearest_neighbours_k5"])
    with pytest.raises(ValueError):
        p.encode_images([], batch_size=8)
    with pytest.raises(AttributeError):
        p.retrieval(["x"])


def test_embedder_drop_in(state_dict, golden):
    from plip_b200.embedders import CLIPEmbedder
    from plip_b200.modeling import PlipCLIPModel
    emb = CLIPEmbedder(PlipCLIPModel(state_dict, max_micro_batch=16), None, "plip", "mem")
    tiles = synth.tiles_u8(32, seed=0)
    out = emb.image_embedder([PIL.Image.fromarray(t) for t in tiles], batch_size=8)
    ref = _t(golden["ref_plip_encode_images_bs8"])
    ref = ref / ref.norm(dim=1, keepdim=True)                          # embedders/plip.py:53
    assert out.shape == (32, 512) and np.abs(np.linalg.norm(out, axis=1) - 1).max() < 1e-5
    assert (1 - O.cosine(_t(out), ref)).max().item() < COS_TOL
    ids, _ = synth.token_ids(8)
    tout = emb.text_embedder(list(ids.numpy()), batch_size=4)
    tref = _t(golden["text_embeds"])
    assert (1 - O.cosine(_t(tout), tref)).max().item() < COS_TOL


def test_evaluation_heads(engine):
    """reproducibility/evaluation: dot + argmax / argsort()[-50:][::-1] on the device == numpy."""
    from plip_b200.evaluation import ImageRetrieval, ZeroShotClassifier
    rng = np.random.default_rng(4)
    img = rng.standard_normal((300, 512)).astype(np.float32)
    img /= np.linalg.norm(img, axis=1, keepdims=True)
    txt = img[:120] + 0.05 * rng.standard_normal((120, 512)).astype(np.float32)     # query i matches image i
    labels = [f"c{i}" for i in range(7)]
    cls_emb = rng.standard_normal((7, 512)).astype(np.float32)
    assert ZeroShotClassifier().predict(img, cls_emb, labels) == ZeroShotClassifier(engine).predict(img, cls_emb, labels)
    preds = ZeroShotClassifier().predict(img, cls_emb, labels)       # zero-argument constructor, as the reference's
    assert preds == [labels[int(np.argmax(r))] for r in img.dot(cls_emb.T)]          # zero_shot.py:12-13
    best = ImageRetrieval().best_scores(img, txt)
    ref = np.stack([t.dot(img.T).argsort()[-50:][::-1] for t in txt])                # retrieval.py:13-16
    assert np.array_equal(best, ref)
    train, test = ImageRetrieval(engine).retrieval(img[:120], txt)
    assert test["p@10"] == 1.0 and train["split"] == "train"


def test_full_size_properties(state_dict):
    """BASELINE cfg2 size (batch 1024 bf16): finite, deterministic, consistent with a small-batch run."""
    from plip_b200.engine import Engine
    eng = Engine(state_dict, max_micro_batch=1024)
    px = synth.pixel_values(16).to(torch.bfloat16)
    big = px.repeat(64, 1, 1, 1).cuda()                                  # 1024 images, 16 distinct
    out = eng.encode_images(big)
    assert torch.isfinite(out).all()
    assert torch.equal(out, eng.encode_images(big))
    small = eng.encode_images(px.cuda())
    rep = out.view(64, 16, 512)
    d = (1 - O.cosine(rep[63].cpu(), small.cpu())).max().item()
    assert d < 1e-5, d
    assert (rep - rep[0:1]).abs().max().item() < 2e-2                    # copies agree across tile positions
    eng.close()
