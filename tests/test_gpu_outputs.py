"""Per-token outputs on the GPU (``output_hidden_states`` / ``output_attentions``): the attention-probabilities kernel
against float64, hidden states bit for bit against the layer-wise hook, the outputs against the CPU oracle, embeddings
left alone, micro-batching, launch accounting and the longest vision sequences."""
import math

import pytest
import torch

import outputs_oracle as OO
from oracle import synth
from plip_b200._lib import check, lib
from plip_b200.modeling import PlipCLIPModel
from plip_b200.synthetic import pixel_values_hw

pytestmark = pytest.mark.gpu
SENTINEL = -7.0e30  # guard rows around the probabilities: bit pattern must survive


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _launches():
    return int(lib().plip_launch_count())


# ---- 1. the probabilities kernel against float64 ------------------------------------------------------------------
def _probs(L, qkv, n_seq, S, heads, causal, km):
    """plip_dbg_attention_probs into a buffer with a sentinel guard of 37 rows on each side."""
    G = 37 * S
    n = n_seq * heads * S * S
    buf = torch.full((n + 2 * G,), SENTINEL, device="cuda", dtype=torch.float32)
    check(L.plip_dbg_attention_probs(qkv.data_ptr(), n_seq, S, heads, int(causal),
                                     km.data_ptr() if km is not None else None, buf[G:].data_ptr(), _stream()),
          "attention_probs")
    torch.cuda.synchronize()
    guard = torch.cat([buf[:G], buf[G + n:]])
    assert torch.equal(guard, torch.full_like(guard, SENTINEL)), "a write left the output"
    return buf[G:G + n].view(n_seq, heads, S, S)


@pytest.mark.parametrize("f16", [0, 1])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("S", [1, 7, 32, 33, 50, 64, 65, 77, 128, 129, 197, 257, 1025])
def test_probs_kernel_vs_float64(S, masked, f16):
    """Bound: the kernel multiplies the same 16-bit q, k exactly and sums 64 products in fp32 (scores here are
    |s| < ~15: absolute error < 1e-5), then exp2 / ex2.approx (2 ulp) and one fp32 reciprocal of the row sum: 1e-4 of
    each probability plus 1e-7 covers that with margin; a wrong mask or row shifts values by ~1/S."""
    L = lib()
    heads = 2 if S > 257 else 3
    n_seq = 2 if S > 257 else 4
    D = heads * 64
    dt = torch.float16 if f16 else torch.bfloat16
    g = torch.Generator().manual_seed(S * 31 + masked)
    qkv = (0.6 * torch.randn(n_seq * S, 3 * D, generator=g)).to(dt)
    km = None
    if masked:
        km = (torch.rand(n_seq, S, generator=g) > 0.3).to(torch.int32)
        km[0, :] = 1
        km[1, 0] = 0                       # sequence 1: row 0 has no visible key (causal + padded position 0)
    check(L.plip_dbg_set_operand_format(f16), "operand format")
    try:
        qd = qkv.cuda()
        got = _probs(L, qd, n_seq, S, heads, masked, km.cuda() if km is not None else None)
        again = _probs(L, qd, n_seq, S, heads, masked, km.cuda() if km is not None else None)
    finally:
        check(L.plip_dbg_set_operand_format(0), "operand format")
    assert torch.equal(got, again)                         # fixed order of operations: bitwise reproducible
    got = got.cpu().double()
    q, k, _ = qkv.double().view(n_seq, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2)                            # q is pre-scaled by 1/8 in the packed weights
    vis = OO.visible_keys(S, km, masked, n_seq)
    s = s.masked_fill(~vis, float("-inf"))
    ref = torch.softmax(s, -1).nan_to_num(0.0)             # rows without a visible key: 0
    err = (got - ref).abs()
    assert (err <= 1e-4 * ref + 1e-7).all(), err.max().item()
    assert torch.equal(got[~vis.expand_as(got)], torch.zeros_like(got[~vis.expand_as(got)]))   # masked: exactly 0
    rows = got.sum(-1)
    empty = ~vis.any(-1).expand_as(rows)
    assert (rows[empty] == 0).all()
    assert ((rows[~empty] - 1).abs() < 1e-4).all(), (rows[~empty] - 1).abs().max().item()
    if masked:
        assert empty[1, :, 0].all()


def test_probs_kernel_rejects_bad_arguments():
    L = lib()
    buf = torch.zeros(16, device="cuda")
    assert L.plip_dbg_attention_probs(buf.data_ptr(), 1, 1026, 12, 0, None, buf.data_ptr(), _stream()) != 0
    assert L.plip_dbg_attention_probs(buf.data_ptr(), 1, 50, 17, 0, None, buf.data_ptr(), _stream()) != 0
    assert L.plip_dbg_attention_probs(None, 1, 50, 12, 0, None, buf.data_ptr(), _stream()) != 0


# ---- 2. hidden states: bitwise against the layer-wise hook, outputs against the oracle -------------------------------
def _hidden_bitwise(engine, tower, x, out, mask=None, ipe=False):
    for layer in range(13):
        ref = engine.hidden_states(tower, x, layer, attention_mask=mask, interpolate_pos_encoding=ipe)
        assert torch.equal(out["hidden_states"][layer], ref), layer


def _close(got, ref, what):
    d = (got.cpu() - ref).abs()
    assert d.max().item() < 0.05 and d.mean().item() < 6e-3, (what, d.max().item(), d.mean().item())


@pytest.mark.parametrize("size", [224, 448])
def test_vision_outputs_hidden_and_oracle(engine, state_dict, size):
    px = pixel_values_hw(3 if size == 224 else 2, size, size, seed=size)
    ipe = size != 224
    out = engine.vision_outputs(px.cuda(), output_hidden_states=True, interpolate_pos_encoding=ipe)
    S = (size // 32) ** 2 + 1
    assert len(out["hidden_states"]) == 13 and out["hidden_states"][0].shape == (px.shape[0], S, 768)
    assert out["attentions"] is None
    assert out["last_hidden_state"].data_ptr() == out["hidden_states"][12].data_ptr()
    _hidden_bitwise(engine, "vision", px.cuda(), out, ipe=ipe)
    ref = OO.vision_outputs(state_dict, px, interpolate_pos_encoding=ipe)
    _close(out["last_hidden_state"], ref["last_hidden_state"], "last_hidden_state")
    _close(out["pooler_output"], ref["pooler_output"], "pooler_output")
    assert torch.equal(out["embeds"], engine.encode_images(px.cuda(), interpolate_pos_encoding=ipe))
    alone = engine.vision_outputs(px.cuda(), interpolate_pos_encoding=ipe)      # no flag: its own last_hidden buffer
    assert torch.equal(alone["last_hidden_state"], out["last_hidden_state"])
    assert torch.equal(alone["pooler_output"], out["pooler_output"])


def test_text_outputs_hidden_and_oracle(engine, state_dict):
    ids, mask = synth.token_ids(3, seed=5)
    mask[1, 4] = 0
    out = engine.text_outputs(ids.cuda(), mask.cuda(), output_hidden_states=True)
    assert out["last_hidden_state"].shape == (3, 77, 512) and out["pooler_output"].shape == (3, 512)
    _hidden_bitwise(engine, "text", ids.cuda(), out, mask=mask.cuda())
    ref = OO.text_outputs(state_dict, ids, mask)
    _close(out["last_hidden_state"], ref["last_hidden_state"], "last_hidden_state")
    _close(out["pooler_output"], ref["pooler_output"], "pooler_output")
    eos = (ids == 49407).int().argmax(-1)
    assert torch.equal(out["pooler_output"].cpu(), out["last_hidden_state"].cpu()[torch.arange(3), eos])
    assert torch.equal(out["embeds"], engine.encode_text(ids.cuda(), mask.cuda()))


# ---- 3. attentions against the oracle ---------------------------------------------------------------------------------
def _attn_bound(ref32, ref16):
    """Emulated device numerics (16-bit operands, oracle dt=bf16) against fp32: the engine may deviate from fp32 by
    at most 4x what the emulation does on the same layer, and never by less than 2e-3 absolute."""
    return [max(4 * (a - b).abs().max().item(), 2e-3) for a, b in zip(ref32["attentions"], ref16["attentions"])]


def _check_attn(got, ref32, bounds, skip_rows=None):
    worst = 0.0
    for layer in range(12):
        g = got[layer].cpu()
        r = ref32["attentions"][layer]
        if skip_rows is not None:
            g, r = g[~skip_rows], r[~skip_rows]
        e = (g - r).abs().max().item()
        worst = max(worst, e / bounds[layer])
        assert e <= bounds[layer], (layer, e, bounds[layer])
    return worst


def test_vision_attentions_vs_oracle(engine, state_dict):
    px = synth.pixel_values(2)
    out = engine.vision_outputs(px.cuda(), output_attentions=True)
    assert len(out["attentions"]) == 12 and out["attentions"][0].shape == (2, 12, 50, 50)
    ref32 = OO.vision_outputs(state_dict, px)
    ref16 = OO.vision_outputs(state_dict, px, dt=torch.bfloat16)
    w = _check_attn(out["attentions"], ref32, _attn_bound(ref32, ref16))
    print(f"vision attentions: worst err / bound {w:.2f}")
    sums = torch.stack(out["attentions"]).sum(-1)
    assert ((sums - 1).abs() < 1e-4).all()


def test_text_attentions_vs_oracle(engine, state_dict):
    ids, mask = synth.token_ids(3, seed=9)
    mask[2, 0] = 0                                           # caption 2: query 0 sees no key
    out = engine.text_outputs(ids.cuda(), mask.cuda(), output_attentions=True)
    A = torch.stack(out["attentions"]).cpu()                 # [12, 3, 8, 77, 77]
    vis = OO.visible_keys(77, mask, True, 3)                 # [3, 1, 77, 77]
    assert torch.equal(A[:, ~vis.expand(3, 8, 77, 77)], torch.zeros_like(A[:, ~vis.expand(3, 8, 77, 77)]))
    assert (A[:, 2, :, 0] == 0).all()                         # the row without a visible key: zeros (HF: uniform)
    ref32 = OO.text_outputs(state_dict, ids, mask)
    ref16 = OO.text_outputs(state_dict, ids, mask, dt=torch.bfloat16)
    empty = ~vis.any(-1).expand(3, 8, 77)                    # rows compared: those with a visible key
    bounds = _attn_bound(ref32, ref16)
    w = _check_attn(out["attentions"], ref32, bounds, skip_rows=empty)
    print(f"text attentions: worst err / bound {w:.2f}")


# ---- 4. the outputs leave the embeddings alone -------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4, 70])       # below / above the CUDA-graph batch limit (n <= max_micro_batch = 64)
def test_forward_with_flags_same_logits(state_dict, n):
    model = PlipCLIPModel(state_dict, max_micro_batch=64)
    try:
        px = synth.pixel_values(n).cuda()
        ids, mask = synth.token_ids(n, seed=n)
        ids, mask = ids.cuda(), mask.cuda()
        base = model(input_ids=ids, pixel_values=px, attention_mask=mask)
        base = model(input_ids=ids, pixel_values=px, attention_mask=mask)          # the replayed graph for n = 4
        full = model(input_ids=ids, pixel_values=px, attention_mask=mask, output_hidden_states=True,
                     output_attentions=True)
        for k in ("logits_per_image", "logits_per_text", "image_embeds", "text_embeds"):
            assert torch.equal(full[k], base[k]), k
        assert base.keys() == ("logits_per_image", "logits_per_text", "text_embeds", "image_embeds")
        assert base.vision_model_output is None and base.text_model_output is None
        assert full.keys()[-2:] == ("text_model_output", "vision_model_output")
        vo, to = full.vision_model_output, full.text_model_output
        assert vo.keys() == ("last_hidden_state", "pooler_output", "hidden_states", "attentions")
        assert len(vo.hidden_states) == 13 and len(to.attentions) == 12 and to.attentions[0].shape == (n, 8, 77, 77)
        only_h = model(input_ids=ids, pixel_values=px, attention_mask=mask, output_hidden_states=True)
        assert only_h.vision_model_output.attentions is None and torch.equal(only_h.logits_per_image,
                                                                              base.logits_per_image)
        sub = model.vision_model(pixel_values=px, output_attentions=True)
        assert torch.equal(sub.attentions[3], vo.attentions[3]) and sub.hidden_states is None
        assert torch.equal(sub.pooler_output, vo.pooler_output)
        tsub = model.text_model(input_ids=ids, attention_mask=mask)
        assert torch.equal(tsub.last_hidden_state, to.last_hidden_state)
    finally:
        model.engine.close()


# ---- 5. micro-batching ----------------------------------------------------------------------------------------------------
def _cat_outputs(parts):
    out = {}
    for k in ("embeds", "pooler_output", "last_hidden_state"):
        out[k] = torch.cat([p[k] for p in parts])
    for k in ("hidden_states", "attentions"):
        out[k] = tuple(torch.cat(t) for t in zip(*[p[k] for p in parts]))
    return out


def _equal_outputs(a, b):
    for k in ("embeds", "pooler_output", "last_hidden_state"):
        assert torch.equal(a[k], b[k]), k
    for k in ("hidden_states", "attentions"):
        assert len(a[k]) == len(b[k])
        for i, (x, y) in enumerate(zip(a[k], b[k])):
            assert torch.equal(x, y), (k, i)


def test_micro_batches_equal_chunks(engine):
    n = 2 * engine.max_micro_batch + 3
    px = synth.pixel_values(n).cuda()
    kw = dict(output_hidden_states=True, output_attentions=True, normalize=True)
    whole = engine.vision_outputs(px, **kw)
    _equal_outputs(whole, engine.vision_outputs(px, **kw))                     # two identical calls
    chunks = [engine.vision_outputs(px[i:i + 50], **kw) for i in range(0, n, 50)]
    _equal_outputs(whole, _cat_outputs(chunks))
    del whole, chunks
    ids, mask = synth.token_ids(n, seed=3)
    ids, mask = ids.cuda(), mask.cuda()
    whole = engine.text_outputs(ids, mask, **kw)
    chunks = [engine.text_outputs(ids[i:i + 50], mask[i:i + 50], **kw) for i in range(0, n, 50)]
    _equal_outputs(whole, _cat_outputs(chunks))


def test_hires_micro_batches_equal_chunks(engine):
    # 3200 token rows per pass -> 16 images of 197 tokens: 19 images take 2 passes
    px = pixel_values_hw(19, 448, 448, seed=2).cuda()
    kw = dict(output_hidden_states=True, output_attentions=True, interpolate_pos_encoding=True)
    whole = engine.vision_outputs(px, **kw)
    _equal_outputs(whole, _cat_outputs([engine.vision_outputs(px[i:i + 7], **kw) for i in range(0, 19, 7)]))
    assert torch.equal(whole["embeds"], engine.encode_images(px, interpolate_pos_encoding=True))


# ---- 6. launch accounting ---------------------------------------------------------------------------------------------------
def test_launch_accounting(engine):
    n = 70                                       # two micro-batches, no graph replay
    px = synth.pixel_values(n).cuda()
    ids, mask = synth.token_ids(n, seed=1)
    ids, mask = ids.cuda(), mask.cuda()

    def count(fn):
        torch.cuda.synchronize()
        c0 = _launches()
        fn()
        torch.cuda.synchronize()
        return _launches() - c0

    enc = count(lambda: engine.encode_images(px, normalize=True))
    assert count(lambda: engine.vision_outputs(px, normalize=True)) == enc      # taps off: the same launches
    h = count(lambda: engine.vision_outputs(px, output_hidden_states=True, normalize=True))
    ha = count(lambda: engine.vision_outputs(px, output_hidden_states=True, output_attentions=True, normalize=True))
    assert h == enc and ha - h == 12 * 2                                     # hidden copies are no kernels
    tenc = count(lambda: engine.encode_text(ids, mask))
    th = count(lambda: engine.text_outputs(ids, mask, output_hidden_states=True))
    tha = count(lambda: engine.text_outputs(ids, mask, output_hidden_states=True, output_attentions=True))
    assert th == tenc + 2 and tha - th == 12 * 2                             # + final_layer_norm of all rows per pass
    engine.profile(True)
    try:
        engine.vision_outputs(px[:3], output_attentions=True)
        engine.text_outputs(ids[:3], mask[:3], output_attentions=True)
        rows = {r["name"]: r for r in engine.profile_read()}
    finally:
        engine.profile(False)
    for tower, heads, S in (("vision", 12, 50), ("text", 8, 77)):
        r = rows[f"{tower}/attention[probs]"]
        assert r["launches"] == 12 and r["bytes"] >= 12 * 3 * heads * S * S * 4


# ---- 7. the longest sequences --------------------------------------------------------------------------------------------
def test_1024_both_flags(engine, state_dict):
    px = pixel_values_hw(1, 1024, 1024, seed=6)
    out = engine.vision_outputs(px.cuda(), output_hidden_states=True, output_attentions=True,
                                interpolate_pos_encoding=True)
    assert out["attentions"][0].shape == (1, 12, 1025, 1025) and out["hidden_states"][12].shape == (1, 1025, 768)
    for layer in (0, 12):
        assert torch.equal(out["hidden_states"][layer],
                           engine.hidden_states("vision", px.cuda(), layer, interpolate_pos_encoding=True))
    ref32 = OO.vision_outputs(state_dict, px, interpolate_pos_encoding=True)
    ref16 = OO.vision_outputs(state_dict, px, dt=torch.bfloat16, interpolate_pos_encoding=True)
    w = _check_attn(out["attentions"], ref32, _attn_bound(ref32, ref16))
    print(f"1024x1024 attentions: worst err / bound {w:.2f}")
    sums = torch.stack(out["attentions"]).sum(-1)
    assert ((sums - 1).abs() < 1e-4).all()
    _close(out["pooler_output"], ref32["pooler_output"], "pooler_output")
    assert math.isfinite(out["last_hidden_state"].abs().max().item())
