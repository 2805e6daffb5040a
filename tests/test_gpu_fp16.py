"""The fp16 operand format (``Engine(..., operand_dtype="fp16")`` / ``plip_create_ex``): same kernels with IEEE-half
GEMM / attention operands.  Bounds are 2-3x what the CPU emulation of this contract gives
(tools/precision_study.py: 1-cos 9e-8 / 4e-7, |dlogits| 1.7e-3 max over 64 x 32)."""
import pytest
import torch

from oracle import clip_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model16(state_dict):
    from plip_b200.modeling import PlipCLIPModel
    m = PlipCLIPModel(state_dict, max_micro_batch=64, operand_dtype="fp16")
    yield m
    m.engine.close()


def test_fp16_operands_embeddings_and_logits(model16, engine, state_dict):
    assert model16.engine.operand_dtype == "fp16" and engine.operand_dtype == "bf16"
    px = synth.pixel_values(64)
    ids, mask = synth.token_ids(32)
    ref = O.clip_forward(state_dict, ids, px, mask)
    out = model16(input_ids=ids.cuda(), pixel_values=px.cuda(), attention_mask=mask.cuda())
    ci = (1 - O.cosine(out.image_embeds.cpu(), ref["image_embeds"])).max().item()
    ct = (1 - O.cosine(out.text_embeds.cpu(), ref["text_embeds"])).max().item()
    d16 = (out.logits_per_image.cpu() - ref["logits_per_image"]).abs()
    img_b = engine.encode_images(px.cuda(), normalize=True)
    txt_b = engine.encode_text(ids.cuda(), mask.cuda(), normalize=True)
    db = (engine.similarity(img_b, txt_b, normalize_image=False, normalize_text=False).cpu() - ref["logits_per_image"]).abs()
    print(f"fp16 operands: 1-cos image {ci:.2e} text {ct:.2e} |dlogits| max {d16.max().item():.2e} mean {d16.mean().item():.2e}"
          f"  (bf16 operands: max {db.max().item():.2e} mean {db.mean().item():.2e})")
    assert ci < 2e-6 and ct < 5e-6, (ci, ct)
    assert d16.max().item() < 4e-3 and d16.mean().item() < 1.2e-3, (d16.max().item(), d16.mean().item())
    assert d16.mean().item() < 0.5 * db.mean().item()                 # the point of the mode
    assert db.max().item() < 2.5e-2                                   # bf16 contract: emulated 1.0e-2 on these inputs
    # uint8 tiles and bf16 pixels through the fp16 engine
    tiles = torch.from_numpy(synth.tiles_u8(8, seed=0))
    o8 = model16.engine.encode_images(tiles.cuda()).cpu()
    assert (1 - O.cosine(o8, O.get_image_features(state_dict, O.preprocess_u8(tiles)))).max().item() < 2e-6
    ob = model16.engine.encode_images(px[:8].to(torch.bfloat16).cuda()).cpu()
    assert (1 - O.cosine(ob, O.get_image_features(state_dict, px[:8].to(torch.bfloat16).float()))).max().item() < 2e-6


def test_fp16_attention_kernel_hook():
    from plip_b200._lib import check, lib
    L = lib()
    check(L.plip_dbg_set_operand_format(1), "fmt")
    try:
        for n_seq, S, heads, causal in ((7, 50, 12, False), (5, 77, 8, True), (6, 20, 8, True)):
            D = heads * 64
            g = torch.Generator().manual_seed(S)
            qkv = torch.randn(n_seq * S, 3 * D, generator=g).cuda().to(torch.float16)
            out = torch.zeros(n_seq * S, D, device="cuda", dtype=torch.float16)
            check(L.plip_dbg_attention(qkv.data_ptr(), n_seq, S, heads, int(causal), None, out.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), "attention")
            torch.cuda.synchronize()
            q, k, v = qkv.float().view(n_seq, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
            att = q @ k.transpose(-1, -2)
            if causal:
                att = att + torch.full((S, S), float("-inf"), device="cuda").triu(1)
            ref = (torch.softmax(att, -1) @ v).permute(0, 2, 1, 3).reshape(n_seq * S, D)
            err = (out.float() - ref).abs()
            assert err.max().item() < 6e-3 and err.mean().item() < 4e-4, (S, err.max().item(), err.mean().item())
    finally:
        check(L.plip_dbg_set_operand_format(0), "fmt")


def test_text_pooling_without_eos(state_dict):
    """Rows without an eos token: position 0 by default (HF, eos_token_id 49407), argmax of the ids in legacy mode."""
    from plip_b200.engine import Engine
    eng = Engine(state_dict, max_micro_batch=16)
    ids, _ = synth.token_ids(6, seed=3, min_len=30)
    ids[ids == 49407] = 1000                     # no eos anywhere
    ids[:, 0] = 1234                             # ... and no bos either (49406 would be the largest id, at position 0)
    ids[:, 17] = 49405                           # the largest id of every row sits at position 17
    ids[2, 9] = 49405                            # ... first occurrence wins
    ref0 = O.get_text_features(state_dict, ids)                                    # (ids == eos).argmax() -> 0
    x = O.text_transformer(state_dict, ids, eos_token_id=2)                        # legacy: argmax(ids)
    ref_legacy = O.linear(x, state_dict["text_projection.weight"])
    out0 = eng.encode_text(ids.cuda()).cpu()
    assert (1 - O.cosine(out0, ref0)).max().item() < 1e-4
    eng.set_text_pooling(True)
    out1 = eng.encode_text(ids.cuda()).cpu()
    assert (1 - O.cosine(out1, ref_legacy)).max().item() < 1e-4
    assert (1 - O.cosine(out1, ref0)).max().item() > 1e-3                          # the two conventions really differ here
    eng.close()
