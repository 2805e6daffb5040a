"""CLIP ViT-B/16 on the host: the oracle against the live-transformers golden vectors, the ViT-B/16 blob layout, the
packer, the checkpoint checks of ``PlipCLIPModel.from_pretrained`` and ``EmbedderFactory``, and patch-size inference
from HF and OpenAI-clip key sets.  Nothing here builds an engine."""
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

import vitb16_oracle as V
from oracle import clip_oracle as O
from plip_b200 import weights as W
from plip_b200._lib import lib
from plip_b200.synthetic import make_state_dict, pixel_values_hw
from test_weights import _to_openai

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vitb16_golden.npz")


@pytest.fixture(scope="module")
def sd16():
    torch.set_grad_enabled(False)
    return make_state_dict(0, "rich", patch=16)


@pytest.fixture(scope="module")
def golden16():
    return dict(np.load(GOLDEN, allow_pickle=False))


# ---- 1. the oracle against transformers ---------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", V.SIZES)
def test_oracle_image_features_vs_golden(sd16, golden16, h, w):
    px = pixel_values_hw(2, h, w)
    got = V.get_image_features(sd16, px, interpolate_pos_encoding=(h, w) != (224, 224))
    ref = torch.from_numpy(golden16[f"image_features_{V.size_key(h, w)}"])
    assert (1 - O.cosine(got, ref)).max().item() < 1e-9
    assert (got - ref).abs().max().item() < 1e-4 * ref.abs().max().item()


@pytest.mark.parametrize("h,w", V.SIZES[:2])
def test_oracle_hidden_states_and_attentions_vs_golden(sd16, golden16, h, w):
    px = pixel_values_hw(2, h, w)
    out = V.vision_outputs(sd16, px, interpolate_pos_encoding=(h, w) != (224, 224))
    S = (h // 16) * (w // 16) + 1
    assert out["hidden_states"][0].shape == (2, S, 768) and out["attentions"][0].shape == (2, 12, S, S)
    k = V.size_key(h, w)
    for l in (0, 1, 12):
        hs = out["hidden_states"][l]
        got = torch.cat([hs[:1, :5], hs[:1, -5:]], dim=1)
        ref = torch.from_numpy(golden16[f"vision_hidden_{l}_{k}"])
        assert (got - ref).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item()), l
    for l in (0, 11):
        got = out["attentions"][l][:1, :, :4]
        ref = torch.from_numpy(golden16[f"vision_attn_{l}_{k}"])
        assert (got - ref).abs().max().item() < 1e-6, l


def test_oracle_224_is_the_stored_table(sd16):
    """224..239 px give the 14 x 14 grid and the stored table: the same embeddings as the 224 crop."""
    px = pixel_values_hw(1, 239, 239)
    a = V.vision_embeddings(sd16, px, interpolate_pos_encoding=True)
    b = V.vision_embeddings(sd16, px[:, :, :224, :224].contiguous())
    assert torch.equal(a, b)


def test_pos_interp_ref_of_14_grid_is_identity_at_14(sd16):
    pos = sd16["vision_model.embeddings.position_embedding.weight"]
    ref, slack = V.pos_interp_ref(pos, 14, 14)
    assert torch.equal(ref, pos.double()) and slack.max().item() < 1e-6
    ref, _ = V.pos_interp_ref(pos, 20, 28)
    assert (ref.float() - V.HO.interpolate_pos(pos, 20, 28)).abs().max().item() < 1e-6


def test_synthetic_b32_draws_unchanged():
    a, b = make_state_dict(3, "hf_init"), make_state_dict(3, "hf_init", patch=32)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    c = make_state_dict(3, "hf_init", patch=16)
    assert c["vision_model.embeddings.patch_embedding.weight"].shape == (768, 3, 16, 16)
    assert c["vision_model.embeddings.position_embedding.weight"].shape == (197, 768)


# ---- 2. the blob layout -------------------------------------------------------------------------------------------
def test_vitb16_tensor_table_differs_in_two_tensors():
    L = lib()
    t32, t16 = W.tensor_table(32), W.tensor_table(16)
    assert len(t32) == len(t16) == L.plip_weights_num_tensors()
    differ = {}
    for a, b in zip(t32, t16):
        assert a.name == b.name and a.dtype == b.dtype and a.fused == b.fused
        if (a.rows, a.cols) != (b.rows, b.cols):
            differ[a.name.decode()] = (b.rows, b.cols)
    assert differ == {"vision_model.embeddings.patch_embedding.weight": (768, 768),
                      "vision_model.embeddings.position_embedding.weight": (197, 768)}
    for prev, ti in zip(t16, t16[1:]):                       # packed in order, 256-byte aligned
        assert ti.offset % 256 == 0 and ti.offset >= prev.offset + prev.numel * (2 if prev.dtype == 1 else 4)
    last = t16[-1]
    assert L.plip_weights_blob_bytes_patch(16) == (last.offset + last.numel * 2 + 255) // 256 * 256
    assert L.plip_weights_blob_bytes_patch(32) == L.plip_weights_blob_bytes()
    assert L.plip_weights_blob_bytes_patch(14) == 0
    with pytest.raises(RuntimeError, match="patch size 14"):
        W.tensor_table(14)


def test_pack_vitb16(sd16):
    blob, scale = W.pack_state_dict(sd16)
    assert blob.numel() == lib().plip_weights_blob_bytes_patch(16)
    table = {ti.name.decode(): ti for ti in W.tensor_table(16)}

    def view(ti, dt):
        n = ti.numel * (2 if ti.dtype == 1 else 4)
        return blob[ti.offset:ti.offset + n].view(dt)

    pe = sd16["vision_model.embeddings.patch_embedding.weight"]
    assert torch.equal(view(table["vision_model.embeddings.patch_embedding.weight"], torch.bfloat16),
                       pe.reshape(-1).to(torch.bfloat16))
    pos = sd16["vision_model.embeddings.position_embedding.weight"]
    assert torch.equal(view(table["vision_model.embeddings.position_embedding.weight"], torch.float32), pos.reshape(-1))
    blob_oa, s2 = W.pack_state_dict(_to_openai(sd16))
    assert s2 == scale and torch.equal(blob_oa, blob)


# ---- 3. patch-size inference --------------------------------------------------------------------------------------
def test_patch_inferred_from_hf_and_openai_keys(sd16, state_dict):
    assert W.vision_patch(sd16) == 16 and W.vision_patch(state_dict) == 32
    assert W.vision_patch(_to_openai(sd16)) == 16 and W.vision_patch(_to_openai(state_dict)) == 32
    assert W.vision_patch({"model." + k: v for k, v in sd16.items()}) == 16
    bad = dict(sd16)
    bad["vision_model.embeddings.patch_embedding.weight"] = torch.zeros(768, 3, 14, 14)
    with pytest.raises(ValueError, match="ViT-B/32 and ViT-B/16 geometries only.*'vision patch_size': 14"):
        W.vision_patch(bad)
    with pytest.raises(ValueError, match="patch_size"):
        W.pack_state_dict(bad)


# ---- 4. checkpoint checks -----------------------------------------------------------------------------------------
def test_from_pretrained_config_check():
    from transformers import CLIPConfig

    from plip_b200.modeling import check_config
    check_config(CLIPConfig())
    check_config(CLIPConfig(vision_config={"patch_size": 16, "hidden_act": "quick_gelu"}))
    for vc, field in (({"patch_size": 14}, "vision patch_size"), ({"patch_size": 8}, "vision patch_size"),
                      ({"patch_size": 16, "hidden_size": 1024, "num_attention_heads": 16}, "vision hidden_size"),
                      ({"patch_size": 16, "image_size": 336}, "vision image_size")):
        with pytest.raises(ValueError, match=f"ViT-B/32 and ViT-B/16 geometries only.*{field}"):
            check_config(CLIPConfig(vision_config=vc))


@pytest.fixture
def no_clip_cache(tmp_path, monkeypatch):
    monkeypatch.setenv("HOME", str(tmp_path))
    monkeypatch.delenv("PLIP_B200_OPENAI_CLIP", raising=False)
    import sys
    monkeypatch.setitem(sys.modules, "clip", None)        # the optional package, absent
    return tmp_path


@pytest.mark.parametrize("arch", ["ViT-L/14", "RN50", "ViT-B/14"])
def test_factory_rejects_other_archs(arch, monkeypatch):
    from plip_b200.embedders import EmbedderFactory
    monkeypatch.setenv("PC_CLIP_ARCH", arch)
    for name in ("plip", "clip"):
        with pytest.raises(ValueError, match=r"ViT-B/32 and ViT-B/16 only"):
            EmbedderFactory().factory(Namespace(model_name=name, backbone="unused.pt"))


def test_factory_vitb16_looks_for_its_weights(no_clip_cache, monkeypatch):
    from plip_b200.embedders import EmbedderFactory
    monkeypatch.setenv("PC_CLIP_ARCH", "ViT-B/16")
    with pytest.raises(FileNotFoundError, match=r"ViT-B/16 weights.*ViT-B-16\.pt"):
        EmbedderFactory().factory(Namespace(model_name="clip", backbone="unused.pt"))


def test_factory_rejects_weights_of_the_other_arch(no_clip_cache, monkeypatch, state_dict, sd16):
    """The reference loads the file into clip.load(arch)'s model, strictly: weights of the other patch size fail
    before any engine is built."""
    from plip_b200.embedders import EmbedderFactory
    p32, p16 = no_clip_cache / "b32.pt", no_clip_cache / "b16.pt"
    torch.save(_to_openai(state_dict), p32)
    torch.save(_to_openai(sd16), p16)
    monkeypatch.setenv("PC_CLIP_ARCH", "ViT-B/16")
    with pytest.raises(ValueError, match="needs 16-pixel patches; the weights of .*b32.pt have 32-pixel"):
        EmbedderFactory().factory(Namespace(model_name="plip", backbone=str(p32)))
    monkeypatch.setenv("PLIP_B200_OPENAI_CLIP", str(p32))
    with pytest.raises(ValueError, match="needs 16-pixel patches; the weights of OpenAI's pretrained checkpoint have 32"):
        EmbedderFactory().factory(Namespace(model_name="clip", backbone="unused.pt"))
    monkeypatch.setenv("PC_CLIP_ARCH", "ViT-B/32")
    with pytest.raises(ValueError, match="needs 32-pixel patches; the weights of .*b16.pt have 16-pixel"):
        EmbedderFactory().factory(Namespace(model_name="plip", backbone=str(p16)))
