"""Weight packer: HuggingFace ``CLIPModel`` / OpenAI-clip state dicts -> the engine's packed blob.

Replaces ``CLIPModel.from_pretrained`` + ``.to(device)`` (reference ``plip.py:18,26``) and
``clip.load`` + ``load_state_dict(torch.load(path))`` (``reproducibility/embedders/factory.py:20-27``)
as the way weights reach the device.  The blob layout is owned by the CUDA library
(``plip_weights_tensor_info``); this module only fills it:

* GEMM weights are rounded once to bf16 (round-to-nearest-even), everything else stays fp32;
* q/k/v projections are concatenated to one ``[3D, D]`` matrix and the q rows (weight and bias) are
  pre-multiplied by ``head_dim ** -0.5 = 0.125`` (exact: power of two), which is the scale HF applies
  inside the attention core (TF:modeling_clip.py:291,322);
* ``layer_norm1`` / ``layer_norm2`` (TF:371,380) are folded into the GEMM that consumes them:
  ``LN(x) W^T + b = rstd (x (gamma o W)^T - mean colsum) + (b + W beta)`` with
  ``colsum[n] = sum_k bf16(gamma o W)[n,k]``; the device keeps ``bf16(gamma o W)``, ``colsum`` and the
  adjusted bias, never the LayerNorm parameters themselves;
* the conv patch embedding ``[768,3,P,P]`` is viewed as ``[768, 3 P^2]`` (c, ky, kx order).

The vision patch size ``P`` is read from the weights, as OpenAI's ``build_model`` reads it from
``visual.conv1.weight.shape[-1]``: 32 (ViT-B/32, PLIP) or 16 (ViT-B/16).  The two blob layouts differ only in the
patch embedding and the stored position table (``plip_weights_tensor_info_patch``).
"""
from __future__ import annotations

import ctypes as C
import math
import re
from typing import Dict, Mapping, Tuple

import torch

from ._lib import TensorInfo, check, lib

HEAD_SCALE = 0.125  # 64 ** -0.5


def _openai_to_hf(sd: Mapping[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Rename an OpenAI-clip ``CLIP`` state dict (``visual.conv1.weight``, ``transformer.resblocks.N…``;
    naming shown at reference ``fine_tuning/finetune.py:269``) to HuggingFace names."""
    out: Dict[str, torch.Tensor] = {}

    def block(src: str, dst: str, d: int) -> None:
        w, b = sd[f"{src}.attn.in_proj_weight"], sd[f"{src}.attn.in_proj_bias"]
        for i, n in enumerate(("q_proj", "k_proj", "v_proj")):
            out[f"{dst}.self_attn.{n}.weight"] = w[i * d:(i + 1) * d]
            out[f"{dst}.self_attn.{n}.bias"] = b[i * d:(i + 1) * d]
        out[f"{dst}.self_attn.out_proj.weight"] = sd[f"{src}.attn.out_proj.weight"]
        out[f"{dst}.self_attn.out_proj.bias"] = sd[f"{src}.attn.out_proj.bias"]
        for a, bname in (("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"), ("mlp.c_fc", "mlp.fc1"),
                         ("mlp.c_proj", "mlp.fc2")):
            out[f"{dst}.{bname}.weight"] = sd[f"{src}.{a}.weight"]
            out[f"{dst}.{bname}.bias"] = sd[f"{src}.{a}.bias"]

    out["vision_model.embeddings.patch_embedding.weight"] = sd["visual.conv1.weight"]
    out["vision_model.embeddings.class_embedding"] = sd["visual.class_embedding"]
    out["vision_model.embeddings.position_embedding.weight"] = sd["visual.positional_embedding"]
    out["vision_model.pre_layrnorm.weight"] = sd["visual.ln_pre.weight"]
    out["vision_model.pre_layrnorm.bias"] = sd["visual.ln_pre.bias"]
    out["vision_model.post_layernorm.weight"] = sd["visual.ln_post.weight"]
    out["vision_model.post_layernorm.bias"] = sd["visual.ln_post.bias"]
    out["visual_projection.weight"] = sd["visual.proj"].t()
    out["text_model.embeddings.token_embedding.weight"] = sd["token_embedding.weight"]
    out["text_model.embeddings.position_embedding.weight"] = sd["positional_embedding"]
    out["text_model.final_layer_norm.weight"] = sd["ln_final.weight"]
    out["text_model.final_layer_norm.bias"] = sd["ln_final.bias"]
    out["text_projection.weight"] = sd["text_projection"].t()
    out["logit_scale"] = sd["logit_scale"]
    for i in range(12):
        block(f"visual.transformer.resblocks.{i}", f"vision_model.encoder.layers.{i}", 768)
        block(f"transformer.resblocks.{i}", f"text_model.encoder.layers.{i}", 512)
    return out


def normalize_state_dict(sd: Mapping[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Accept HF names (optionally prefixed, e.g. ``model.``) or OpenAI-clip names; return HF names."""
    if "visual.conv1.weight" in sd:
        return _openai_to_hf(sd)
    if "vision_model.embeddings.class_embedding" in sd:
        return dict(sd)
    for k in sd:
        m = re.match(r"^(.*\.)vision_model\.embeddings\.class_embedding$", k)
        if m:
            p = m.group(1)
            return {kk[len(p):]: v for kk, v in sd.items() if kk.startswith(p)}
    raise KeyError("state dict is neither a HuggingFace CLIPModel nor an OpenAI-clip CLIP state dict")


PATCH_SIZES = (32, 16)  # vision patch sizes the engine runs: CLIP ViT-B/32 (PLIP) and ViT-B/16


def vision_patch(sd: Mapping[str, torch.Tensor]) -> int:
    """The vision patch size of a state dict (HF, prefixed HF or OpenAI-clip names): the last dimension of the conv
    patch embedding.  ``ValueError`` for a size the engine does not run."""
    w = normalize_state_dict(sd)["vision_model.embeddings.patch_embedding.weight"]
    patch = int(w.shape[-1])
    if patch not in PATCH_SIZES:
        raise ValueError("plip_b200 implements the CLIP ViT-B/32 and ViT-B/16 geometries only; this checkpoint "
                         f"differs in {{'vision patch_size': {patch}}}")
    return patch


def tensor_table(patch: int = 32):
    """The library's blob layout for a vision patch size (32 or 16) as a list of :class:`TensorInfo`."""
    L = lib()
    infos = []
    for i in range(L.plip_weights_num_tensors()):
        ti = TensorInfo()
        check(L.plip_weights_tensor_info_patch(int(patch), i, C.byref(ti)), "plip_weights_tensor_info_patch")
        infos.append(ti)
    return infos


OPERAND_DTYPES = {"bf16": (0, torch.bfloat16), "bfloat16": (0, torch.bfloat16),
                  "fp16": (1, torch.float16), "float16": (1, torch.float16), "half": (1, torch.float16)}


def operand_format(operand_dtype) -> Tuple[int, torch.dtype]:
    """``"bf16"`` / ``"fp16"`` (or the torch dtype) -> ``(plip_operand_format, torch dtype)``."""
    key = str(operand_dtype).replace("torch.", "")
    if key not in OPERAND_DTYPES:
        raise ValueError(f"operand_dtype must be 'bf16' or 'fp16', got {operand_dtype!r}")
    return OPERAND_DTYPES[key]


def pack_state_dict(state_dict: Mapping[str, torch.Tensor], operand_dtype="bf16") -> Tuple[torch.Tensor, float]:
    """Return ``(blob, exp(logit_scale))``; ``blob`` is a contiguous CPU uint8 tensor in the layout of the weights'
    vision patch size (:func:`vision_patch`).  GEMM weights are rounded once to ``operand_dtype`` (the format the
    engine is created with: ``plip_create_patch``)."""
    _, odt = operand_format(operand_dtype)
    sd = normalize_state_dict(state_dict)
    patch = vision_patch(sd)
    L = lib()
    blob = torch.zeros(int(L.plip_weights_blob_bytes_patch(patch)), dtype=torch.uint8)
    folded = {}  # (base name, "weight"/"bias"/"colsum") -> fp32 tensor, computed once per projection

    def fold(base: str, flags: int):
        """base = '<layer>.self_attn.q_proj' or '<layer>.mlp.fc1' -> folded weight / bias / colsum."""
        if (base, "weight") in folded:
            return
        if flags & 1:
            ws, bs = [], []
            for i, n in enumerate(("q_proj", "k_proj", "v_proj")):
                w = sd[base.replace("q_proj", n) + ".weight"].detach().to(torch.float32)
                b = sd[base.replace("q_proj", n) + ".bias"].detach().to(torch.float32)
                ws.append(w * HEAD_SCALE if i == 0 else w)
                bs.append(b * HEAD_SCALE if i == 0 else b)
            w, b = torch.cat(ws, dim=0), torch.cat(bs, dim=0)
        else:
            w = sd[base + ".weight"].detach().to(torch.float32)
            b = sd[base + ".bias"].detach().to(torch.float32)
        if flags & 2:
            layer = base.rsplit(".", 2)[0]                      # "...encoder.layers.N"
            ln = layer + (".layer_norm1" if "q_proj" in base else ".layer_norm2")
            gamma = sd[ln + ".weight"].detach().to(torch.float32)
            beta = sd[ln + ".bias"].detach().to(torch.float32)
            b = b + w @ beta
            w = (w * gamma[None, :]).to(odt).to(torch.float32)
        folded[(base, "weight")] = w
        folded[(base, "bias")] = b
        folded[(base, "colsum")] = w.to(odt).to(torch.float32).sum(dim=1)

    for ti in tensor_table(patch):
        name = ti.name.decode()
        if ti.fused:
            base, kind = name.rsplit(".", 1)
            fold(base, ti.fused)
            t = folded[(base, kind)]
        else:
            if name not in sd:
                raise KeyError(f"missing weight {name!r}")
            t = sd[name].detach().to(torch.float32)
        t = t.reshape(-1)
        if t.numel() != ti.numel:
            raise ValueError(f"{name}: expected {ti.numel} elements ({ti.rows}x{ti.cols}), got {t.numel()}")
        if ti.dtype == 1:
            raw = t.to(odt).contiguous().view(torch.uint8)
        else:
            raw = t.contiguous().view(torch.uint8)
        blob[ti.offset: ti.offset + raw.numel()] = raw
    scale = float(sd["logit_scale"].detach().float().exp()) if "logit_scale" in sd else math.exp(2.6592)
    return blob, scale
