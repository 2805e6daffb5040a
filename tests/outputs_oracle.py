"""TEST INFRASTRUCTURE — CPU restatement of the per-token outputs of CLIP's towers (fp32, torch-CPU ops).

``CLIPVisionTransformer`` / ``CLIPTextTransformer`` with ``output_hidden_states`` and ``output_attentions`` under the
eager attention implementation (TF:modeling_clip.py:261-279, 477-507, 531-589, 667-691): ``last_hidden_state``,
``pooler_output``, the 13 ``hidden_states`` and the 12 ``attentions``.  Built on ``oracle.clip_oracle`` (layers,
masks) and ``hires_oracle`` (any image size); ``oracle/`` itself is not changed.  ``tests/golden/make_outputs_golden.py``
pins it against the live ``transformers.CLIPModel``.

``dt`` emulates the device's 16-bit operands as in ``oracle.clip_oracle``.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

import hires_oracle as HO
from oracle import clip_oracle as O
from oracle.weights import EOS, TEXT, VISION

# golden selection (tests/golden/outputs_golden.npz): layers and rows kept of each output
GOLDEN_HIDDEN_LAYERS = (0, 1, 12)
GOLDEN_ATTN_LAYERS = (0, 5, 11)
GOLDEN_CASES = {"vision_224": (2, 224), "vision_448": (1, 448)}  # name: (images, size)


def golden_rows(S: int, k: int) -> list:
    """The first k and last k token rows of a sequence of S."""
    return list(range(k)) + list(range(S - k, S))


def golden_text_inputs():
    """3 captions [3, 77]: two as the tokenizer emits them, the third with a padding mask that also has a hole."""
    from plip_b200.synthetic import token_ids
    ids, mask = token_ids(3, seed=77)
    mask = mask.clone()
    mask[2, 3] = 0
    return ids, mask


def attention_probs(x, sd, p: str, heads: int, mask: Optional[torch.Tensor], dt=None) -> torch.Tensor:
    """softmax(q k^T * dh^-0.5 + mask, fp32) of CLIPAttention's eager core (TF:261-279) on the layer input x (after
    layer_norm1): [B, heads, S, S]."""
    B, S, D = x.shape
    dh = D // heads
    q = O.linear(x, sd[f"{p}.q_proj.weight"], sd[f"{p}.q_proj.bias"], dt).view(B, S, heads, dh).transpose(1, 2)
    k = O.linear(x, sd[f"{p}.k_proj.weight"], sd[f"{p}.k_proj.bias"], dt).view(B, S, heads, dh).transpose(1, 2)
    att = (O._r(q, dt) @ O._r(k, dt).transpose(-1, -2)) * (dh ** -0.5)
    if mask is not None:
        att = att + mask
    return torch.softmax(att, dim=-1, dtype=torch.float32)


def _encoder(x, sd, prefix: str, heads: int, mask, dt):
    """CLIPEncoder.forward (TF:477-507) collecting hidden_states (13) and attentions (12)."""
    hidden, attns = [], []
    for i in range(12):
        hidden.append(x)
        p = f"{prefix}.encoder.layers.{i}"
        ln1 = O.layer_norm(x, sd[f"{p}.layer_norm1.weight"], sd[f"{p}.layer_norm1.bias"])
        attns.append(attention_probs(ln1, sd, f"{p}.self_attn", heads, mask, dt))
        x = O.encoder_layer(x, sd, p, heads, mask, dt)
    hidden.append(x)
    return x, hidden, attns


def vision_outputs(sd, pixel_values, dt=None, interpolate_pos_encoding: bool = False) -> Dict[str, object]:
    """CLIPVisionTransformer.forward (TF:667-691): last_hidden_state is the encoder output (before post_layernorm),
    pooler_output = post_layernorm(CLS row) [B, 768]; hidden_states[0] is the input after pre_layrnorm."""
    x = HO.vision_embeddings(sd, pixel_values, dt, interpolate_pos_encoding)
    x = O.layer_norm(x, sd["vision_model.pre_layrnorm.weight"], sd["vision_model.pre_layrnorm.bias"])
    x, hidden, attns = _encoder(x, sd, "vision_model", VISION["heads"], None, dt)
    pooled = O.layer_norm(x[:, 0, :], sd["vision_model.post_layernorm.weight"], sd["vision_model.post_layernorm.bias"])
    return {"last_hidden_state": x, "pooler_output": pooled, "hidden_states": hidden, "attentions": attns}


def text_outputs(sd, input_ids, attention_mask=None, dt=None, eos_token_id: int = EOS) -> Dict[str, object]:
    """CLIPTextTransformer.forward (TF:531-589): last_hidden_state = final_layer_norm of every row, pooler_output its
    row of the first eos [B, 512]; hidden_states[0] is token + position embeddings.  A row whose keys are all masked
    gets HF's uniform probabilities here (the engine writes zeros there)."""
    x = O.text_embeddings(sd, input_ids)
    mask = O.causal_mask(input_ids.shape[-1], attention_mask)
    x, hidden, attns = _encoder(x, sd, "text_model", TEXT["heads"], mask, dt)
    last = O.layer_norm(x, sd["text_model.final_layer_norm.weight"], sd["text_model.final_layer_norm.bias"])
    if eos_token_id == 2:
        pos = input_ids.to(torch.int).argmax(dim=-1)
    else:
        pos = (input_ids.to(torch.int) == eos_token_id).int().argmax(dim=-1)
    pooled = last[torch.arange(last.shape[0]), pos]
    return {"last_hidden_state": last, "pooler_output": pooled, "hidden_states": hidden, "attentions": attns}


def visible_keys(S: int, attention_mask: Optional[torch.Tensor], causal: bool, B: int) -> torch.Tensor:
    """[B, 1, S, S] bool: which keys a query row may attend to (the zeros of the engine's probabilities elsewhere)."""
    vis = torch.ones(B, 1, S, S, dtype=torch.bool)
    if causal:
        vis &= torch.ones(S, S, dtype=torch.bool).tril()[None, None]
    if attention_mask is not None:
        vis &= (attention_mask != 0)[:, None, None, :]
    return vis
