"""TEST INFRASTRUCTURE — CPU restatement of the CLIP ViT-B/16 vision tower (fp32, torch-CPU ops).

ViT-B/16 is ViT-B/32 with a 16-pixel patch: the conv patch embedding is ``[768, 3, 16, 16]`` and the stored position
table ``[197, 768]`` (a 14 x 14 grid).  Everything here takes the patch size from the weights' shapes, as
``CLIPVisionEmbeddings`` does from its config (TF:modeling_clip.py:138-218), and reuses ``oracle.clip_oracle`` for the
encoder, ``hires_oracle.interpolate_pos`` for the bicubic position table and ``outputs_oracle`` for the per-layer
outputs.  ``tests/golden/make_vitb16_golden.py`` pins it against the live ``transformers.CLIPModel`` with
``patch_size=16``.

Also here: the bit-exact patch-16 im2col and the per-element position-table reference of a 14 x 14 source grid, the
device kernels' contracts restated from ``helper_oracle``'s patch-32 / 7 x 7 ones.
"""
from __future__ import annotations

from fractions import Fraction
from functools import lru_cache
from typing import Dict, List, Optional

import numpy as np
import torch

import helper_oracle as H
import hires_oracle as HO
import outputs_oracle as OO
from oracle import clip_oracle as O
from oracle.weights import VISION

PATCH = 16
GRID = 14                                   # the stored table's grid: 224 / 16
SEQ = GRID * GRID + 1                       # 197 tokens at 224 x 224
SIZES = [(224, 224), (320, 448), (512, 512)]  # golden image sizes (H, W); 512 x 512 is the largest grid, 1025 tokens


def size_key(h: int, w: int) -> str:
    return f"{h}x{w}"


def patch_of(sd) -> int:
    return int(sd["vision_model.embeddings.patch_embedding.weight"].shape[-1])


def vision_embeddings(sd, pixel_values, dt=None, interpolate_pos_encoding: bool = False):
    """CLIPVisionEmbeddings.forward (TF:202-218) at the weights' patch size P: stride-P patches (the H % P / W % P
    remainder is dropped, as by the conv), class row, the stored position table when the grid is the stored one and
    the image square (TF:174-175), else the bicubic one."""
    B, Cc, H, W = pixel_values.shape
    if not interpolate_pos_encoding and (H != VISION["image"] or W != VISION["image"]):
        raise ValueError(f"Input image size ({H}*{W}) doesn't match model (224*224).")  # TF:204-207
    w = sd["vision_model.embeddings.patch_embedding.weight"]
    D, P = w.shape[0], w.shape[-1]
    gh, gw = H // P, W // P
    x = pixel_values[:, :, :gh * P, :gw * P]
    patches = x.reshape(B, Cc, gh, P, gw, P).permute(0, 2, 4, 1, 3, 5).reshape(B, gh * gw, Cc * P * P)
    pe = O.linear(patches, w.reshape(D, -1), None, dt)
    cls = sd["vision_model.embeddings.class_embedding"].expand(B, 1, D)
    emb = torch.cat([cls, pe], dim=1)
    pos = sd["vision_model.embeddings.position_embedding.weight"]
    if not (gh * gw == pos.shape[0] - 1 and H == W):
        pos = HO.interpolate_pos(pos, gh, gw)
    return emb + pos[None]


def vision_transformer(sd, pixel_values, dt=None, hidden: Optional[List] = None, interpolate_pos_encoding: bool = False):
    """CLIPVisionTransformer.forward (TF:667-691).  Returns pooled [B,768]."""
    x = vision_embeddings(sd, pixel_values, dt, interpolate_pos_encoding)
    x = O.layer_norm(x, sd["vision_model.pre_layrnorm.weight"], sd["vision_model.pre_layrnorm.bias"])
    x = O.encoder(x, sd, "vision_model", VISION["heads"], VISION["layers"], None, dt, hidden)
    return O.layer_norm(x[:, 0, :], sd["vision_model.post_layernorm.weight"], sd["vision_model.post_layernorm.bias"])


def get_image_features(sd, pixel_values, dt=None, interpolate_pos_encoding: bool = False):
    """CLIPModel.get_image_features (TF:829-863): [B,512], not normalised."""
    return O.linear(vision_transformer(sd, pixel_values, dt, None, interpolate_pos_encoding),
                    sd["visual_projection.weight"], None, dt)


def vision_outputs(sd, pixel_values, dt=None, interpolate_pos_encoding: bool = False) -> Dict[str, object]:
    """``outputs_oracle.vision_outputs`` at the weights' patch size: last_hidden_state, pooler_output, the 13
    hidden_states and the 12 attentions [B, 12, S, S]."""
    x = vision_embeddings(sd, pixel_values, dt, interpolate_pos_encoding)
    x = O.layer_norm(x, sd["vision_model.pre_layrnorm.weight"], sd["vision_model.pre_layrnorm.bias"])
    x, hidden, attns = OO._encoder(x, sd, "vision_model", VISION["heads"], None, dt)
    pooled = O.layer_norm(x[:, 0, :], sd["vision_model.post_layernorm.weight"], sd["vision_model.post_layernorm.bias"])
    return {"last_hidden_state": x, "pooler_output": pooled, "hidden_states": hidden, "attentions": attns}


# ---- device kernel contracts ---------------------------------------------------------------------------------------
def im2col_ref(pixels, fmt, dt, patch: int = PATCH):
    """What im2col_kernel<fmt, *, patch> writes, bit for bit (helper_oracle.im2col_ref at any patch size): row
    b * gh * gw + py * gw + px, column c * patch^2 + ky * patch + kx from pixel (py * patch + ky, px * patch + kx);
    f32 the RNE cast, bf16 a copy (re-rounded through fp32 for fp16), u8 helper_oracle.u8_table then the cast."""
    if fmt == 2:
        n, Hh, W, _ = pixels.shape
        vals = H.u8_table().to(pixels.device)
        chw = pixels.permute(0, 3, 1, 2).long()
        x = torch.stack([vals[c][chw[:, c]] for c in range(3)], 1)
    else:
        n, _, Hh, W = pixels.shape
        x = pixels.float()
    gh, gw = Hh // patch, W // patch
    x = x[:, :, :gh * patch, :gw * patch].reshape(n, 3, gh, patch, gw, patch).permute(0, 2, 4, 1, 3, 5)
    return x.reshape(n * gh * gw, 3 * patch * patch).to(dt)


@lru_cache(maxsize=None)
def cubic_taps32(src: int, g: int, i: int):
    """helper_oracle.cubic_taps32 for a src x src stored grid: scale = fl(src / g), taps clamped to [0, src - 1], every
    operation the fp32 rounding the sm_90a build performs."""
    scale = H._round32(Fraction(src) / Fraction(g))
    real = H._fma32(float(i) + 0.5, scale, -0.5)
    fl = float(np.floor(real))
    t = H._add32(real, -fl)
    t1, t2, t3 = H._add32(t, 1.0), H._add32(1.0, -t), H._add32(2.0, -t)

    def outer(s):
        return H._fma32(s, H._fma32(s, H._fma32(s, -0.75, 3.75), -6.0), 3.0)

    def inner(s):
        return H._fma32(s, H._mul32(s, H._fma32(s, 1.25, -2.25)), 1.0)

    return tuple(min(max(int(fl) - 1 + k, 0), src - 1) for k in range(4)), (outer(t1), inner(t), inner(t2), outer(t3))


def pos_interp_ref(pos, gh: int, gw: int):
    """helper_oracle.pos_interp_ref for a stored table of any square grid (14 x 14 for ViT-B/16): the float64 table
    from the kernel's fp32 weights and the per-element slack gamma(8) sum_a |wy_a| sum_b |wx_b| |p[iy_a, ix_b]|."""
    D = pos.shape[-1]
    src = int(round((pos.shape[0] - 1) ** 0.5))
    p = pos[1:].double().reshape(src, src, D)

    def matrix(g):
        M = torch.zeros(g, src, dtype=torch.float64)
        Ma = torch.zeros_like(M)
        for i in range(g):
            taps, w = cubic_taps32(src, g, i)
            for k in range(4):
                M[i, taps[k]] += w[k]
                Ma[i, taps[k]] += abs(w[k])
        return M, Ma

    My, May = matrix(gh)
    Mx, Max = matrix(gw)
    ref = torch.einsum("ya,xb,abd->yxd", My, Mx, p).reshape(gh * gw, D)
    slack = H.gamma(8) * torch.einsum("ya,xb,abd->yxd", May, Max, p.abs()).reshape(gh * gw, D)
    ref = torch.cat([pos[:1].double(), ref], 0)
    slack = torch.cat([torch.zeros(1, D, dtype=torch.float64), slack], 0) * (1 + 2.0 ** -20)
    return ref, slack
