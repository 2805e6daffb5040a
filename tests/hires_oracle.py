"""TEST INFRASTRUCTURE — CPU restatement of CLIP's ``interpolate_pos_encoding`` path (fp32, torch-CPU ops).

Extends ``oracle.clip_oracle`` to images of any size: ``CLIPVisionEmbeddings.interpolate_pos_encoding`` and
``forward(..., interpolate_pos_encoding=True)`` (TF:modeling_clip.py:161-218), threaded through the vision transformer
and ``get_image_features`` (TF:670-676, 832-856).  With the flag off every function defers to ``oracle.clip_oracle``,
error included.  ``tests/golden/make_hires_golden.py`` pins it against the live ``transformers.CLIPModel``.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn.functional as F

from oracle import clip_oracle as O
from oracle.weights import VISION

HIRES_SIZES = [(256, 256), (448, 448), (320, 480), (266, 250), (1024, 1024)]  # golden image sizes (H, W)


def size_key(h: int, w: int) -> str:
    return f"{h}x{w}"


def interpolate_pos(pos: torch.Tensor, gh: int, gw: int) -> torch.Tensor:
    """TF:161-200: class row kept, rows 1..49 viewed as [768, 7, 7] and resized to [768, gh, gw] (bicubic,
    align_corners=False) -> [1 + gh * gw, 768].  HF skips the resize for a square 7 x 7 input; bicubic 7 -> 7 has the
    weights (0, 1, 0, 0), so resizing anyway gives the same table."""
    D = pos.shape[-1]
    g = int(round((pos.shape[0] - 1) ** 0.5))
    patch = pos[1:].reshape(1, g, g, D).permute(0, 3, 1, 2)
    patch = F.interpolate(patch, size=(gh, gw), mode="bicubic", align_corners=False)
    return torch.cat([pos[:1], patch.permute(0, 2, 3, 1).reshape(gh * gw, D)], dim=0)


def vision_embeddings(sd, pixel_values, dt=None, interpolate_pos_encoding: bool = False):
    """CLIPVisionEmbeddings.forward (TF:202-218) at any size: stride-32 patches (the H % 32 / W % 32 remainder is
    dropped, as by the conv), class row, interpolated position table."""
    if not interpolate_pos_encoding:
        return O.vision_embeddings(sd, pixel_values, dt)
    B, Cc, H, W = pixel_values.shape
    P = VISION["patch"]
    gh, gw = H // P, W // P
    w = sd["vision_model.embeddings.patch_embedding.weight"]
    D = w.shape[0]
    x = pixel_values[:, :, :gh * P, :gw * P]
    patches = x.reshape(B, Cc, gh, P, gw, P).permute(0, 2, 4, 1, 3, 5).reshape(B, gh * gw, Cc * P * P)
    pe = O.linear(patches, w.reshape(D, -1), None, dt)
    cls = sd["vision_model.embeddings.class_embedding"].expand(B, 1, D)
    emb = torch.cat([cls, pe], dim=1)
    pos = sd["vision_model.embeddings.position_embedding.weight"]
    if not (gh * gw == pos.shape[0] - 1 and H == W):  # TF:174-175
        pos = interpolate_pos(pos, gh, gw)
    return emb + pos[None]


def vision_transformer(sd, pixel_values, dt=None, hidden: Optional[List] = None, interpolate_pos_encoding: bool = False):
    """CLIPVisionTransformer.forward (TF:667-691) with ``interpolate_pos_encoding``.  Returns pooled [B,768]."""
    x = vision_embeddings(sd, pixel_values, dt, interpolate_pos_encoding)
    x = O.layer_norm(x, sd["vision_model.pre_layrnorm.weight"], sd["vision_model.pre_layrnorm.bias"])
    x = O.encoder(x, sd, "vision_model", VISION["heads"], VISION["layers"], None, dt, hidden)
    return O.layer_norm(x[:, 0, :], sd["vision_model.post_layernorm.weight"], sd["vision_model.post_layernorm.bias"])


def get_image_features(sd, pixel_values, dt=None, interpolate_pos_encoding: bool = False):
    """CLIPModel.get_image_features(..., interpolate_pos_encoding) (TF:829-863): [B,512], not normalised."""
    return O.linear(vision_transformer(sd, pixel_values, dt, None, interpolate_pos_encoding),
                    sd["visual_projection.weight"], None, dt)
