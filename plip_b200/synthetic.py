"""Seeded synthetic CLIP ViT-B/32 (and ViT-B/16) weights and inputs (the BASELINE.json configs' data).

No pretrained PLIP checkpoint is reachable offline (``vinid/plip`` needs the network; SURVEY.md §8c), so the
benchmark, the smoke test and the parity tests all run on seeded random weights with the exact state-dict names /
shapes of ``transformers.CLIPModel(CLIPConfig())`` (SURVEY.md §8a), and on seeded synthetic tiles / token ids
(SURVEY.md §8d).  This module is plain data generation (torch CPU generators: bit-reproducible for a given torch
version); ``oracle.weights`` / ``oracle.synth`` re-export it for the tests.

Weights come in two flavours:

* ``mode="hf_init"`` follows the distributions of ``CLIPPreTrainedModel._init_weights``
  (TF:modeling_clip.py:402-459): zero biases, unit LayerNorm gains.
* ``mode="rich"`` additionally draws non-zero biases and non-trivial LayerNorm gain/shift so that every bias /
  affine code path of the kernels is exercised (strictly stronger test).
* ``mode="outlier"`` is "rich" reshaped to stress the numerics the way a *trained* CLIP ViT-B/32 does
  (massive-activation channels in the residual stream, non-zero per-token means, LayerNorm gains spread over
  two orders of magnitude): see :func:`_add_outliers`.  Used by the parity tests of the LayerNorm-folded GEMMs.
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np
import torch

VISION = dict(dim=768, heads=12, ff=3072, layers=12, seq=50, patch=32, image=224)
TEXT = dict(dim=512, heads=8, ff=2048, layers=12, seq=77, vocab=49408)
PROJ = 512
LOGIT_SCALE_INIT = 2.6592  # TF:configuration_clip.py:160-161
BOS, EOS = 49406, 49407


def _tower(sd, g, prefix: str, dim: int, ff: int, layers: int, rich: bool) -> None:
    def randn(*shape, std):
        return torch.randn(*shape, generator=g) * std

    in_proj_std = dim ** -0.5 * (2 * layers) ** -0.5
    out_proj_std = dim ** -0.5
    fc_std = (2 * dim) ** -0.5
    b_std = 0.02 if rich else 0.0
    for i in range(layers):
        p = f"{prefix}.encoder.layers.{i}"
        for name in ("k_proj", "v_proj", "q_proj"):  # HF parameter order inside CLIPAttention
            sd[f"{p}.self_attn.{name}.weight"] = randn(dim, dim, std=in_proj_std)
            sd[f"{p}.self_attn.{name}.bias"] = randn(dim, std=b_std)
        sd[f"{p}.self_attn.out_proj.weight"] = randn(dim, dim, std=out_proj_std)
        sd[f"{p}.self_attn.out_proj.bias"] = randn(dim, std=b_std)
        sd[f"{p}.layer_norm1.weight"] = 1.0 + randn(dim, std=0.1 if rich else 0.0)
        sd[f"{p}.layer_norm1.bias"] = randn(dim, std=0.05 if rich else 0.0)
        sd[f"{p}.mlp.fc1.weight"] = randn(ff, dim, std=fc_std)
        sd[f"{p}.mlp.fc1.bias"] = randn(ff, std=b_std)
        sd[f"{p}.mlp.fc2.weight"] = randn(dim, ff, std=in_proj_std)
        sd[f"{p}.mlp.fc2.bias"] = randn(dim, std=b_std)
        sd[f"{p}.layer_norm2.weight"] = 1.0 + randn(dim, std=0.1 if rich else 0.0)
        sd[f"{p}.layer_norm2.bias"] = randn(dim, std=0.05 if rich else 0.0)


def _add_outliers(sd, g, prefix: str, dim: int, layers: int) -> None:
    """Reshape a "rich" tower so that its residual stream looks like a trained CLIP's:

    * two "massive activation" channels switched on by the MLP of layer 1 (constant part through ``fc2.bias``,
      token-dependent part through 20x larger ``fc2.weight`` rows) and a third one in layer 3 — |x| of 60...300
      against a typical |x| of ~1, persisting through every later layer of the residual stream;
    * a common shift of all channels (``out_proj.bias`` of layer 0): per-token mean ~1.5 standard deviations;
    * LayerNorm gains from 0.05 (on the massive channels, as trained models learn) to ~10 on a few others, and a
      few shifts of +-2."""
    ch = [int(c) for c in torch.randperm(dim, generator=g)[:3]]
    sd[f"{prefix}.encoder.layers.0.self_attn.out_proj.bias"] += 1.5
    fc2b, fc2w = f"{prefix}.encoder.layers.1.mlp.fc2.bias", f"{prefix}.encoder.layers.1.mlp.fc2.weight"
    sd[fc2b][ch[0]] += 120.0
    sd[fc2b][ch[1]] -= 60.0
    sd[fc2w][ch[0]] *= 20.0
    sd[fc2w][ch[1]] *= 20.0
    sd[f"{prefix}.encoder.layers.3.mlp.fc2.bias"][ch[2]] += 250.0
    for i in range(layers):
        for ln in ("layer_norm1", "layer_norm2"):
            w, b = sd[f"{prefix}.encoder.layers.{i}.{ln}.weight"], sd[f"{prefix}.encoder.layers.{i}.{ln}.bias"]
            w[ch] = 0.05
            big = torch.randperm(dim, generator=g)[:8]
            w[big] = 4.0 + 6.0 * torch.rand(8, generator=g)
            sh = torch.randperm(dim, generator=g)[:4]
            b[sh] = torch.tensor([2.0, -2.0, 1.0, -1.0])


def make_state_dict(seed: int = 0, mode: str = "rich", patch: int = 32) -> "OrderedDict[str, torch.Tensor]":
    """fp32 state dict with the HF ``CLIPModel`` key set (``load_state_dict(strict=True)``-able).  ``patch``: the
    vision patch size, 32 (ViT-B/32; ``CLIPConfig()``) or 16 (ViT-B/16: ``patch_embedding.weight`` ``[768,3,16,16]``,
    a ``[197,768]`` position table).  The ViT-B/32 draws are those of the generator before the argument existed."""
    assert mode in ("rich", "hf_init", "outlier")
    assert patch in (32, 16)
    vseq = (VISION["image"] // patch) ** 2 + 1
    rich = mode != "hf_init"
    g = torch.Generator(device="cpu").manual_seed(seed)

    def randn(*shape, std):
        return torch.randn(*shape, generator=g) * std

    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    sd["logit_scale"] = torch.tensor(LOGIT_SCALE_INIT)
    # ---- text tower (TF:modeling_clip.py:221-258, 510-589)
    td = TEXT["dim"]
    sd["text_model.embeddings.token_embedding.weight"] = randn(TEXT["vocab"], td, std=0.02)
    sd["text_model.embeddings.position_embedding.weight"] = randn(TEXT["seq"], td, std=0.02)
    _tower(sd, g, "text_model", td, TEXT["ff"], TEXT["layers"], rich)
    sd["text_model.final_layer_norm.weight"] = 1.0 + randn(td, std=0.1 if rich else 0.0)
    sd["text_model.final_layer_norm.bias"] = randn(td, std=0.05 if rich else 0.0)
    # ---- vision tower (TF:modeling_clip.py:138-218, 647-691)
    vd = VISION["dim"]
    sd["vision_model.embeddings.class_embedding"] = randn(vd, std=vd ** -0.5)
    sd["vision_model.embeddings.patch_embedding.weight"] = randn(vd, 3, patch, patch, std=0.02)
    sd["vision_model.embeddings.position_embedding.weight"] = randn(vseq, vd, std=0.02)
    sd["vision_model.pre_layrnorm.weight"] = 1.0 + randn(vd, std=0.1 if rich else 0.0)
    sd["vision_model.pre_layrnorm.bias"] = randn(vd, std=0.05 if rich else 0.0)
    _tower(sd, g, "vision_model", vd, VISION["ff"], VISION["layers"], rich)
    sd["vision_model.post_layernorm.weight"] = 1.0 + randn(vd, std=0.1 if rich else 0.0)
    sd["vision_model.post_layernorm.bias"] = randn(vd, std=0.05 if rich else 0.0)
    # ---- projections (TF:modeling_clip.py:784-786)
    sd["visual_projection.weight"] = randn(PROJ, vd, std=vd ** -0.5)
    sd["text_projection.weight"] = randn(PROJ, td, std=td ** -0.5)
    if mode == "outlier":
        go = torch.Generator(device="cpu").manual_seed(seed + 7919)
        _add_outliers(sd, go, "vision_model", vd, VISION["layers"])
        _add_outliers(sd, go, "text_model", td, TEXT["layers"])
        for ln in ("vision_model.post_layernorm", "text_model.final_layer_norm"):
            sd[ln + ".weight"][torch.randperm(sd[ln + ".weight"].numel(), generator=go)[:8]] = 5.0
    return sd


# ---- synthetic inputs ----------------------------------------------------------------------------


def tiles_u8(n: int, seed: int = 0) -> np.ndarray:
    """cfg1: n synthetic 224x224 RGB tiles, uint8 [n,224,224,3]."""
    return np.random.default_rng(seed).integers(0, 256, (n, 224, 224, 3), dtype=np.uint8)


def pixel_values(n: int, seed: int = 1234) -> torch.Tensor:
    """cfg2: normalised pixels (U[0,1) - mean) / std, fp32 [n,3,224,224]."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, 224, 224, generator=g)
    mean = torch.tensor((0.48145466, 0.4578275, 0.40821073)).view(1, 3, 1, 1)
    std = torch.tensor((0.26862954, 0.26130258, 0.27577711)).view(1, 3, 1, 1)
    return (x - mean) / std


def pixel_values_hw(n: int, h: int, w: int, seed: int = 4321) -> torch.Tensor:
    """Normalised pixels of any size (``interpolate_pos_encoding`` inputs): fp32 [n,3,h,w], drawn like
    :func:`pixel_values`."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, h, w, generator=g)
    mean = torch.tensor((0.48145466, 0.4578275, 0.40821073)).view(1, 3, 1, 1)
    std = torch.tensor((0.26862954, 0.26130258, 0.27577711)).view(1, 3, 1, 1)
    return (x - mean) / std


def token_ids(n: int, seed: int = 1235, full_length: bool = False, min_len: int = 8):
    """cfg3: random caption ids [n,77] int64 with bos at 0, first eos at len-1, eos padding after it
    (what the CLIP tokenizer emits), plus the matching attention_mask (1 up to and incl. the eos)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, BOS, (n, 77), generator=g)
    if full_length:
        lens = torch.full((n,), 77)
    else:
        lens = torch.randint(min_len, 78, (n,), generator=g)
    ids[:, 0] = BOS
    ar = torch.arange(77)[None]
    ids = torch.where(ar >= (lens[:, None] - 1), torch.full_like(ids, EOS), ids)
    mask = (ar < lens[:, None]).to(torch.int64)
    return ids, mask


# The 19 tissue types of PanNuke's types.npy.
PANNUKE_TISSUES = ("Adrenal_gland", "Bile-duct", "Bladder", "Breast", "Cervix", "Colon", "Esophagus", "HeadNeck",
                   "Kidney", "Liver", "Lung", "Ovarian", "Pancreatic", "Prostate", "Skin", "Stomach", "Testis",
                   "Thyroid", "Uterus")


def _pannuke_counts(rng: np.random.Generator, n: int) -> list:
    """Per image, the nucleus instances of channels 0..4 and what the rest of the mask does: the labelling rule's
    edge cases first (in a fixed rotation), then random draws."""
    cases = [
        dict(counts=(0, 0, 0, 0, 0)),                          # no cells: dropped
        dict(counts=(10, 5, 5, 7, 5)),                         # n0 = 10, 10 / 33 > 0.3 (with channel 5's id)
        dict(counts=(10, 5, 5, 8, 5)),                         # n0 = 10, 10 / 34 < 0.3
        dict(counts=(9, 2, 0, 0, 0)),                          # n0 = 9: neither malignant nor benign
        dict(counts=(0, 4, 3, 0, 2)),                          # benign
        dict(counts=(12, 3, 0, 0, 0), big_ids=True),           # float ids past 255 (they wrap in the uint8 cast)
        dict(counts=(0, 3, 2, 0, 0), no_zero=1),               # channel 1 has no zero anywhere
        dict(counts=(15, 0, 0, 2, 0), background=False),       # channel 5 all zero
        dict(counts=(0, 0, 0, 0, 0), background=False, no_zero=5),  # background only: dropped
    ]
    out = [cases[i] if i < len(cases) else None for i in range(n)]
    for i in range(len(cases), n):
        kind = rng.integers(0, 3)
        n0 = (0, int(rng.integers(1, 10)), int(rng.integers(10, 20)))[kind]
        out[i] = dict(counts=(n0, *(int(x) for x in rng.integers(0, 8, size=4))), big_ids=bool(rng.integers(0, 4) == 0),
                      background=bool(rng.integers(0, 5) != 0))
    return out


def make_pannuke_folds(seed: int = 0, sizes=(20, 16, 12), size: int = 256, dtype=np.float64):
    """Seeded synthetic PanNuke folds: a list of ``(images [n, size, size, 3], masks [n, size, size, 6], types [n])``
    as ``np.load`` returns PanNuke's ``images.npy`` / ``masks.npy`` / ``types.npy`` (float64 arrays, ``<U`` types).

    Every mask channel 0..4 holds a drawn number of nucleus instances as disks of distinct ids, each in its own cell
    of a 6 x 6 grid while the cells last (so the edge cases' counts are exact); channel 5 is 1 where no nucleus is (the background channel) or all
    zero.  The first images of each fold are the labelling rule's edge cases (no cells, ``n0 = 10`` at ratios just
    above and below 0.3, ``n0 = 9``, ids past 255, a channel without a zero, channel 5 empty); every one of the 19
    tissue strings occurs.  ``dtype``: of the image and mask arrays (``np.uint8`` for large runs)."""
    rng = np.random.default_rng(seed)
    grid = 6
    cell = size // grid
    yy, xx = np.mgrid[0:cell, 0:cell]
    folds = []
    tissue_at = 0
    for n in sizes:
        images = np.empty((n, size, size, 3), dtype=dtype)
        masks = np.zeros((n, size, size, 6), dtype=dtype)
        types = []
        for i, spec in enumerate(_pannuke_counts(rng, n)):
            base = rng.integers(120, 230, size=3)
            img = base + rng.integers(-25, 26, size=(size, size, 3))
            slots = rng.permutation(grid * grid)
            s = 0
            for ch, cnt in enumerate(spec["counts"]):
                ids = rng.choice(np.arange(1, 600 if spec.get("big_ids") else 250), size=cnt, replace=False)
                for inst in ids:
                    cy, cx = divmod(int(slots[s % (grid * grid)]), grid)
                    s += 1
                    r = int(rng.integers(3, cell // 2))
                    disk = (yy - cell // 2) ** 2 + (xx - cell // 2) ** 2 <= r * r
                    tile = masks[i, cy * cell:(cy + 1) * cell, cx * cell:(cx + 1) * cell, ch]
                    tile[disk] = inst
                    img[cy * cell:(cy + 1) * cell, cx * cell:(cx + 1) * cell][disk] -= 60 + 20 * ch
            if "no_zero" in spec:
                ch = spec["no_zero"]
                masks[i, ..., ch][masks[i, ..., ch] == 0] = 7
            if spec.get("background", True):
                masks[i, ..., 5] = np.all(masks[i, ..., :5] == 0, axis=-1)
            images[i] = np.clip(img, 0, 255)
            # every tissue once, then mostly the first four, so that some (tissue, label) subsets split
            types.append(PANNUKE_TISSUES[tissue_at] if tissue_at < len(PANNUKE_TISSUES) else
                         PANNUKE_TISSUES[int(rng.integers(0, 4))])
            tissue_at += 1
        folds.append((images, masks, np.array(types)))
    return folds
