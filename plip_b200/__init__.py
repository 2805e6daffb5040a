"""plip_b200 — H100-native PLIP (CLIP ViT-B/32) inference engine.

Python host code over a hand-written sm_90a CUDA library (``libplip_b200.so``, C ABI in
``include/plip_b200.h``).  Public surface mirrors the reference:

* :class:`plip_b200.plip.PLIP` — drop-in for ``plip.PLIP`` (encode_images / encode_text / zero-shot / retrieval)
* :class:`plip_b200.modeling.PlipCLIPModel` — ``CLIPModel``-style ``get_image_features`` / ``get_text_features`` /
  ``model(**inputs).logits_per_image`` and OpenAI-clip ``encode_image`` / ``encode_text``
* :class:`plip_b200.embedders.CLIPEmbedder` / ``EmbedderFactory`` — ``reproducibility/embedders``
* :class:`plip_b200.engine.Engine` — the raw engine handle; :mod:`plip_b200.distributed` — multi-GPU sharding
* :class:`plip_b200.tokenizer.ClipTokenizer` — CLIP byte-level BPE (HF ``vocab.json``/``merges.txt`` or OpenAI merge file)

Importing the package does not load the CUDA library; the first engine / packer call does and raises if it
is missing (there is no CPU fallback).
"""
__version__ = "0.1.0"

__all__ = ["PLIP", "PlipCLIPModel", "CLIPOutput", "CLIPEmbedder", "EmbedderFactory", "Engine", "ClipTokenizer"]


def __getattr__(name):
    if name == "PLIP":
        from .plip import PLIP
        return PLIP
    if name in ("PlipCLIPModel", "CLIPOutput"):
        from . import modeling
        return getattr(modeling, name)
    if name in ("CLIPEmbedder", "EmbedderFactory"):
        from . import embedders
        return getattr(embedders, name)
    if name == "Engine":
        from .engine import Engine
        return Engine
    if name == "ClipTokenizer":
        from .tokenizer import ClipTokenizer
        return ClipTokenizer
    raise AttributeError(name)
