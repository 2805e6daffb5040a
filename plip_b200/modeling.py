"""Drop-in for the ``transformers.CLIPModel`` call surface used by the reference.

``PlipCLIPModel`` keeps the three entry points the reference touches —
``get_image_features`` (reference ``plip.py:50``), ``get_text_features`` (``plip.py:68``) and
``model(**inputs).logits_per_image`` (``README.md:45-49``; TF:modeling_clip.py:867-944) — and the OpenAI-clip
``encode_image`` / ``encode_text`` used by ``reproducibility/embedders/plip.py:48,66``.  All compute runs in the
CUDA engine; outputs are torch tensors on the engine's device, like the HF model's.

Return types follow what the reference code expects (transformers v4 semantics): ``get_*_features`` return
the ``[n,512]`` tensor itself — the reference calls ``.detach().cpu().numpy()`` on it directly.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Mapping, Optional, Tuple, Union

import torch

from .engine import Engine
from .weights import PATCH_SIZES


@dataclass
class BaseModelOutputWithPooling:
    """``transformers.modeling_outputs.BaseModelOutputWithPooling``: what ``vision_model`` / ``text_model`` return.
    ``keys()`` lists the fields that are set, in HF's order."""

    last_hidden_state: torch.Tensor
    pooler_output: torch.Tensor
    hidden_states: Optional[Tuple[torch.Tensor, ...]] = None
    attentions: Optional[Tuple[torch.Tensor, ...]] = None

    def __getitem__(self, k):
        return getattr(self, k)

    def keys(self):
        return tuple(k for k in ("last_hidden_state", "pooler_output", "hidden_states", "attentions")
                     if getattr(self, k) is not None)


@dataclass
class CLIPOutput:
    """Fields of ``transformers.models.clip.modeling_clip.CLIPOutput`` (TF:104-135) that the engine produces.
    ``text_model_output`` / ``vision_model_output`` are set only by a forward with ``output_hidden_states`` or
    ``output_attentions``, and listed by ``keys()`` only then."""

    logits_per_image: torch.Tensor
    logits_per_text: torch.Tensor
    text_embeds: torch.Tensor
    image_embeds: torch.Tensor
    loss: Optional[torch.Tensor] = None
    text_model_output: Optional[BaseModelOutputWithPooling] = None
    vision_model_output: Optional[BaseModelOutputWithPooling] = None

    def __getitem__(self, k):
        return getattr(self, k)

    def keys(self):
        return ("logits_per_image", "logits_per_text", "text_embeds", "image_embeds") + tuple(
            k for k in ("text_model_output", "vision_model_output") if getattr(self, k) is not None)


def _model_output(o) -> BaseModelOutputWithPooling:
    return BaseModelOutputWithPooling(last_hidden_state=o["last_hidden_state"], pooler_output=o["pooler_output"],
                                      hidden_states=o["hidden_states"], attentions=o["attentions"])


def check_config(cfg) -> None:
    """``ValueError`` unless a ``CLIPConfig`` has a geometry the kernels run: every field they hard-code (common.cuh
    model constants; TF:configuration_clip.py:47-64,97-109), the vision patch size 32 (ViT-B/32, PLIP's architecture)
    or 16 (ViT-B/16)."""
    v, t = cfg.vision_config, cfg.text_config
    want = {"vision hidden_size": (v.hidden_size, 768),
            "vision patch_size": (v.patch_size, v.patch_size if v.patch_size in PATCH_SIZES else PATCH_SIZES),
            "vision image_size": (v.image_size, 224), "vision num_hidden_layers": (v.num_hidden_layers, 12),
            "vision num_attention_heads": (v.num_attention_heads, 12), "vision intermediate_size": (v.intermediate_size, 3072),
            "vision hidden_act": (v.hidden_act, "quick_gelu"), "vision layer_norm_eps": (float(v.layer_norm_eps), 1e-5),
            "text hidden_size": (t.hidden_size, 512), "text num_hidden_layers": (t.num_hidden_layers, 12),
            "text num_attention_heads": (t.num_attention_heads, 8), "text intermediate_size": (t.intermediate_size, 2048),
            "text hidden_act": (t.hidden_act, "quick_gelu"), "text layer_norm_eps": (float(t.layer_norm_eps), 1e-5),
            "text max_position_embeddings": (t.max_position_embeddings, 77), "text vocab_size": (t.vocab_size, 49408),
            "projection_dim": (cfg.projection_dim, 512)}
    bad = {k: got for k, (got, exp) in want.items() if got != exp}
    if bad:
        raise ValueError("plip_b200 implements the CLIP ViT-B/32 and ViT-B/16 geometries only (PLIP's architecture, "
                         f"and the same towers behind a 16-pixel patch); this checkpoint differs in {bad}")


class PlipCLIPModel:
    """CUDA-engine-backed stand-in for ``CLIPModel``: the CLIP ViT-B/32 geometry PLIP ships, or ViT-B/16 (the same
    towers behind a 16-pixel patch), as the weights say."""

    def __init__(self, state_dict: Mapping[str, torch.Tensor], device: Union[int, str, torch.device, None] = None,
                 max_micro_batch: int = 1024, operand_dtype="bf16"):
        self.engine = Engine(state_dict, device=device, max_micro_batch=max_micro_batch, operand_dtype=operand_dtype)
        self.device = self.engine.device
        self.training = False

    # ---- construction -------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, name_or_path: str, device=None, max_micro_batch: int = 1024, operand_dtype="bf16",
                        **hf_kwargs):
        """Read a HuggingFace CLIP checkpoint (e.g. ``vinid/plip`` or a local directory) on the host and pack
        it for the engine.  ``transformers`` is only the checkpoint *reader* here; its forward never runs.
        ``use_auth_token`` (reference ``plip.py:26``) is translated to ``token`` for transformers >= 5."""
        from transformers import CLIPModel  # host-side weight loading only

        tok = hf_kwargs.pop("use_auth_token", None)
        if tok is not None:
            hf_kwargs.setdefault("token", tok)
        hf = CLIPModel.from_pretrained(name_or_path, **hf_kwargs)
        check_config(hf.config)
        m = cls(hf.state_dict(), device=device, max_micro_batch=max_micro_batch, operand_dtype=operand_dtype)
        # legacy configs (eos_token_id == 2) pool at argmax(input_ids) (TF:564-570); same row whenever an eos exists
        m.engine.set_text_pooling(getattr(hf.config.text_config, "eos_token_id", 49407) == 2)
        return m

    @classmethod
    def from_openai_state_dict(cls, state_dict, device=None, max_micro_batch: int = 1024, operand_dtype="bf16"):
        """``clip.load(arch)`` + ``load_state_dict(torch.load(path))`` (``embedders/factory.py:20-27``).  The patch size
        (ViT-B/32 or ViT-B/16) is read from ``visual.conv1.weight``, as ``clip.model.build_model`` does."""
        m = cls(state_dict, device=device, max_micro_batch=max_micro_batch, operand_dtype=operand_dtype)
        m.engine.set_text_pooling(True)          # OpenAI clip: x[arange, text.argmax(-1)] (eot has the largest id)
        return m

    # ---- nn.Module-ish no-ops the reference calls -------------------------------------------------
    def to(self, *args, **kwargs):
        return self

    def eval(self):
        return self

    def float(self):
        return self

    @property
    def logit_scale_exp(self) -> float:
        return self.engine.logit_scale_exp

    # ---- HF surface ---------------------------------------------------------------------------
    def get_image_features(self, pixel_values: torch.Tensor = None, interpolate_pos_encoding: bool = False,
                           **_ignored) -> torch.Tensor:
        """TF:829-863 — vision tower + visual_projection, un-normalised ``[n,512]`` float32.
        ``interpolate_pos_encoding=True`` accepts other image sizes (TF:161-218; ``Engine.encode_images``)."""
        if pixel_values is None:
            raise ValueError("You have to specify pixel_values")
        return self.engine.encode_images(pixel_values, interpolate_pos_encoding=interpolate_pos_encoding)

    def get_text_features(self, input_ids: torch.Tensor = None, attention_mask: Optional[torch.Tensor] = None,
                          **_ignored) -> torch.Tensor:
        """TF:793-825 — text tower + text_projection, un-normalised ``[n,512]`` float32."""
        if input_ids is None:
            raise ValueError("You have to specify input_ids")  # TF:540-541
        return self.engine.encode_text(input_ids, attention_mask)

    def vision_model(self, pixel_values: torch.Tensor = None, output_hidden_states: bool = False,
                     output_attentions: bool = False, interpolate_pos_encoding: bool = False) -> BaseModelOutputWithPooling:
        """``CLIPModel.vision_model(...)`` (TF:667-691): ``last_hidden_state`` ``[n,S,768]`` (before post_layernorm),
        ``pooler_output`` ``[n,768]`` (post_layernorm of the CLS row, not projected), and with the flags the 13
        ``hidden_states`` and 12 ``attentions`` ``[n,12,S,S]`` (eager-attention values), all from one tower pass."""
        if pixel_values is None:
            raise ValueError("You have to specify pixel_values")  # TF:670-671
        return _model_output(self.engine.vision_outputs(pixel_values, bool(output_hidden_states), bool(output_attentions),
                                                        interpolate_pos_encoding))

    def text_model(self, input_ids: torch.Tensor = None, attention_mask: Optional[torch.Tensor] = None,
                   output_hidden_states: bool = False, output_attentions: bool = False) -> BaseModelOutputWithPooling:
        """``CLIPModel.text_model(...)`` (TF:531-589): ``last_hidden_state`` ``[n,S,512]`` (after final_layer_norm),
        ``pooler_output`` ``[n,512]`` (its pooled row, not projected), and with the flags the 13 ``hidden_states`` and
        12 ``attentions`` ``[n,8,S,S]`` (eager-attention values; a row with no visible key is all zeros)."""
        if input_ids is None:
            raise ValueError("You have to specify input_ids")  # TF:540-541
        return _model_output(self.engine.text_outputs(input_ids, attention_mask, bool(output_hidden_states),
                                                      bool(output_attentions)))

    def forward(self, input_ids: torch.Tensor = None, pixel_values: torch.Tensor = None,
                attention_mask: Optional[torch.Tensor] = None, return_loss: Optional[bool] = None,
                interpolate_pos_encoding: bool = False, output_hidden_states: Optional[bool] = None,
                output_attentions: Optional[bool] = None, **_ignored) -> CLIPOutput:
        """TF:867-944 — both towers, L2-normalise, ``exp(logit_scale) * I . T^T``.  With ``output_hidden_states`` or
        ``output_attentions`` each tower runs once through ``vision_model`` / ``text_model``'s path, which also fills
        ``vision_model_output`` / ``text_model_output``; the embeddings and logits are the same either way."""
        if input_ids is None:
            raise ValueError("You have to specify input_ids")
        if pixel_values is None:
            raise ValueError("You have to specify pixel_values")
        ipe = interpolate_pos_encoding
        vout = tout = None
        if output_hidden_states or output_attentions:
            ohs, oa = bool(output_hidden_states), bool(output_attentions)
            vo = self.engine.vision_outputs(pixel_values, ohs, oa, ipe, normalize=True)
            to = self.engine.text_outputs(input_ids, attention_mask, ohs, oa, normalize=True)
            img, txt = vo.pop("embeds"), to.pop("embeds")
            vout, tout = _model_output(vo), _model_output(to)
        elif not pixel_values.is_cuda:
            # host inputs (an extension: HF would raise on a device mismatch): the pixel upload runs on the engine's
            # copy stream while the text tower computes, so ~3 ms of PCIe time per 1024 uint8 tiles stay hidden
            # ... and batches larger than one micro-batch are uploaded micro-batch by micro-batch, each one computed as
            # soon as it has landed while the next one travels
            mb = self.engine.max_micro_batch
            parts = [self.engine.upload_async(pixel_values[i:i + mb]) for i in range(0, pixel_values.shape[0], mb)]
            txt = self.engine.encode_text(input_ids, attention_mask, normalize=True)
            embs = []
            for chunk, uploaded in parts:
                torch.cuda.current_stream(self.device).wait_event(uploaded)
                embs.append(self.engine.encode_images(chunk, normalize=True, interpolate_pos_encoding=ipe))
            img = embs[0] if len(embs) == 1 else torch.cat(embs, dim=0)
        elif not ipe:
            # both towers side by side (one call each where that does not apply, see Engine.encode_pair)
            img, txt = self.engine.encode_pair(pixel_values, input_ids, attention_mask, normalize=True)
        else:
            img = self.engine.encode_images(pixel_values, normalize=True, interpolate_pos_encoding=ipe)
            txt = self.engine.encode_text(input_ids, attention_mask, normalize=True)
        lpi = self.engine.similarity(img, txt, normalize_image=False, normalize_text=False)
        loss = None
        if return_loss:  # clip_loss (TF:68-76): symmetric cross entropy; tiny, done with torch on the logits
            lpt = lpi.t()
            tgt = torch.arange(lpt.shape[0], device=lpt.device)
            loss = (torch.nn.functional.cross_entropy(lpt, tgt) + torch.nn.functional.cross_entropy(lpt.t(), tgt)) / 2
        return CLIPOutput(logits_per_image=lpi, logits_per_text=lpi.t(), text_embeds=txt, image_embeds=img, loss=loss,
                          text_model_output=tout, vision_model_output=vout)

    __call__ = forward

    # ---- OpenAI-clip surface (reproducibility/embedders/plip.py:48,66) ---------------------------------
    def encode_image(self, images: torch.Tensor) -> torch.Tensor:
        return self.engine.encode_images(images)

    def encode_text(self, idx: torch.Tensor) -> torch.Tensor:
        return self.engine.encode_text(idx)
