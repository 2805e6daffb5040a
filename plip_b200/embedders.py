"""Drop-in for ``reproducibility/embedders`` (``plip.py`` ``CLIPEmbedder``, ``factory.py``, ``abst.py``).

``CLIPEmbedder`` keeps the reference's constructor ``(model, preprocess, name, backbone)`` and its four methods
(``image_embedder``, ``text_embedder``, ``embed_images``, ``embed_text``; ``embedders/plip.py:11-75``) and returns
**L2-normalised** float32 numpy embeddings like the reference does (``:53,:73``).  ``model`` is any object with
the OpenAI-clip surface ``encode_image`` / ``encode_text`` returning torch tensors — here a
:class:`plip_b200.modeling.PlipCLIPModel` — so the reference's evaluation scripts run unchanged on top of it.
The ``.npy`` embedding cache of the reference (``utils/cacher.py``) is a disk cache orthogonal to compute and is
out of scope: ``image_embedder`` / ``text_embedder`` always compute.
"""
from __future__ import annotations

import os
from abc import ABC, abstractmethod
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from .modeling import PlipCLIPModel
from .tokenizer import find_tokenizer
from .preprocess import decode_native_then_rgb, SIZE, chunks, decode_rgb, device_resizable, pack_rgb, to_uint8_tiles
from .preprocess import to_uint8_tiles_bilinear


class AbstractEmbedder(ABC):
    """``reproducibility/embedders/abst.py:3-11``."""

    @abstractmethod
    def image_embedder(self, list_of_images, device="cuda", num_workers=1, batch_size=32, additional_cache_name=""):
        ...

    @abstractmethod
    def text_embedder(self, list_of_labels, device="cuda", num_workers=1, batch_size=32, additional_cache_name=""):
        ...


def _default_tokenize(*asset_dirs) -> Optional[Callable]:
    """``clip.tokenize(captions, truncate=True)`` (``embedders/plip.py:65``): the OpenAI package when installed,
    else the built-in BPE on merge-table assets found next to the checkpoint or via ``$PLIP_B200_TOKENIZER``."""
    try:
        import clip  # OpenAI clip package (not installed in this image; SURVEY.md §8c)
        return lambda captions: clip.tokenize(captions, truncate=True)
    except Exception:  # noqa: BLE001
        pass
    tok = find_tokenizer(*asset_dirs)
    if tok is None:
        return None
    return lambda captions: torch.from_numpy(tok.tokenize(list(captions), truncate=True))


class CLIPEmbedder(AbstractEmbedder):

    def __init__(self, model, preprocess, name, backbone, tokenize: Optional[Callable] = None):
        self.model = model
        self.preprocess = preprocess  # kept for API parity; tiles are prepared by plip_b200.preprocess
        self.name = name
        self.backbone = backbone
        self.tokenize = tokenize or _default_tokenize(
            os.path.dirname(backbone) if isinstance(backbone, str) and backbone else None)

    def image_embedder(self, list_of_images, device="cuda", num_workers=1, batch_size=32, additional_cache_name=""):
        return self.embed_images(list_of_images, device=device, num_workers=num_workers, batch_size=batch_size)

    def text_embedder(self, list_of_labels, device="cuda", num_workers=1, batch_size=32, additional_cache_name=""):
        return self.embed_text(list_of_labels, device=device, num_workers=num_workers, batch_size=batch_size)

    def embed_images(self, list_of_images: Sequence, device="cuda", num_workers=1, batch_size=32) -> np.ndarray:
        """``embedders/plip.py:37-54``: paths / PIL images -> normalised ``[N,512]`` float32."""
        outs: List[torch.Tensor] = []
        eng = getattr(self.model, "engine", None)
        for chunk in chunks(list(list_of_images), max(int(batch_size), 256)):
            # torchvision's CenterCrop rounding (transform.py:45-52), not CLIPImageProcessor's floor
            if eng is not None:
                arrays = decode_native_then_rgb(chunk, int(num_workers), crop="round")  # non-RGB modes: PIL, native mode
                if all(a.shape == (SIZE, SIZE, 3) for a in arrays):
                    outs.append(eng.encode_images_host(np.stack(arrays, axis=0), normalize=True))
                elif not all(device_resizable(a.shape[1], a.shape[0]) for a in arrays):  # too large: PIL
                    outs.append(eng.encode_images_host(to_uint8_tiles(arrays, int(num_workers), crop="round"),
                                                       normalize=True))
                else:  # Pillow-exact bicubic resize + crop on the device
                    buf, descs = pack_rgb(arrays, crop="round", pinned=True)
                    tiles = eng.resize_crop(buf.to(eng.device, non_blocking=True), descs)
                    outs.append(eng.encode_images(tiles, normalize=True).cpu())
            else:  # any OpenAI-clip-like model
                tiles = to_uint8_tiles(chunk, int(num_workers), crop="round")
                t = torch.from_numpy(tiles).to(device)
                e = self.model.encode_image(t).detach().float().cpu()
                outs.append(e / e.norm(dim=1, keepdim=True))
        return torch.cat(outs, dim=0).numpy()

    def embed_text(self, list_of_labels: Sequence, device="cuda", num_workers=1, batch_size=32) -> np.ndarray:
        """``embedders/plip.py:56-75``: captions (or pre-tokenised id rows) -> normalised ``[N,512]`` float32."""
        labels = list(list_of_labels)
        if len(labels) and not isinstance(labels[0], str):
            idx = torch.as_tensor(np.asarray(labels))
        else:
            if self.tokenize is None:
                raise RuntimeError("no tokenizer available (the `clip` package is not installed and no merge table was "
                                   "found next to the checkpoint or in $PLIP_B200_TOKENIZER): pass a `tokenize` "
                                   "callable or pre-tokenised id rows")
            idx = self.tokenize(labels)
        outs = []
        for chunk in chunks(idx, max(int(batch_size), 1024)):
            e = self.model.encode_text(chunk.to(device)).detach().float()
            outs.append((e / e.norm(dim=1, keepdim=True)).cpu())
        return torch.cat(outs, dim=0).numpy()


class DenseNetEmbedder:
    """``reproducibility/embedders/mudipath.py:187-215``: the MuDiPath DenseNet-121 baseline.  ``model`` is a
    :class:`plip_b200.densenet.DenseNetEngine`.  ``embed_images`` returns the **un-normalised** pooled features as
    float32 numpy ``[N,1024]``.

    Deliberate differences from the reference: the result is always ``[N,1024]`` (the reference's ``.squeeze()``
    turns a final batch of one image into ``[1024]`` and its ``np.concatenate`` then raises); there is no
    ``text_embedder``, as in the reference; the ``.npy`` cache is out of scope, as for :class:`CLIPEmbedder`."""

    def __init__(self, model, preprocess, name, backbone):
        self.model = model
        self.preprocess = preprocess  # kept for API parity; tiles are prepared by plip_b200.preprocess
        self.name = name
        self.backbone = backbone

    def image_embedder(self, list_of_images, device="cuda", num_workers=1, batch_size=32, additional_cache_name=""):
        return self.embed_images(list_of_images, device=device, num_workers=num_workers, batch_size=batch_size)

    def embed_images(self, list_of_images: Sequence, device="cuda", num_workers=1, batch_size=32) -> np.ndarray:
        """Paths / PIL images / RGB arrays -> ``[N,1024]`` float32.  Images are converted to RGB first, as the
        reference's ``CLIPImageDataset`` does, then routed as ``CLIPEmbedder.embed_images`` routes them: a chunk of
        224 x 224 images goes straight to the engine, a chunk the device resize takes gets ``Resize(224)`` (bilinear) +
        ``CenterCrop(224)`` on the device (``plip_resize_crop_bilinear_u8``), and a chunk with an image too large
        for it is resized with PIL on host threads.  Both resize routes give the same tiles, bit for bit."""
        images = list(list_of_images)
        eng = self.model
        outs = [np.empty((0, 1024), dtype=np.float32)]
        for chunk in chunks(images, max(int(batch_size), eng.max_micro_batch)):
            arrays = decode_rgb(chunk, int(num_workers))
            if all(a.shape == (SIZE, SIZE, 3) for a in arrays):
                outs.append(eng.encode_images_host(np.stack(arrays, axis=0)))
            elif not all(device_resizable(a.shape[1], a.shape[0]) for a in arrays):   # too large: PIL
                outs.append(eng.encode_images_host(to_uint8_tiles_bilinear(arrays, int(num_workers))))
            else:
                buf, descs = pack_rgb(arrays, crop="round", pinned=True)
                tiles = eng.resize_crop(buf.to(eng.device, non_blocking=True), descs)
                outs.append(eng.encode_images(tiles).cpu().numpy())
        return np.concatenate(outs, axis=0)


def mudipath_checkpoint() -> str:
    """Path of ``densenet121-mh-best-191205-141200.pth``.  ``$PLIP_B200_MTDP``, when set, is the only place looked at
    (the file, or a directory holding it): a value that resolves to nothing raises instead of falling through to
    another checkpoint.  Otherwise the directory the reference's ``load_dox_url`` downloads to: ``$TORCH_MODEL_ZOO``,
    else ``$TORCH_HOME/models`` (``~/.torch/models``).  Nothing is downloaded."""
    from .densenet import CHECKPOINT_NAME
    env = os.environ.get("PLIP_B200_MTDP")
    if env:
        path = os.path.join(env, CHECKPOINT_NAME) if os.path.isdir(env) else env
        if not os.path.isfile(path):
            raise FileNotFoundError(f"$PLIP_B200_MTDP={env!r} names no file (looked at {path}); point it at "
                                    f"{CHECKPOINT_NAME} or at a directory holding it")
        return path
    torch_home = os.path.expanduser(os.environ.get("TORCH_HOME", "~/.torch"))
    path = os.path.join(os.environ.get("TORCH_MODEL_ZOO", os.path.join(torch_home, "models")), CHECKPOINT_NAME)
    if os.path.isfile(path):
        return path
    raise FileNotFoundError(
        f"embedder 'mudipath' needs the MuDiPath DenseNet-121 checkpoint {CHECKPOINT_NAME} (the reference downloads "
        "it from dox.uliege.be; plip_b200 never downloads): point $PLIP_B200_MTDP at the file, or put it into "
        f"$TORCH_MODEL_ZOO (default $TORCH_HOME/models, ~/.torch/models).  Looked at: {path}")


class EmbedderFactory:
    """``reproducibility/embedders/factory.py:15-47``: ``args.model_name`` selects the flavour.  For ``plip`` / ``clip``
    ``args.backbone`` is the path of an OpenAI-clip (or HF) state dict saved with ``torch.save``; for ``mudipath`` it
    is only a name kept on the embedder, as in the reference, and the weights come from :func:`mudipath_checkpoint`."""

    def factory(self, args):
        name, path = args.model_name, args.backbone
        if name == "mudipath":  # build_densenet(pretrained="mtdp") + Resize/CenterCrop/Normalize (factory.py:34-47)
            from .densenet import DenseNetEngine
            # The reference hands this file straight to clean_state_dict(...).items() and then to a strict
            # load_state_dict, so it is a mapping of tensors: the tensors-only unpickler (weights_only) is enough and
            # runs no code from the file.
            sd = torch.load(mudipath_checkpoint(), map_location="cpu", weights_only=True)
            return DenseNetEmbedder(DenseNetEngine(sd), None, name, path)
        arch = os.environ.get("PC_CLIP_ARCH", "ViT-B/32")
        if arch != "ViT-B/32":
            raise ValueError(f"plip_b200 implements ViT-B/32 only (PC_CLIP_ARCH={arch!r})")
        if name == "plip":      # clip.load(arch) + load_state_dict(torch.load(path))     (factory.py:20-27)
            sd = torch.load(path, map_location="cpu")
            if isinstance(sd, dict) and "state_dict" in sd:
                sd = sd["state_dict"]
            model = PlipCLIPModel.from_openai_state_dict(sd) if "visual.conv1.weight" in sd else PlipCLIPModel(sd)
            model.eval()
            return CLIPEmbedder(model, None, name, path)
        if name == "clip":      # the PRETRAINED OpenAI weights; `path` is only a cache key there (factory.py:29-32)
            model = PlipCLIPModel.from_openai_state_dict(self._openai_pretrained_state_dict(arch))
            model.eval()
            return CLIPEmbedder(model, None, name, path)
        raise ValueError(f"unsupported embedder {name!r} (plip / clip / mudipath)")

    @staticmethod
    def _openai_pretrained_state_dict(arch: str):
        """``clip.load(arch)``'s weights without running its model: through the ``clip`` package when it is
        installed, else from its download cache (``~/.cache/clip/ViT-B-32.pt``, a TorchScript archive) or
        ``$PLIP_B200_OPENAI_CLIP``.  Never falls back to ``args.backbone``: that is the PLIP checkpoint."""
        try:
            import clip                                   # noqa: PLC0415 - optional, as in the reference
            model, _ = clip.load(arch, device="cpu")
            return model.state_dict()
        except ImportError:
            pass
        cands = [os.environ.get("PLIP_B200_OPENAI_CLIP"), os.path.expanduser("~/.cache/clip/ViT-B-32.pt")]
        for c in cands:
            if c and os.path.isfile(c):
                try:
                    return torch.jit.load(c, map_location="cpu").state_dict()
                except RuntimeError:
                    sd = torch.load(c, map_location="cpu")
                    return sd["state_dict"] if isinstance(sd, dict) and "state_dict" in sd else sd
        raise FileNotFoundError(
            "embedder 'clip' needs OpenAI's pretrained ViT-B/32 weights: install the `clip` package, or put "
            "ViT-B-32.pt into ~/.cache/clip/ (or point $PLIP_B200_OPENAI_CLIP at it).  args.backbone is NOT used for "
            "this branch (reproducibility/embedders/factory.py:29-32 never loads it).")
