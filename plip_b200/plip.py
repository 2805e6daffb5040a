"""Drop-in for the reference's ``plip.PLIP`` class (``/root/reference/plip.py:11-117``).

Same constructor, attributes and method signatures; the HuggingFace ``CLIPModel`` forward it wrapped is
replaced by the CUDA engine.  Differences are confined to *how* the work is scheduled:

* images are turned into uint8 tiles on the host and normalised on the device (fused into the patch
  im2col kernel) instead of a float32 ``CLIPProcessor`` pass per batch (``plip.py:32-35``);
* ``batch_size`` keeps its meaning as the host-side chunk (and progress-bar tick, ``plip.py:46``), but
  chunks are merged into engine micro-batches and uploaded through the pipelined host path, instead of
  one synchronous H2D + D2H per batch (``plip.py:49-50``);
* the numpy similarity / argsort heads (``plip.py:73-87``) run on the device in fp32.
Results: float32 ``[N,512]`` numpy arrays, un-normalised, order-preserving — as the reference returns.
"""
from __future__ import annotations

import os
from typing import List, Optional, Union

import numpy as np
import PIL.Image
import torch
from tqdm import tqdm

from .modeling import PlipCLIPModel
from .tokenizer import find_tokenizer
from .preprocess import SIZE, chunks, decode_rgb, device_resizable, pack_rgb, to_uint8_tiles


class PLIP:

    def __init__(self, model_name, auth_token=None, *, model: Optional[PlipCLIPModel] = None, preprocess=None,
                 max_micro_batch: int = 1024, num_workers: int = 0, device_resize: bool = True, tokenizer=None):
        if not torch.cuda.is_available():
            raise RuntimeError("plip_b200.PLIP needs a CUDA device; there is no CPU fallback")
        self.device = "cuda"
        self.model_name = model_name
        self.max_micro_batch = max_micro_batch
        self.num_workers = int(num_workers)      # host threads for image decode / resize (0 = in-line)
        self.device_resize = bool(device_resize)  # images that are not 224x224: resize on the GPU (else PIL)
        if model is not None:
            self.model, self.preprocess, self.model_hash = model, preprocess, hash
        else:
            self.model, self.preprocess, self.model_hash = self._load_model(model_name, auth_token=auth_token)
        self.model = self.model.to(self.device)
        # string captions: the checkpoint's vocab.json + merges.txt (or $PLIP_B200_TOKENIZER) through the built-in BPE
        self.tokenizer = tokenizer if tokenizer is not None else find_tokenizer(
            model_name if isinstance(model_name, str) and os.path.isdir(model_name) else None)
        self.image_vectors = None  # the reference reads this in retrieval() without ever setting it

    @classmethod
    def from_state_dict(cls, state_dict, preprocess=None, model_name="state_dict", max_micro_batch: int = 1024,
                        tokenizer=None):
        """Build from an in-memory HF / OpenAI-clip state dict (no checkpoint directory needed)."""
        return cls(model_name, model=PlipCLIPModel(state_dict, max_micro_batch=max_micro_batch),
                   preprocess=preprocess, max_micro_batch=max_micro_batch, tokenizer=tokenizer)

    def _load_model(self, name: str, device: Union[str, torch.device] = "cuda", auth_token=None):
        model = PlipCLIPModel.from_pretrained(name, max_micro_batch=self.max_micro_batch, use_auth_token=auth_token)
        preprocessing = None
        try:  # tokenizer / processor: host-side plumbing, only needed for string captions
            from transformers import CLIPProcessor
            preprocessing = CLIPProcessor.from_pretrained(name, **({"token": auth_token} if auth_token else {}))
        except Exception:  # noqa: BLE001 - a checkpoint dir without tokenizer assets still encodes images / ids
            preprocessing = None
        tok = getattr(preprocessing, "tokenizer", None)
        if tok is not None and len(tok) < 49408:
            # without vocab.json / merges.txt transformers silently builds a 3-token tokenizer (SURVEY.md §8c)
            preprocessing = None
        return model, preprocessing, hash

    # ---- encoders ---------------------------------------------------------------------------------
    def encode_images(self, images: Union[List[str], List[PIL.Image.Image]], batch_size: int):
        """``plip.py:31-53``: list of paths / PIL images -> ``np.ndarray [N,512] float32`` (un-normalised)."""
        if len(images) == 0:
            raise ValueError("need at least one array to stack")  # np.stack([]) in the reference
        eng = self.model.engine
        flush = max(int(batch_size), eng.max_micro_batch)
        flush_bytes = 1 << 30            # decoded pixels held on the host (and uploaded at once) per flush
        out = np.empty((len(images), 512), dtype=np.float32)
        pending: List[np.ndarray] = []   # decoded RGB arrays, any size
        done = 0
        pbar = tqdm(total=len(images) // batch_size, position=0)

        def _tile_buffer(n: int) -> torch.Tensor:
            # ONE reusable (pinned, when a GPU exists) uint8 buffer for batches of 224x224 tiles: no np.stack
            # allocation per flush, and the upload inside plip_encode_images_host is a direct DMA (no staging copy)
            if getattr(self, "_pin", None) is None or self._pin.shape[0] < n:
                self._pin = torch.empty((max(n, flush), SIZE, SIZE, 3), dtype=torch.uint8)
                if torch.cuda.is_available():
                    self._pin = self._pin.pin_memory()
            return self._pin[:n]

        def _flush():
            nonlocal pending, done
            if not pending:
                return
            if all(a.shape == (SIZE, SIZE, 3) for a in pending):
                buf = _tile_buffer(len(pending))
                view = buf.numpy()
                for i, a in enumerate(pending):
                    view[i] = a
                res = eng.encode_images_host(buf).numpy()
            elif self.device_resize and all(device_resizable(a.shape[1], a.shape[0]) for a in pending):
                # upload the decoded images once; Pillow-exact bicubic resize + centre crop on the device
                buf, descs = pack_rgb(pending, crop="floor", pinned=True)
                tiles = eng.resize_crop(buf.to(eng.device, non_blocking=True), descs)
                res = eng.encode_images(tiles).cpu().numpy()
            else:  # PIL on the host (device_resize=False, or an image shrinks too much for the device kernel)
                res = eng.encode_images_host(to_uint8_tiles(pending, self.num_workers)).numpy()
            out[done:done + len(pending)] = res
            done += len(pending)
            pending = []

        for chunk in chunks(images, int(batch_size)):
            pending.extend(decode_rgb(chunk, self.num_workers))
            if len(pending) >= flush or sum(a.nbytes for a in pending) >= flush_bytes:
                _flush()
            pbar.update(1)
        _flush()
        pbar.close()
        return out

    def encode_region(self, region, crop_overlap: float = 0.1, non_bg_threshold: float = 0.5):
        """The crops the reference's slide preprocessing keeps (``random_crop`` with ``downsample = 1``,
        ``preprocess_DigestPath.py:36-108``), encoded: ``region`` is an RGB uint8 ``[H, W, 3]`` array, CPU / CUDA tensor
        or PIL image.  Returns ``(embeddings [k,512] float32 un-normalised, origins [k,2] int32 (row, col),
        tissue_ratio [k] float64)`` as numpy arrays, in the reference's crop order (``regions.encode_region``)."""
        from .regions import encode_region
        if isinstance(region, PIL.Image.Image):
            region = np.asarray(region.convert("RGB"))
        res = encode_region(self.model.engine, region, crop_overlap=crop_overlap, non_bg_threshold=non_bg_threshold)
        return res.embeddings.cpu().numpy(), res.origins, res.tissue_ratio

    def encode_region_pyramid(self, region, mask=None, downsample_list=(2, 4, 8, 16, 32), crop_overlap: float = 0.1,
                              non_bg_threshold: float = 0.5):
        """The reference's step 1 for one image (``random_crop`` at every ``downsample``,
        ``preprocess_DigestPath.py:117-140``), encoded: ``region`` as in :meth:`encode_region`; ``mask`` an L / RGB PIL
        image or a uint8 ``[H, W]`` / ``[H, W, 3]`` array (any size: it is resized per level with NEAREST, as there).
        Returns ``(embeddings [k,512] float32 un-normalised, stats)``, levels outer in list order; ``stats`` is a dict of
        numpy columns ``origin_row``, ``origin_col``, ``tissue_ratio``, ``tumor_to_patch_ratio``,
        ``tumor_to_tissue_ratio``, ``downsample``, ``cropsize``, ``crop_overlap``, ``non_bg_threshold`` in the
        reference's row order, so ``pandas.DataFrame(stats)`` has its ``df_stat`` columns
        (``regions.encode_region_pyramid``)."""
        from .regions import WINDOW, encode_region_pyramid
        if isinstance(region, PIL.Image.Image):
            region = np.asarray(region.convert("RGB"))
        if isinstance(mask, PIL.Image.Image):
            if mask.mode not in ("L", "RGB"):
                raise ValueError(f"a mask image must be mode L or RGB, got {mask.mode}")
            mask = np.asarray(mask)
        levels = encode_region_pyramid(self.model.engine, region, mask, downsample_list, crop_overlap,
                                       non_bg_threshold)
        emb = np.concatenate([lv.embeddings.cpu().numpy() for lv in levels]).reshape(-1, 512)
        col = lambda f: np.concatenate([f(lv) for lv in levels])  # noqa: E731
        n = lambda lv: len(lv.origins)  # noqa: E731
        stats = {"origin_row": col(lambda lv: lv.origins[:, 0]), "origin_col": col(lambda lv: lv.origins[:, 1]),
                 "tissue_ratio": col(lambda lv: lv.tissue_ratio),
                 "tumor_to_patch_ratio": col(lambda lv: lv.tumor_to_patch_ratio),
                 "tumor_to_tissue_ratio": col(lambda lv: lv.tumor_to_tissue_ratio),
                 "downsample": col(lambda lv: np.full(n(lv), lv.downsample)),
                 "cropsize": col(lambda lv: np.full(n(lv), WINDOW)),
                 "crop_overlap": col(lambda lv: np.full(n(lv), float(crop_overlap))),
                 "non_bg_threshold": col(lambda lv: np.full(n(lv), float(non_bg_threshold)))}
        return emb, stats

    def _tokenize(self, text: List[str]):
        if self.preprocess is None and self.tokenizer is None:
            raise RuntimeError("no tokenizer available for this checkpoint (no vocab.json + merges.txt next to it, "
                               "$PLIP_B200_TOKENIZER unset): pass token ids to encode_token_ids()")
        if self.tokenizer is not None:   # built-in byte-level BPE on the checkpoint's own vocabulary
            enc = self.tokenizer(list(text), return_tensors="pt", max_length=77, padding="max_length", truncation=True)
            return enc["input_ids"], enc["attention_mask"]
        enc = self.preprocess(text=list(text), return_tensors="pt", max_length=77, padding="max_length",
                              truncation=True)  # plip.py:57-58
        return enc["input_ids"], enc.get("attention_mask")

    def encode_text(self, text: List[str], batch_size: int):
        """``plip.py:55-71``: captions -> ``np.ndarray [N,512] float32`` (tokenised to 77 ids on the host)."""
        if len(text) == 0:
            raise ValueError("need at least one array to stack")
        ids, mask = self._tokenize(text)
        pbar = tqdm(total=len(text) // batch_size, position=0)
        out = self.encode_token_ids(ids, mask)
        pbar.update(len(text) // batch_size)
        pbar.close()
        return out

    def encode_token_ids(self, input_ids, attention_mask=None) -> np.ndarray:
        """Text tower on already-tokenised captions (``[N,<=77]`` int ids) — what ``get_text_features`` sees."""
        ids = torch.as_tensor(np.asarray(input_ids)) if not torch.is_tensor(input_ids) else input_ids
        if ids.dtype not in (torch.int32, torch.int64):
            ids = ids.to(torch.int64)
        mask = None
        if attention_mask is not None:
            mask = torch.as_tensor(np.asarray(attention_mask)) if not torch.is_tensor(attention_mask) else attention_mask
        return self.model.engine.encode_text_host(ids.cpu(), None if mask is None else mask.cpu()).numpy()

    # ---- similarity heads ---------------------------------------------------------------------------
    def _cosine_similarity(self, key_vectors: np.ndarray, space_vectors: np.ndarray, normalize=True):
        """``plip.py:73-76``: only the key side is normalised."""
        eng = self.model.engine
        k = torch.from_numpy(np.ascontiguousarray(key_vectors, dtype=np.float32))
        s = torch.from_numpy(np.ascontiguousarray(space_vectors, dtype=np.float32))
        sim = eng.similarity(k, s, scale=1.0, normalize_image=bool(normalize), normalize_text=False)
        return sim.cpu().numpy()

    def _nearest_neighbours(self, k, key_vectors, space_vectors, normalize=True, debug=False):
        """``plip.py:78-87``: indices of the k most similar space vectors, most similar first."""
        key_vectors = np.asarray(key_vectors, dtype=np.float32)
        space_vectors = np.asarray(space_vectors, dtype=np.float32)
        eng = self.model.engine
        kq = torch.from_numpy(np.ascontiguousarray(key_vectors))
        sp = torch.from_numpy(np.ascontiguousarray(space_vectors))
        k = int(min(k, space_vectors.shape[0]))
        if k <= 64:
            idx, _ = eng.similarity_topk(kq, sp, k, scale=1.0, normalize_query=bool(normalize), normalize_space=False)
            return idx.cpu().numpy().astype(np.int64)
        sim = eng.similarity(kq, sp, scale=1.0, normalize_image=bool(normalize), normalize_text=False)
        return torch.topk(sim, k, dim=-1).indices.cpu().numpy()

    def zero_shot_classification(self, images, text_labels: List[str], debug=False):
        """``plip.py:89-103``."""
        text_vectors = self.encode_text(text_labels, batch_size=8)
        image_vectors = self.encode_images(images, batch_size=8)
        cosine_sim = self._cosine_similarity(image_vectors, text_vectors)
        if debug:
            print(cosine_sim)
        preds = np.argmax(cosine_sim, axis=-1)
        return [text_labels[idx] for idx in preds]

    def retrieval(self, queries: List[str], top_k: int = 10):
        """``plip.py:105-114``: needs ``self.image_vectors`` (set it to a gallery of image embeddings first)."""
        if self.image_vectors is None:
            raise AttributeError("'PLIP' object has no attribute 'image_vectors' set: assign the gallery "
                                 "embeddings (e.g. plip.image_vectors = plip.encode_images(...)) before retrieval()")
        text_vectors = self.encode_text(queries, batch_size=8)
        return self._nearest_neighbours(k=top_k, key_vectors=text_vectors, space_vectors=self.image_vectors)
