"""The reference's MuDiPath baseline: torchvision DenseNet-121 features + global average pool on the device.

``reproducibility/embedders/mudipath.py`` builds ``NoHeadDenseNet`` (``forward = adaptive_avg_pool2d(features(x))``,
no final ReLU, no classifier) from the multi-task pathology checkpoint ``densenet121-mh-best-191205-141200.pth``, and
``DenseNetEmbedder.embed_images`` returns its un-normalised pooled features ``[N, 1024]``.  This module packs such a
state dict into the blob of ``plip_densenet_create`` (``include/plip_b200.h``) and wraps the handle.

Packing: every BatchNorm becomes ``y = x * scale + shift`` with the eval running statistics,
``scale = gamma / sqrt(running_var + 1e-5)`` and ``shift = beta - running_mean * scale``, computed in float64 and rounded
to float32 once.  Convolution weights are rounded to bfloat16 once, in the K order the kernels read (``(ky, kx, c)``
for the 7x7 stem and the 3x3 convolutions).
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Dict, Mapping, Optional, Union

import numpy as np
import torch

from ._lib import TensorInfo, check, lib

OUT_DIM = 1024
IMAGE_SIZE = 224
BN_EPS = 1e-5
CHECKPOINT_NAME = "densenet121-mh-best-191205-141200.pth"


def clean_state_dict(state_dict: Mapping, prefix: str, filter: Optional[Callable[[str], bool]] = None) -> Dict:
    """The reference's rule for the raw MuDiPath checkpoint (``mudipath.py:169``, ``clean_state_dict(sd,
    prefix="features.", filter=lambda k: not k.startswith("heads."))``): keep the keys ``filter`` accepts and strip
    ``prefix`` from those that carry it."""
    if filter is None:
        filter = lambda k: True  # noqa: E731
    return {(k[len(prefix):] if k.startswith(prefix) else k): v for k, v in state_dict.items() if filter(k)}


def fold_bn(weight, bias, running_mean, running_var, eps: float = BN_EPS):
    """Eval BatchNorm as ``(scale, shift)`` float32, folded in float64 and rounded once."""
    g, b, m, v = (torch.as_tensor(t).detach().to("cpu", torch.float64) for t in (weight, bias, running_mean, running_var))
    scale = g / torch.sqrt(v + eps)
    shift = b - m * scale
    return scale.to(torch.float32), shift.to(torch.float32)


def _tensor_table():
    L = lib()
    out = []
    for i in range(L.plip_densenet_num_tensors()):
        ti = TensorInfo()
        check(L.plip_densenet_tensor_info(i, C.byref(ti)), "plip_densenet_tensor_info")
        out.append((ti.name.decode(), int(ti.offset), int(ti.numel), int(ti.dtype), int(ti.rows), int(ti.cols)))
    return out


def _torchvision_names(state_dict: Mapping) -> Mapping:
    """Accept torchvision names (``features.conv0.weight`` ...) or a raw MuDiPath checkpoint, whose DenseNet sits
    under ``features.features.*`` next to its multi-task ``heads.*``: the latter goes through the reference's own
    cleaning rule first."""
    if any(k.startswith(("heads.", "features.features.")) for k in state_dict):
        return clean_state_dict(state_dict, prefix="features.", filter=lambda k: not k.startswith("heads."))
    return state_dict


def pack_state_dict(state_dict: Mapping) -> torch.Tensor:
    """torchvision DenseNet-121 state dict (``classifier.*`` and ``num_batches_tracked`` ignored) or a raw MuDiPath
    checkpoint -> the packed uint8 host blob.  A missing tensor raises ``KeyError`` naming it."""
    sd = _torchvision_names(state_dict)

    def get(name):
        if name not in sd:
            raise KeyError(f"DenseNet-121 state dict has no {name!r}")
        return torch.as_tensor(sd[name]).detach().to("cpu")

    blob = torch.zeros(int(lib().plip_densenet_blob_bytes()), dtype=torch.uint8)
    bn_cache = {}
    for name, off, numel, dtype, rows, cols in _tensor_table():
        if name.endswith(".scale") or name.endswith(".shift"):
            bn = name.rsplit(".", 1)[0]
            if bn not in bn_cache:
                bn_cache[bn] = fold_bn(get(bn + ".weight"), get(bn + ".bias"), get(bn + ".running_mean"),
                                       get(bn + ".running_var"))
            t = bn_cache[bn][0 if name.endswith(".scale") else 1]
        else:
            w = get(name).to(torch.float32)
            if w.dim() != 4 or w.shape[0] != rows:
                raise ValueError(f"{name}: expected {rows} output channels, got shape {tuple(w.shape)}")
            w = w.permute(0, 2, 3, 1).reshape(rows, -1)           # K order (ky, kx, c)
            if w.shape[1] > cols:
                raise ValueError(f"{name}: {w.shape[1]} inputs per output, the kernels take {cols}")
            t = torch.zeros(rows, cols, dtype=torch.float32)
            t[:, :w.shape[1]] = w
            t = t.to(torch.bfloat16)
        if t.numel() != numel:
            raise ValueError(f"{name}: {t.numel()} elements, expected {numel}")
        raw = t.contiguous().view(torch.uint8).reshape(-1)
        blob[off:off + raw.numel()] = raw
    return blob


class DenseNetEngine:
    """One DenseNet-121 handle on one CUDA device: packed weights + activations for ``max_micro_batch`` images."""

    def __init__(self, state_dict: Mapping, device: Union[int, str, torch.device, None] = None,
                 max_micro_batch: int = 256):
        if not torch.cuda.is_available():
            raise RuntimeError("plip_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self._L = lib()
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError(f"plip_b200 runs on CUDA devices only, got {dev}")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        blob = pack_state_dict(state_dict)
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            torch.cuda.init()
            check(self._L.plip_densenet_create(blob.data_ptr(), blob.numel(), self.device.index, int(max_micro_batch),
                                               C.byref(h)), "plip_densenet_create")
        self._h = h
        self.max_micro_batch = int(max_micro_batch)

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._L.plip_densenet_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _check_tiles(tiles) -> None:
        if tiles.dtype not in (torch.uint8, np.dtype("uint8")) or tuple(tiles.shape[1:]) != (IMAGE_SIZE, IMAGE_SIZE, 3) \
                or len(tiles.shape) != 4:
            raise ValueError(f"tiles must be uint8 [n,224,224,3] (NHWC), got {tiles.dtype} {tuple(tiles.shape)}")

    @torch.no_grad()
    def encode_images(self, tiles: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """uint8 ``[n,224,224,3]`` tiles -> float32 ``[n,1024]`` pooled features, on the device, on the current
        stream (``NoHeadDenseNet(x).squeeze()`` with ``x`` = ToTensor + Normalize of the tiles, but always 2-D)."""
        self._check_tiles(tiles)
        if tiles.device != self.device:
            tiles = tiles.to(self.device, non_blocking=True)
        tiles = tiles.contiguous()
        n = int(tiles.shape[0])
        if out is None:
            out = torch.empty(n, OUT_DIM, dtype=torch.float32, device=self.device)
        elif out.shape != (n, OUT_DIM) or out.dtype != torch.float32 or out.device != self.device \
                or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous float32 [{n},{OUT_DIM}] tensor on {self.device}")
        with torch.cuda.device(self.device):
            check(self._L.plip_densenet_encode(self._h, tiles.data_ptr(), n, out.data_ptr(),
                                               torch.cuda.current_stream(self.device).cuda_stream),
                  "plip_densenet_encode")
        return out

    def resize_crop(self, src: torch.Tensor, descs: np.ndarray, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Packed RGB uint8 images on the device + host descriptors (``preprocess.pack_rgb(..., crop="round")``) ->
        uint8 tiles ``[n,224,224,3]``: Pillow-exact bilinear resize and crop (``plip_resize_crop_bilinear_u8``), i.e.
        torchvision's ``Resize(224)`` + ``CenterCrop(224)`` on the device, on the current stream."""
        from .preprocess import RESIZE_DESC_DTYPE
        if not (src.is_cuda and src.dtype == torch.uint8 and src.is_contiguous() and src.dim() == 1):
            raise ValueError("src must be a contiguous 1-D uint8 CUDA tensor (preprocess.pack_rgb)")
        descs = np.ascontiguousarray(descs, dtype=RESIZE_DESC_DTYPE)
        n = int(descs.shape[0])
        if out is None:
            out = torch.empty((n, IMAGE_SIZE, IMAGE_SIZE, 3), device=src.device, dtype=torch.uint8)
        elif not (out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous()
                  and out.numel() == n * IMAGE_SIZE * IMAGE_SIZE * 3):
            raise ValueError(f"out must be a contiguous uint8 [{n},224,224,3] CUDA tensor")
        if n:
            with torch.cuda.device(src.device):
                check(self._L.plip_resize_crop_bilinear_u8(src.data_ptr(), int(src.numel()), descs.ctypes.data, n,
                                                           out.data_ptr(),
                                                           torch.cuda.current_stream(src.device).cuda_stream),
                      "plip_resize_crop_bilinear_u8")
        return out

    @torch.no_grad()
    def encode_images_host(self, tiles: Union[np.ndarray, torch.Tensor]) -> np.ndarray:
        """Host uint8 ``[n,224,224,3]`` -> numpy float32 ``[n,1024]``: uploaded and encoded one micro-batch at a
        time, so device memory stays bounded by the micro-batch whatever ``n`` is."""
        self._check_tiles(tiles)
        t = torch.from_numpy(np.ascontiguousarray(tiles)) if isinstance(tiles, np.ndarray) else tiles.contiguous()
        n = int(t.shape[0])
        res = np.empty((n, OUT_DIM), dtype=np.float32)
        for i in range(0, n, self.max_micro_batch):
            d = t[i:i + self.max_micro_batch].to(self.device)
            res[i:i + d.shape[0]] = self.encode_images(d).cpu().numpy()
        return res
