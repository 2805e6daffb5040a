"""Image preparation: PIL / path -> 224x224 RGB uint8 tiles, on the host (PIL) or on the device.

The arithmetic part of ``CLIPImageProcessor`` (rescale 1/255, normalise by the CLIP mean/std;
TF:models/clip/image_processing_clip.py:50-62, ``reproducibility/embedders/transform.py:45-52``) is fused
into the device im2col kernel (``PLIP_PIX_U8_NHWC``), so the host only has to deliver uint8 tiles:
shortest-edge-224 bicubic resize + centre crop for images that are not already 224x224, which is what
the reference's processor does with PIL before its float conversion.

Two routes produce those tiles, bit-identically: ``to_uint8_tiles`` (PIL on host threads) and
``to_uint8_tiles_device`` (decoded RGB arrays are packed, uploaded once and resized + cropped by the
``plip_resize_crop_u8`` kernel, which restates Pillow's fixed-point bicubic exactly).
"""
from __future__ import annotations

from typing import Iterable, List, Sequence, Union

import numpy as np
import PIL.Image

SIZE = 224
ImageLike = Union[str, PIL.Image.Image, np.ndarray]


def load_rgb(img: ImageLike) -> PIL.Image.Image:
    """Path / PIL image / HxWx3 uint8 array -> RGB PIL image (``Image().decode_example`` + convert_rgb)."""
    if isinstance(img, str):
        img = PIL.Image.open(img)
    elif isinstance(img, np.ndarray):
        img = PIL.Image.fromarray(img)
    if img.mode != "RGB":
        img = img.convert("RGB")
    return img


def resize_plan(w: int, h: int, size: int = SIZE, crop: str = "floor"):
    """``(new_w, new_h, left, top)`` of shortest-edge-``size`` resize + centre crop.

    ``crop="floor"``: offsets ``(dim - size) // 2`` (CLIPImageProcessor.center_crop, what ``plip.py:35`` runs);
    ``crop="round"``: ``int(round((dim - size) / 2.0))`` (torchvision ``CenterCrop``,
    ``reproducibility/embedders/transform.py:47``) — they differ when the excess is odd."""
    short, long = (w, h) if w <= h else (h, w)
    new_long = int(size * long / short)
    nw, nh = (size, new_long) if w <= h else (new_long, size)
    if crop == "floor":
        left, top = (nw - size) // 2, (nh - size) // 2
    elif crop == "round":
        left, top = int(round((nw - size) / 2.0)), int(round((nh - size) / 2.0))
    else:
        raise ValueError(f"crop must be 'floor' or 'round', got {crop!r}")
    return nw, nh, left, top


def resize_center_crop(img: PIL.Image.Image, size: int = SIZE, crop: str = "floor") -> PIL.Image.Image:
    """Shortest edge -> ``size`` (bicubic, aspect preserved, long edge ``int(size * long / short)``),
    then centre crop ``size x size`` (see :func:`resize_plan` for the two offset conventions)."""
    w, h = img.size
    if (w, h) == (size, size):
        return img
    nw, nh, left, top = resize_plan(w, h, size, crop)
    if (nw, nh) != (w, h):
        img = img.resize((nw, nh), resample=PIL.Image.BICUBIC)
    return img.crop((left, top, left + size, top + size))


# numpy twin of ``plip_resize_desc_t`` (include/plip_b200.h)
RESIZE_DESC_DTYPE = np.dtype([("offset", "<i8"), ("width", "<i4"), ("height", "<i4"), ("new_width", "<i4"),
                              ("new_height", "<i4"), ("left", "<i4"), ("top", "<i4")])


def device_resizable(w: int, h: int, size: int = SIZE) -> bool:
    """Whether ``plip_resize_crop_u8`` takes a ``w x h`` image: its filter banks (224 horizontal + 32 vertical rows of
    ``2*ceil(2*scale)+1`` taps, padded to 4) plus one output row's strip of source rows must fit 200 KB of shared
    memory — shortest edges up to ~6,000 px at ordinary aspect ratios.  Larger images go through PIL."""
    import math
    nw, nh, _, _ = resize_plan(w, h, size)
    if min(w, h) < 1 or max(w, h) > 65536 or max(nw, nh) > 65536:
        return False

    def taps4(i, o):
        return (2 * math.ceil(2.0 * max(i / o, 1.0)) + 1 + 3) // 4 * 4

    vs = h / nh
    tables = (size * taps4(w, nw) + 32 * taps4(h, nh) + 2 * (size + 32)) * 4
    strip_rows = min(h, math.ceil(4.0 * max(vs, 1.0)) + 3) + 3
    return tables + strip_rows * size * 3 <= 200 * 1024


def pack_rgb(arrays: Sequence[np.ndarray], crop: str = "floor", pinned: bool = False):
    """Concatenate ``[h,w,3] uint8`` arrays into one byte buffer + their resize descriptors.

    Returns ``(buffer uint8 torch tensor [total], descs np.ndarray[RESIZE_DESC_DTYPE])``; image offsets are
    rounded up to 16 bytes."""
    import torch
    descs = np.zeros(len(arrays), dtype=RESIZE_DESC_DTYPE)
    off = 0
    for i, a in enumerate(arrays):
        if a.ndim != 3 or a.shape[2] != 3 or a.dtype != np.uint8:
            raise ValueError(f"image {i}: expected an [h,w,3] uint8 array, got {a.dtype} {a.shape}")
        h, w = int(a.shape[0]), int(a.shape[1])
        nw, nh, left, top = resize_plan(w, h, SIZE, crop)
        descs[i] = (off, w, h, nw, nh, left, top)
        off += (h * w * 3 + 15) // 16 * 16
    buf = torch.empty(off, dtype=torch.uint8, pin_memory=pinned)
    view = buf.numpy()
    for d, a in zip(descs, arrays):
        n = int(d["width"]) * int(d["height"]) * 3
        view[int(d["offset"]):int(d["offset"]) + n] = np.ascontiguousarray(a).reshape(-1)
    return buf, descs


def decode_rgb(images: Sequence[ImageLike], workers: int = 0) -> List[np.ndarray]:
    """Paths / PIL images / arrays -> list of ``[h,w,3] uint8`` arrays (decode only, no resize)."""
    if workers > 1 and len(images) > 1:
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=workers) as ex:
            return list(ex.map(lambda im: np.asarray(load_rgb(im)), images))
    return [np.asarray(load_rgb(im)) for im in images]


def decode_native_then_rgb(images: Sequence[ImageLike], workers: int = 0, crop: str = "round") -> List[np.ndarray]:
    """Decode for the OpenAI-clip ``_transform`` order (``reproducibility/embedders/transform.py:45-52``: Resize ->
    CenterCrop -> convert("RGB")): images that are already RGB come back as decoded arrays of any size (the caller
    resizes them, on the device or with PIL — same result); images in ANY OTHER MODE (P / 1 / L / LA / RGBA / I;16 …)
    are resized and cropped by PIL in their native mode first — Pillow picks NEAREST for palette / bilevel images and
    resamples alpha-premultiplied for RGBA / LA, so converting first would change the tile — and come back as
    finished 224x224 RGB tiles."""
    def _one(im: ImageLike) -> np.ndarray:
        if isinstance(im, str):
            im = PIL.Image.open(im)
        elif isinstance(im, np.ndarray):
            im = PIL.Image.fromarray(im)
        if im.mode != "RGB":
            im = resize_center_crop(im, SIZE, crop).convert("RGB")
        return np.asarray(im)

    if workers > 1 and len(images) > 1:
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=workers) as ex:
            return list(ex.map(_one, images))
    return [_one(im) for im in images]


def to_uint8_tiles_device(images: Sequence[ImageLike], engine, crop: str = "floor", workers: int = 0):
    """Batch of images -> uint8 CUDA tensor ``[n,224,224,3]``: decode on the host, resize + crop on the device."""
    import torch
    arrays = decode_rgb(images, workers)
    buf, descs = pack_rgb(arrays, crop=crop, pinned=torch.cuda.is_available())
    return engine.resize_crop(buf.to(engine.device, non_blocking=True), descs)


def to_uint8_tiles(images: Sequence[ImageLike], workers: int = 0, crop: str = "floor") -> np.ndarray:
    """Batch of images -> contiguous uint8 array ``[n,224,224,3]`` (NHWC).

    ``workers > 1`` decodes / resizes in a thread pool (PIL releases the GIL in its C loops) — the host-side
    counterpart of the reference's ``DataLoader(num_workers=…)`` (``embedders/plip.py:39``)."""
    out = np.empty((len(images), SIZE, SIZE, 3), dtype=np.uint8)

    def _one_tile(im: ImageLike) -> np.ndarray:
        return np.asarray(resize_center_crop(load_rgb(im), SIZE, crop))

    if workers > 1 and len(images) > 1:
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=workers) as ex:
            for i, tile in enumerate(ex.map(_one_tile, images)):
                out[i] = tile
        return out
    for i, im in enumerate(images):
        out[i] = _one_tile(im)
    return out


def resize_center_crop_bilinear(img: PIL.Image.Image, size: int = SIZE) -> PIL.Image.Image:
    """torchvision ``Resize(size)`` (PIL ``BILINEAR``, shortest edge to ``size``, long edge ``int(size * long /
    short)``) + ``CenterCrop(size)`` (``round`` offsets): the MuDiPath transform (``reproducibility/embedders/
    factory.py:41-46``) before ``ToTensor``.  A ``size x size`` image is returned as it is, as Pillow's same-size
    ``resize`` copies it."""
    w, h = img.size
    if (w, h) == (size, size):
        return img
    nw, nh, left, top = resize_plan(w, h, size, crop="round")
    if (nw, nh) != (w, h):
        img = img.resize((nw, nh), resample=PIL.Image.BILINEAR)
    return img.crop((left, top, left + size, top + size))


def to_uint8_tiles_bilinear(images: Sequence[ImageLike], workers: int = 0) -> np.ndarray:
    """Batch of images -> uint8 ``[n,224,224,3]`` through :func:`resize_center_crop_bilinear`, after the RGB
    conversion the reference's ``CLIPImageDataset`` applies first (``internal_datasets.py:42``)."""
    out = np.empty((len(images), SIZE, SIZE, 3), dtype=np.uint8)

    def _one(im: ImageLike) -> np.ndarray:
        return np.asarray(resize_center_crop_bilinear(load_rgb(im), SIZE))

    if workers > 1 and len(images) > 1:
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=workers) as ex:
            for i, tile in enumerate(ex.map(_one, images)):
                out[i] = tile
        return out
    for i, im in enumerate(images):
        out[i] = _one(im)
    return out


def chunks(seq: Sequence, n: int) -> Iterable[Sequence]:
    for i in range(0, len(seq), n):
        yield seq[i:i + n]
