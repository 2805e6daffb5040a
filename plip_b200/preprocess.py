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

import math

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
    return resize_crop_at(img, *resize_plan(w, h, size, crop), size=size)


def resize_crop_at(img: PIL.Image.Image, nw: int, nh: int, left: int, top: int, size: int = SIZE) -> PIL.Image.Image:
    """Bicubic resize to ``nw x nh`` (skipped when the size does not change, as Pillow copies then), then the
    ``size x size`` crop at ``(left, top)``: what ``plip_resize_crop_u8`` computes for one descriptor."""
    if (nw, nh) != img.size:
        img = img.resize((nw, nh), resample=PIL.Image.BICUBIC)
    return img.crop((left, top, left + size, top + size))


# numpy twin of ``plip_resize_desc_t`` (include/plip_b200.h)
RESIZE_DESC_DTYPE = np.dtype([("offset", "<i8"), ("width", "<i4"), ("height", "<i4"), ("new_width", "<i4"),
                              ("new_height", "<i4"), ("left", "<i4"), ("top", "<i4")])


def device_resizable(w: int, h: int, size: int = SIZE) -> bool:
    """Whether ``plip_resize_crop_u8`` takes a ``w x h`` image: its filter banks (224 horizontal + 32 vertical rows of
    ``2*ceil(2*scale)+1`` taps, padded to 4) plus one output row's strip of source rows must fit 200 KB of shared
    memory — shortest edges up to ~6,000 px at ordinary aspect ratios.  Larger images go through PIL."""
    nw, nh, _, _ = resize_plan(w, h, size)
    return resize_fits_device(w, h, nw, nh, size)


def resize_fits_device(w: int, h: int, nw: int, nh: int, size: int = SIZE) -> bool:
    """Whether the tile resize kernels take a ``w x h`` image resized to ``nw x nh`` (sizes 1..65536; the shared-memory
    plan of :func:`device_resizable`)."""
    import math
    if min(w, h, nw, nh) < 1 or max(w, h, nw, nh) > 65536:
        return False

    def taps4(i, o):
        return (2 * math.ceil(2.0 * max(i / o, 1.0)) + 1 + 3) // 4 * 4

    vs = h / nh
    tables = (size * taps4(w, nw) + 32 * taps4(h, nh) + 2 * (size + 32)) * 4
    strip_rows = min(h, math.ceil(4.0 * max(vs, 1.0)) + 3) + 3
    return tables + strip_rows * size * 3 <= 200 * 1024


def pack_rgb(arrays: Sequence[np.ndarray], crop: str = "floor", pinned: bool = False, plan=None):
    """Concatenate ``[h,w,3] uint8`` arrays into one byte buffer + their resize descriptors.

    ``plan``: per image ``(new_width, new_height, left, top)`` (any array with those fields, e.g.
    ``TrainTransform`` parameters); by default the shortest-edge-224 resize + centre crop of :func:`resize_plan`.
    Returns ``(buffer uint8 torch tensor [total], descs np.ndarray[RESIZE_DESC_DTYPE])``; image offsets are
    rounded up to 16 bytes."""
    import torch
    descs = np.zeros(len(arrays), dtype=RESIZE_DESC_DTYPE)
    off = 0
    for i, a in enumerate(arrays):
        if a.ndim != 3 or a.shape[2] != 3 or a.dtype != np.uint8:
            raise ValueError(f"image {i}: expected an [h,w,3] uint8 array, got {a.dtype} {a.shape}")
        h, w = int(a.shape[0]), int(a.shape[1])
        if plan is None:
            nw, nh, left, top = resize_plan(w, h, SIZE, crop)
        else:
            nw, nh, left, top = (int(plan[i][k]) for k in ("new_width", "new_height", "left", "top"))
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


# numpy twin of ``plip_warp_desc_t`` (include/plip_b200.h)
WARP_DESC_DTYPE = np.dtype([("affine", "<f8", (6,)), ("perspective", "<f8", (8,)), ("flip", "<i4"),
                            ("apply_perspective", "<i4"), ("fill", "<i4"), ("reserved", "<i4")])

# One image's draw of :class:`TrainTransform`: the decoded size, the resize + crop, the affine and perspective
# parameters as torchvision draws them, and the warp descriptor built from them.
TRAIN_PARAMS_DTYPE = np.dtype([
    ("width", "<i4"), ("height", "<i4"),            # decoded RGB image
    ("new_width", "<i4"), ("new_height", "<i4"),    # Resize([first_resize])
    ("left", "<i4"), ("top", "<i4"),                # RandomCrop origin (j, i)
    ("angle", "<f8"), ("translate", "<i4", (2,)), ("scale", "<f8"), ("shear", "<f8", (2,)),  # RandomAffine
    ("endpoints", "<i4", (4, 2)),                   # RandomPerspective corners (when warp.apply_perspective)
    ("warp", WARP_DESC_DTYPE)])

FILL = 127
PERSPECTIVE_CORNERS = [[0, 0], [SIZE - 1, 0], [SIZE - 1, SIZE - 1], [0, SIZE - 1]]


def inverse_affine_matrix(angle: float, translate, scale: float, shear, center=(SIZE * 0.5, SIZE * 0.5)) -> List[float]:
    """Pillow AFFINE coefficients (output pixel -> source point) of a rotation by ``angle`` degrees, a translation,
    a scale and x / y shears in degrees about ``center``: torchvision's ``_get_inverse_affine_matrix`` with the same
    double operations in the same order, so the coefficients are the same bits."""
    rot, sx, sy = math.radians(angle), math.radians(shear[0]), math.radians(shear[1])
    cx, cy = center
    tx, ty = translate
    a = math.cos(rot - sy) / math.cos(sy)
    b = -math.cos(rot - sy) * math.tan(sx) / math.cos(sy) - math.sin(rot)
    c = math.sin(rot - sy) / math.cos(sy)
    d = -math.sin(rot - sy) * math.tan(sx) / math.cos(sy) + math.cos(rot)
    m = [x / scale for x in (d, -b, 0.0, -c, a, 0.0)]   # (R S Sh)^-1, determinant 1 before the scale
    m[2] += m[0] * (-cx - tx) + m[1] * (-cy - ty)
    m[5] += m[3] * (-cx - tx) + m[4] * (-cy - ty)
    m[2] += cx
    m[5] += cy
    return m


def perspective_coeffs(startpoints, endpoints) -> List[float]:
    """Pillow PERSPECTIVE coefficients mapping ``endpoints`` back to ``startpoints``: torchvision's
    ``_get_perspective_coeffs``, a float64 least-squares solve on the CPU rounded to float32."""
    import torch
    a = torch.zeros(8, 8, dtype=torch.float64)
    for i, ((sx, sy), (ex, ey)) in enumerate(zip(startpoints, endpoints)):
        a[2 * i] = torch.tensor([ex, ey, 1, 0, 0, 0, -sx * ex, -sx * ey], dtype=torch.float64)
        a[2 * i + 1] = torch.tensor([0, 0, 0, ex, ey, 1, -sy * ex, -sy * ey], dtype=torch.float64)
    b = torch.tensor(startpoints, dtype=torch.float64).view(8)
    return torch.linalg.lstsq(a, b, driver="gels").solution.to(torch.float32).tolist()


class ParamStream:
    """The random draws of one pass of the reference's ``DataLoader(CLIPImageDataset(images, _train_transform(...)),
    batch_size, num_workers)`` over a list of images, handed out in image order.

    Creating it draws the iterator's int64 base seed from torch's default generator, as the ``DataLoader`` iterator
    does.  With ``num_workers == 0`` the transforms then draw from the default generator, image after image; with
    ``k`` workers, worker ``w`` is seeded with ``base_seed + w`` and transforms batches ``w, w + k, w + 2k, ...``, and the
    default generator moves by the base-seed draw only."""

    def __init__(self, transform: "TrainTransform", num_workers: int = 0, batch_size: int = 1):
        import torch
        if int(num_workers) < 0 or int(batch_size) < 1:
            raise ValueError(f"num_workers must be >= 0 and batch_size >= 1, got {num_workers} and {batch_size}")
        self.transform, self.num_workers, self.batch_size = transform, int(num_workers), int(batch_size)
        base = int(torch.empty((), dtype=torch.int64).random_().item())
        self.generators = [torch.Generator().manual_seed(base + w) for w in range(self.num_workers)]
        self.index = 0

    def draw(self, sizes) -> np.ndarray:
        """Parameters of the next ``len(sizes)`` images, given their ``(width, height)``: ``TRAIN_PARAMS_DTYPE``."""
        out = np.zeros(len(sizes), dtype=TRAIN_PARAMS_DTYPE)
        for k, (w, h) in enumerate(sizes):
            gen = None
            if self.num_workers:
                gen = self.generators[(self.index // self.batch_size) % self.num_workers]
            out[k] = self.transform.draw_one(int(w), int(h), gen)
            self.index += 1
        return out


class TrainTransform:
    """The reference's train-time transform ``_train_transform(first_resize, n_px)``
    (``reproducibility/embedders/transform.py:18-42``; the OpenPath preprocess of ``scripts/extract_embedding.py``)
    up to ``ToTensor``, on the GPU and bit-identical to torchvision on PIL:
    ``Resize([first_resize], BICUBIC)``, ``RandomCrop([224])``, ``RandomHorizontalFlip()``,
    ``RandomAffine(10, (0.1, 0.1), (0.8, 1.2), (-15, 15, -15, 15), BILINEAR, fill=127)`` and
    ``RandomPerspective(0.3, p=0.3, BILINEAR, fill=127)``.  ToTensor and CLIP's Normalize are fused into the engine's
    uint8 input.

    The random parameters are drawn on the host with torch's generators, in torchvision's order, and laid out as the
    reference's ``DataLoader`` lays them out (:class:`ParamStream`): under the same torch RNG state the tiles equal
    torchvision's, bit for bit.  The resize + crop is ``plip_resize_crop_u8`` (images it cannot take are resized with
    PIL on host threads), the flip and warps are ``plip_warp_tiles_u8``."""

    def __init__(self, first_resize: int = 512, n_px: int = SIZE):
        if int(n_px) != SIZE:
            raise ValueError(f"n_px must be {SIZE}: the image tower encodes {SIZE}x{SIZE} tiles (got {n_px})")
        if int(first_resize) < SIZE:
            raise ValueError(f"first_resize must be >= n_px = {SIZE}: RandomCrop([{SIZE}]) needs an image at least "
                             f"that large (got {first_resize})")
        self.first_resize, self.n_px = int(first_resize), SIZE

    def __repr__(self) -> str:
        return f"TrainTransform(first_resize={self.first_resize}, n_px={self.n_px})"

    def draw_one(self, w: int, h: int, generator=None) -> tuple:
        """One image's parameters (a ``TRAIN_PARAMS_DTYPE`` row as a tuple), drawn from ``generator`` (``None``: torch's
        default generator) with torchvision's calls in torchvision's order."""
        import torch
        g = generator
        nw, nh, _, _ = resize_plan(w, h, self.first_resize)
        top = left = 0
        if (nw, nh) != (SIZE, SIZE):                    # RandomCrop.get_params draws nothing for an exact fit
            top = int(torch.randint(0, nh - SIZE + 1, size=(1,), generator=g).item())
            left = int(torch.randint(0, nw - SIZE + 1, size=(1,), generator=g).item())
        flip = bool(torch.rand(1, generator=g) < 0.5)
        angle = float(torch.empty(1).uniform_(-10.0, 10.0, generator=g).item())
        max_d = float(0.1 * SIZE)
        tx = int(round(torch.empty(1).uniform_(-max_d, max_d, generator=g).item()))
        ty = int(round(torch.empty(1).uniform_(-max_d, max_d, generator=g).item()))
        scale = float(torch.empty(1).uniform_(0.8, 1.2, generator=g).item())
        shx = float(torch.empty(1).uniform_(-15.0, 15.0, generator=g).item())
        shy = float(torch.empty(1).uniform_(-15.0, 15.0, generator=g).item())
        affine = inverse_affine_matrix(angle, (tx, ty), scale, (shx, shy))
        ends, coeffs, persp = np.zeros((4, 2), np.int32), [0.0] * 8, bool(torch.rand(1, generator=g) < 0.3)
        if persp:                                        # RandomPerspective.get_params(224, 224, 0.3)
            dx = dy = int(0.3 * (SIZE // 2))
            lo_x, hi_x, lo_y, hi_y = (0, dx + 1), (SIZE - dx - 1, SIZE), (0, dy + 1), (SIZE - dy - 1, SIZE)
            for k, (rx, ry) in enumerate([(lo_x, lo_y), (hi_x, lo_y), (hi_x, hi_y), (lo_x, hi_y)]):
                ends[k, 0] = int(torch.randint(rx[0], rx[1], size=(1,), generator=g).item())
                ends[k, 1] = int(torch.randint(ry[0], ry[1], size=(1,), generator=g).item())
            coeffs = perspective_coeffs(PERSPECTIVE_CORNERS, ends.tolist())
        warp = (affine, coeffs, int(flip), int(persp), FILL, 0)
        return (w, h, nw, nh, left, top, angle, (tx, ty), scale, (shx, shy), ends, warp)

    def stream(self, num_workers: int = 0, batch_size: int = 1) -> ParamStream:
        """A new pass over a list of images (draws the ``DataLoader`` base seed now)."""
        return ParamStream(self, num_workers, batch_size)

    def draw(self, sizes, num_workers: int = 0, batch_size: int = 1) -> np.ndarray:
        """Parameters of one ``DataLoader`` pass over images of these ``(width, height)``."""
        return self.stream(num_workers, batch_size).draw(sizes)

    def apply(self, arrays: Sequence[np.ndarray], params: np.ndarray, device="cuda", workers: int = 0):
        """Decoded RGB ``[h,w,3]`` uint8 arrays + their drawn parameters -> CUDA uint8 ``[n,224,224,3]`` tiles."""
        import torch
        from .engine import resize_crop, warp_tiles
        device = torch.device(device)
        if len(arrays) != len(params):
            raise ValueError(f"{len(arrays)} images but {len(params)} parameter rows")
        for i, (a, p) in enumerate(zip(arrays, params)):
            if a.ndim != 3 or a.shape[2] != 3 or a.dtype != np.uint8:
                raise ValueError(f"image {i}: expected an [h,w,3] uint8 array, got {a.dtype} {a.shape}")
            if (a.shape[1], a.shape[0]) != (int(p["width"]), int(p["height"])):
                raise ValueError(f"image {i} is {a.shape[1]}x{a.shape[0]}, its parameters were drawn for "
                                 f"{int(p['width'])}x{int(p['height'])}")
        if not len(arrays):
            return torch.empty((0, SIZE, SIZE, 3), dtype=torch.uint8, device=device)
        if all(device_resizable(a.shape[1], a.shape[0], self.first_resize) for a in arrays):
            buf, descs = pack_rgb(arrays, pinned=True, plan=params)
            tiles = resize_crop(buf.to(device, non_blocking=True), descs)
        else:                                            # too large for the device resize: PIL on host threads
            def _one(k):
                p = params[k]
                return np.asarray(resize_crop_at(PIL.Image.fromarray(arrays[k]), int(p["new_width"]),
                                                 int(p["new_height"]), int(p["left"]), int(p["top"])))
            host = np.empty((len(arrays), SIZE, SIZE, 3), dtype=np.uint8)
            if workers > 1 and len(arrays) > 1:
                from concurrent.futures import ThreadPoolExecutor
                with ThreadPoolExecutor(max_workers=workers) as ex:
                    for k, t in enumerate(ex.map(_one, range(len(arrays)))):
                        host[k] = t
            else:
                for k in range(len(arrays)):
                    host[k] = _one(k)
            tiles = torch.from_numpy(host).pin_memory().to(device, non_blocking=True)
        return warp_tiles(tiles, params["warp"], out=tiles)

    def tiles(self, images: Sequence[ImageLike], device="cuda", num_workers: int = 0, batch_size: int = 1):
        """Paths / PIL images / arrays -> CUDA uint8 ``[n,224,224,3]``: what the reference's ``DataLoader`` with this
        ``batch_size`` and ``num_workers`` hands to the model, before ToTensor, under the same torch RNG state.  Images
        are converted to RGB first, as ``CLIPImageDataset`` does.  ``batch_size`` / ``num_workers`` only decide how the
        random draws are laid out; decoding uses ``num_workers`` host threads."""
        arrays = decode_rgb(list(images), int(num_workers))
        params = self.draw([(a.shape[1], a.shape[0]) for a in arrays], num_workers, batch_size)
        return self.apply(arrays, params, device, int(num_workers))


def chunks(seq: Sequence, n: int) -> Iterable[Sequence]:
    for i in range(0, len(seq), n):
        yield seq[i:i + n]
