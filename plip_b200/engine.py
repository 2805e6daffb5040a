"""Python handle on the CUDA engine: device memory and streams come from torch, compute from the
C ABI (``libplip_b200.so``).  There is no fallback path: a missing library or GPU raises."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Mapping, Optional, Tuple, Union

import numpy as np
import torch

from ._lib import SgdProblem as _SgdProblem
from ._lib import check, lib
from .weights import operand_format, pack_state_dict, vision_patch

PIX_F32_NCHW, PIX_BF16_NCHW, PIX_U8_NHWC = 0, 1, 2
IDS_I32, IDS_I64 = 0, 1
EMBED_DIM = 512
# Embedding widths the linear probe (plip_sgd_fit / plip_linear_decision) runs at: the CLIP projection and MuDiPath's
# DenseNet-121 features.
PROBE_DIMS = (EMBED_DIM, 1024)
IMAGE_SIZE = 224
MAX_TEXT_LEN = 77


VISION_DIM, VISION_HEADS = 768, 12
TEXT_DIM, TEXT_HEADS = 512, 8
NUM_LAYERS = 12

# Module-level defaults are CLIP ViT-B/32's (PLIP); an Engine on ViT-B/16 weights passes its own patch size (16).
PATCH = 32
MAX_GRID = 32  # interpolate_pos_encoding: at most 32 x 32 patches (1024 px per side at patch 32, 512 at 16; 1025 tokens)


def _check_size(h: int, w: int, interpolate_pos_encoding: bool, patch: int = PATCH) -> None:
    if not interpolate_pos_encoding:
        if h != IMAGE_SIZE or w != IMAGE_SIZE:
            raise ValueError(f"Input image size ({h}*{w}) doesn't match model (224*224).")  # TF:204-207
    elif not (h >= patch and w >= patch and h // patch <= MAX_GRID and w // patch <= MAX_GRID):
        raise ValueError(f"Input image size ({h}*{w}) out of range for interpolate_pos_encoding: height and width "
                         f"must be >= {patch} with at most {MAX_GRID} patches of {patch} per side "
                         f"(<= {(MAX_GRID + 1) * patch - 1} px)")


def _pixel_format(t: Union[torch.Tensor, np.ndarray], interpolate_pos_encoding: bool = False, patch: int = PATCH) -> int:
    """Validate an image batch and return its C-ABI pixel format (error text mirrors TF:204-207).  With
    ``interpolate_pos_encoding`` any height / width with ``P <= H, W`` and ``H // P, W // P <= 32`` is accepted
    (``P``: the vision patch size, 32 or 16)."""
    shape, dtype = tuple(t.shape), t.dtype
    if dtype in (torch.uint8, np.dtype("uint8")):
        if len(shape) != 4 or shape[3] != 3:
            raise ValueError(f"uint8 images must be [n,224,224,3] (NHWC), got {shape}")
        _check_size(shape[1], shape[2], interpolate_pos_encoding, patch)
        return PIX_U8_NHWC
    if len(shape) != 4 or shape[1] != 3:
        raise ValueError(f"pixel_values must be [n,3,224,224], got {shape}")
    _check_size(shape[2], shape[3], interpolate_pos_encoding, patch)
    if dtype in (torch.float32, np.dtype("float32")):
        return PIX_F32_NCHW
    if dtype == torch.bfloat16:
        return PIX_BF16_NCHW
    raise TypeError(f"unsupported pixel dtype {dtype} (float32, bfloat16 or uint8)")


def _pixel_hw(t: Union[torch.Tensor, np.ndarray], fmt: int) -> Tuple[int, int]:
    """``(height, width)`` of a batch ``_pixel_format`` accepted as ``fmt``."""
    return (int(t.shape[1]), int(t.shape[2])) if fmt == PIX_U8_NHWC else (int(t.shape[2]), int(t.shape[3]))


def vision_seq_len(height: int, width: int, patch: int = PATCH) -> int:
    """Tokens of one image: ``(H // P) * (W // P)`` patches of ``P`` pixels + the class token (50 at 224 x 224 for
    ``P = 32``, 197 for ``P = 16``)."""
    return (height // patch) * (width // patch) + 1


def _ids_dtype(dtype) -> int:
    if dtype in (torch.int64, np.dtype("int64")):
        return IDS_I64
    if dtype in (torch.int32, np.dtype("int32")):
        return IDS_I32
    raise TypeError(f"input_ids must be int32 or int64, got {dtype}")


def _check_ids(input_ids, attention_mask) -> Tuple[int, int]:
    if len(input_ids.shape) != 2:
        raise ValueError(f"input_ids must be [n, seq_len], got {tuple(input_ids.shape)}")
    n, s = int(input_ids.shape[0]), int(input_ids.shape[1])
    if s > MAX_TEXT_LEN:
        raise ValueError(
            "Sequence length must be less than max_position_embeddings (got `sequence length`: "
            f"{s} and max_position_embeddings: {MAX_TEXT_LEN}")  # TF:243-247
    if attention_mask is not None and tuple(attention_mask.shape) != (n, s):
        raise ValueError(f"attention_mask shape {tuple(attention_mask.shape)} != input_ids shape {(n, s)}")
    return n, s


WINDOW = IMAGE_SIZE  # the side of a region window (plip_encode_windows)


def check_region(region: Union[torch.Tensor, np.ndarray]) -> Tuple[int, int, int]:
    """Validate a uint8 RGB region ``[H, W, 3]`` whose pixels are packed (channel stride 1, pixel stride 3; rows may be
    any number of bytes apart, e.g. a view into a wider array) and at least one window in size.  Returns
    ``(H, W, row_pitch_bytes)``; raises ``ValueError`` otherwise."""
    if region.dtype not in (torch.uint8, np.dtype("uint8")):
        raise ValueError(f"a region must be uint8 RGB [H, W, 3], got dtype {region.dtype}")
    shape = tuple(region.shape)
    if len(shape) != 3 or shape[2] != 3:
        raise ValueError(f"a region must be uint8 RGB [H, W, 3], got shape {shape}")
    h, w = int(shape[0]), int(shape[1])
    if h < WINDOW or w < WINDOW:
        raise ValueError(f"region {h}x{w} is smaller than one {WINDOW}x{WINDOW} window")
    strides = region.stride() if torch.is_tensor(region) else tuple(s // region.itemsize for s in region.strides)
    if strides[2] != 1 or strides[1] != 3 or strides[0] < 3 * w:
        raise ValueError(f"a region needs packed RGB pixels (strides (>= 3 * W, 3, 1) in bytes), got strides {strides}")
    return h, w, int(strides[0])


def check_origins(origins, height: int, width: int) -> np.ndarray:
    """``[n, 2]`` (row, col) window origins as a contiguous int32 array, each window inside the ``height x width``
    region; ``ValueError`` naming the first window that is not."""
    o = np.asarray(origins.cpu() if torch.is_tensor(origins) else origins)
    if o.size == 0:
        return np.zeros((0, 2), np.int32)
    if o.ndim != 2 or o.shape[1] != 2 or o.dtype.kind not in "iu":
        raise ValueError(f"origins must be integer [n, 2] (row, col), got {o.dtype} {o.shape}")
    bad = (o[:, 0] < 0) | (o[:, 1] < 0) | (o[:, 0] > height - WINDOW) | (o[:, 1] > width - WINDOW)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise ValueError(f"window {i} at ({int(o[i, 0])}, {int(o[i, 1])}) is outside the {height}x{width} region "
                         f"(rows 0..{height - WINDOW}, columns 0..{width - WINDOW})")
    return np.ascontiguousarray(o, dtype=np.int32)


def _device_region(region) -> Tuple[int, int, int]:
    if not (torch.is_tensor(region) and region.is_cuda):
        raise ValueError("the region must be a CUDA tensor here; host regions go through plip_b200.regions.encode_region")
    return check_region(region)


@torch.no_grad()
def window_background_counts(region: torch.Tensor, origins, threshold: int = 200) -> torch.Tensor:
    """Per window, the pixels whose three channels are all ``>= threshold``: int32 ``[n]`` on the region's device,
    exact (``plip_window_background_counts``; needs no engine).  ``count / 50176`` is the reference's
    ``background_ratio`` of the window."""
    h, w, pitch = _device_region(region)
    o = check_origins(origins, h, w)
    n = int(o.shape[0])
    out = torch.empty(n, device=region.device, dtype=torch.int32)
    if n:
        with torch.cuda.device(region.device):
            check(lib().plip_window_background_counts(region.data_ptr(), h, w, pitch, o.ctypes.data, n, int(threshold),
                                                      out.data_ptr(), torch.cuda.current_stream(region.device).cuda_stream),
                  "plip_window_background_counts")
    return out


def _packed_u8(t, what: str, channels) -> Tuple[int, int, int, int]:
    """``(H, W, C, row_pitch_bytes)`` of a uint8 ``[H, W]`` / ``[H, W, C]`` array with packed pixels (rows may be any
    number of bytes apart), ``C`` in ``channels``; ``ValueError`` otherwise."""
    if t.dtype not in (torch.uint8, np.dtype("uint8")):
        raise ValueError(f"{what} must be uint8, got dtype {t.dtype}")
    shape = tuple(t.shape)
    c = shape[2] if len(shape) == 3 else 1
    if len(shape) not in (2, 3) or c not in channels:
        raise ValueError(f"{what} must be uint8 {' or '.join('[H, W]' if k == 1 else f'[H, W, {k}]' for k in channels)}"
                         f", got shape {shape}")
    h, w = int(shape[0]), int(shape[1])
    if h < 1 or w < 1:
        raise ValueError(f"{what} is empty ({h}x{w})")
    strides = tuple(t.stride()) if torch.is_tensor(t) else tuple(s // t.itemsize for s in t.strides)
    if (len(shape) == 3 and strides[2] != 1) or strides[1] != c or strides[0] < c * w:
        raise ValueError(f"{what} needs packed pixels (strides (>= {c} * W, {c}{', 1' if len(shape) == 3 else ''}) in "
                         f"bytes), got strides {strides}")
    return h, w, c, int(strides[0])


MAX_RESIZE = 65536
_RC_BAD_ARGUMENT = -2  # PLIP_REQUIRE: an argument the library rejected before any launch


def _check_args(rc: int, what: str) -> None:
    """``check``, but an argument the library rejected raises ``ValueError`` (nothing was launched)."""
    if rc == _RC_BAD_ARGUMENT:
        from ._lib import last_error
        raise ValueError(f"{what}: {last_error()}")
    check(rc, what)


def resize_filter_bounds(in_size: int, out_size: int) -> np.ndarray:
    """The filter window of every output index of one resize axis, as the device resize computes it
    (``plip_resize_filter_bounds``; host only): int32 ``[out_size, 2]`` = (first source index, count)."""
    if not (1 <= in_size <= MAX_RESIZE and 1 <= out_size <= MAX_RESIZE):
        raise ValueError(f"resize sizes {in_size} -> {out_size} are outside 1..{MAX_RESIZE}")
    b = np.zeros((out_size, 2), np.int32)
    check(lib().plip_resize_filter_bounds(int(in_size), int(out_size), b.ctypes.data), "plip_resize_filter_bounds")
    return b


class ResizeWorkspace:
    """Device scratch of ``plip_resize_region_u8``, grown on demand and reused across calls on one stream."""

    def __init__(self, device):
        self.device, self.buf = torch.device(device), None

    def get(self, nbytes: int) -> torch.Tensor:
        if self.buf is None or self.buf.numel() < nbytes:
            self.buf = torch.empty(nbytes, dtype=torch.uint8, device=self.device)  # caching-allocator blocks: 512-aligned
        return self.buf


@torch.no_grad()
def resize_rows(band: torch.Tensor, src_row0: int, height: int, new_h: int, new_w: int, rows: Tuple[int, int],
                out: torch.Tensor, workspace: Optional[ResizeWorkspace] = None) -> torch.Tensor:
    """Output rows ``[o0, o1)`` of the ``new_h x new_w`` Pillow-bicubic resize of a ``height x W`` RGB uint8 image, of
    which ``band`` (CUDA ``[rows, W, 3]``, rows may be strided) holds the rows from ``src_row0`` on; written into
    ``out`` (CUDA uint8 ``[o1 - o0, new_w, 3]``, rows may be strided).  The filters are the full image's, so ranges
    stitched together are the whole resize bit for bit.  ``plip_resize_region_u8``; every argument, including that the
    band holds the source rows the range reads, is checked before any launch (``ValueError``)."""
    if not (torch.is_tensor(band) and band.is_cuda):
        raise ValueError("resize_rows: the source must be a CUDA tensor")
    bh, w, _, pitch = _packed_u8(band, "the source", (3,))
    o0, o1 = int(rows[0]), int(rows[1])
    if not (1 <= height <= MAX_RESIZE and 1 <= w <= MAX_RESIZE and 1 <= new_h <= MAX_RESIZE and 1 <= new_w <= MAX_RESIZE):
        raise ValueError(f"resize {height}x{w} -> {new_h}x{new_w}: sizes must be in 1..{MAX_RESIZE}")
    if not 0 <= o0 < o1 <= new_h:
        raise ValueError(f"output rows [{o0}, {o1}) are not a non-empty range of 0..{new_h}")
    if not (0 <= src_row0 and src_row0 + bh <= height):
        raise ValueError(f"a band of {bh} rows at row {src_row0} is not inside the {height} source rows")
    if not (torch.is_tensor(out) and out.is_cuda and out.device == band.device):
        raise ValueError(f"the output must be a CUDA tensor on {band.device}")
    oh, ow, _, opitch = _packed_u8(out, "the output", (3,))
    if (oh, ow) != (o1 - o0, new_w):
        raise ValueError(f"the output is {oh}x{ow}, rows [{o0}, {o1}) of width {new_w} need {o1 - o0}x{new_w}")
    L = lib()
    need = C.c_uint64(0)
    _check_args(L.plip_resize_region_workspace(int(height), w, int(new_h), int(new_w), o0, o1, C.byref(need)),
                "plip_resize_region_workspace")
    ws = (workspace or ResizeWorkspace(band.device)).get(int(need.value))
    with torch.cuda.device(band.device):
        _check_args(L.plip_resize_region_u8(band.data_ptr(), pitch, int(src_row0), bh, int(height), w, out.data_ptr(),
                                            opitch, int(new_h), int(new_w), o0, o1, ws.data_ptr(), ws.numel(),
                                            torch.cuda.current_stream(band.device).cuda_stream), "plip_resize_region_u8")
    return out


def resize_region(region: torch.Tensor, new_h: int, new_w: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``PIL.Image.fromarray(region).resize((new_w, new_h))`` on the device, bit for bit (antialiased BICUBIC, no
    reducing_gap), at any ratio from upscaling to shrinks of over 64x: CUDA uint8 ``[H, W, 3]`` (rows may be strided)
    -> ``[new_h, new_w, 3]`` (``out``, which may be a row-strided view, or a new tensor).  Needs no engine."""
    if not (torch.is_tensor(region) and region.is_cuda):
        raise ValueError("resize_region: the region must be a CUDA tensor")
    h = _packed_u8(region, "a region", (3,))[0]
    if out is None:
        if not (1 <= new_h <= MAX_RESIZE and 1 <= new_w <= MAX_RESIZE):
            raise ValueError(f"output size {new_h}x{new_w} is outside 1..{MAX_RESIZE}")
        out = torch.empty((int(new_h), int(new_w), 3), dtype=torch.uint8, device=region.device)
    return resize_rows(region, 0, h, int(new_h), int(new_w), (0, int(new_h)), out)


def _device_tiles(t, what: str) -> int:
    """``n`` of a contiguous CUDA uint8 ``[n,224,224,3]`` tensor; ``ValueError`` otherwise."""
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.uint8 and t.dim() == 4
            and tuple(t.shape[1:]) == (IMAGE_SIZE, IMAGE_SIZE, 3) and t.is_contiguous()):
        raise ValueError(f"{what} must be a contiguous CUDA uint8 [n,224,224,3] tensor, got "
                         f"{getattr(t, 'dtype', type(t))} {tuple(getattr(t, 'shape', ()))}")
    return int(t.shape[0])


@torch.no_grad()
def resize_crop(src: torch.Tensor, descs: np.ndarray, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Packed RGB uint8 images on the device + host descriptors (``preprocess.pack_rgb``) -> uint8 tiles
    ``[n,224,224,3]`` on the same device; Pillow-exact bicubic resize and crop (``plip_resize_crop_u8``).  Needs no
    engine."""
    from .preprocess import RESIZE_DESC_DTYPE
    assert src.is_cuda and src.dtype == torch.uint8 and src.is_contiguous() and src.dim() == 1
    descs = np.ascontiguousarray(descs, dtype=RESIZE_DESC_DTYPE)
    n = int(descs.shape[0])
    if out is None:
        out = torch.empty((n, 224, 224, 3), device=src.device, dtype=torch.uint8)
    assert out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and out.numel() == n * 224 * 224 * 3
    if n:
        with torch.cuda.device(src.device):
            check(lib().plip_resize_crop_u8(src.data_ptr(), int(src.numel()), descs.ctypes.data, n, out.data_ptr(),
                                            torch.cuda.current_stream(src.device).cuda_stream), "plip_resize_crop_u8")
    return out


@torch.no_grad()
def resize_crop_fill(src: torch.Tensor, descs: np.ndarray, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """:func:`resize_crop` with the resized size and crop origin unrestricted (``plip_resize_crop_fill_u8``): tile pixel
    ``(x, y)`` is the resized image's ``(left + x, top + y)`` when that lies inside it, else ``(0, 0, 0)`` — PIL's
    ``resize(...).crop(...)`` past the image edge.  Every descriptor is checked before any launch (``ValueError``).
    Needs no engine."""
    from .preprocess import RESIZE_DESC_DTYPE
    if not (torch.is_tensor(src) and src.is_cuda and src.dtype == torch.uint8 and src.is_contiguous()
            and src.dim() == 1):
        raise ValueError("resize_crop_fill: src must be a contiguous 1-D CUDA uint8 tensor")
    descs = np.ascontiguousarray(descs, dtype=RESIZE_DESC_DTYPE).reshape(-1)
    n = int(descs.shape[0])
    if out is None:
        out = torch.empty((n, IMAGE_SIZE, IMAGE_SIZE, 3), device=src.device, dtype=torch.uint8)
    elif _device_tiles(out, "out") != n or out.device != src.device:
        raise ValueError(f"resize_crop_fill: out must be [{n},224,224,3] on {src.device}")
    if n:
        with torch.cuda.device(src.device):
            _check_args(lib().plip_resize_crop_fill_u8(src.data_ptr(), int(src.numel()), descs.ctypes.data, n,
                                                       out.data_ptr(), torch.cuda.current_stream(src.device).cuda_stream),
                        "plip_resize_crop_fill_u8")
    return out


@torch.no_grad()
def mask_value_sets(masks: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The byte values present in every (image, channel) of a contiguous CUDA uint8 ``[n, h, w, c]`` array (``c`` 1..8)
    as 256-bit sets: int32 ``[n, c, 8]`` on the same device (the bits of uint32 words; bit ``v & 31`` of word ``v >> 5``
    is value ``v``), one pass over the array (``plip_mask_value_sets_u8``).  ``out``: a contiguous int32 ``[n, c, 8]``
    tensor to fill.  Needs no engine."""
    if not (torch.is_tensor(masks) and masks.is_cuda and masks.dtype == torch.uint8 and masks.dim() == 4
            and masks.is_contiguous()):
        raise ValueError("mask_value_sets: masks must be a contiguous CUDA uint8 [n, h, w, c] tensor")
    n, h, w, c = (int(x) for x in masks.shape)
    if out is None:
        out = torch.empty((n, c, 8), dtype=torch.int32, device=masks.device)
    elif not (out.is_cuda and out.dtype == torch.int32 and tuple(out.shape) == (n, c, 8) and out.is_contiguous()
              and out.device == masks.device):
        raise ValueError(f"mask_value_sets: out must be a contiguous int32 [{n}, {c}, 8] tensor on {masks.device}")
    if n:
        with torch.cuda.device(masks.device):
            _check_args(lib().plip_mask_value_sets_u8(masks.data_ptr(), n, h, w, c, out.data_ptr(),
                                                      torch.cuda.current_stream(masks.device).cuda_stream),
                        "plip_mask_value_sets_u8")
    return out


@torch.no_grad()
def warp_tiles(tiles: torch.Tensor, params: np.ndarray, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Flip / affine / perspective warps of CUDA uint8 tiles ``[n,224,224,3]``, bit-identical to Pillow's
    ``Image.transpose`` and ``Image.transform(AFFINE | PERSPECTIVE, BILINEAR, fillcolor)`` (``plip_warp_tiles_u8``).
    ``params``: ``preprocess.WARP_DESC_DTYPE`` rows, one per tile (``TrainTransform`` draws them).  ``out``: a tensor
    of the same shape on the same device, ``tiles`` itself (in place) or a new tensor.  Every argument is checked
    before any launch (``ValueError``).  Needs no engine."""
    from .preprocess import WARP_DESC_DTYPE
    n = _device_tiles(tiles, "tiles")
    params = np.ascontiguousarray(params, dtype=WARP_DESC_DTYPE).reshape(-1)
    if params.shape[0] != n:
        raise ValueError(f"warp_tiles: {params.shape[0]} descriptors for {n} tiles")
    if out is None:
        out = torch.empty_like(tiles)
    elif _device_tiles(out, "out") != n or out.device != tiles.device:
        raise ValueError(f"warp_tiles: out must be [{n},224,224,3] on {tiles.device}")
    if n:
        with torch.cuda.device(tiles.device):
            _check_args(lib().plip_warp_tiles_u8(tiles.data_ptr(), out.data_ptr(), params.ctypes.data, n,
                                                 torch.cuda.current_stream(tiles.device).cuda_stream),
                        "plip_warp_tiles_u8")
    return out


@torch.no_grad()
def window_mask_counts(mask: torch.Tensor, origins, threshold: int = 10) -> torch.Tensor:
    """Per window, the mask elements ``> threshold``: int32 ``[n]`` on the mask's device, exact
    (``plip_window_mask_counts``; needs no engine).  ``mask``: CUDA uint8 ``[H, W]`` or ``[H, W, 3]`` (a decoded L or
    RGB mask; rows may be strided).  An RGB mask counts every channel, as the reference's ``np.sum(msk_patch_np > 0)``
    does, so ``count / 50176`` can exceed 1 there."""
    if not (torch.is_tensor(mask) and mask.is_cuda):
        raise ValueError("window_mask_counts: the mask must be a CUDA tensor")
    h, w, c, pitch = _packed_u8(mask, "a mask", (1, 3))
    if h < WINDOW or w < WINDOW:
        raise ValueError(f"mask {h}x{w} is smaller than one {WINDOW}x{WINDOW} window")
    if not -(2 ** 31) <= int(threshold) < 2 ** 31:
        raise ValueError(f"threshold {threshold} does not fit int32")
    o = check_origins(origins, h, w)
    n = int(o.shape[0])
    out = torch.empty(n, device=mask.device, dtype=torch.int32)
    if n:
        with torch.cuda.device(mask.device):
            check(lib().plip_window_mask_counts(mask.data_ptr(), h, w, c, pitch, o.ctypes.data, n, int(threshold),
                                                out.data_ptr(), torch.cuda.current_stream(mask.device).cuda_stream),
                  "plip_window_mask_counts")
    return out


@torch.no_grad()
def similarity_topk(query: torch.Tensor, space: torch.Tensor, k: int, scale: float = 1.0, normalize_query: bool = True,
                    normalize_space: bool = False, device: Union[int, str, torch.device, None] = None):
    """``plip_similarity_topk`` needs no engine handle (no weights involved): fused scores + top-k over ``space`` rows on
    ``device`` (default: the current CUDA device).  Returns ``(idx int32 [n,k], val f32 [n,k])``, best first."""
    if not torch.cuda.is_available():
        raise RuntimeError("plip_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    L = lib()
    q = query.to(torch.float32).to(dev, non_blocking=True).contiguous()
    s = space.to(torch.float32).to(dev, non_blocking=True).contiguous()
    n = int(q.shape[0])
    idx = torch.empty(n, k, device=dev, dtype=torch.int32)
    val = torch.empty(n, k, device=dev, dtype=torch.float32)
    if n == 0:
        return idx, val
    with torch.cuda.device(dev):
        check(L.plip_similarity_topk(q.data_ptr(), n, s.data_ptr(), int(s.shape[0]), C.c_float(scale), int(normalize_query),
                                     int(normalize_space), int(k), idx.data_ptr(), val.data_ptr(),
                                     torch.cuda.current_stream(dev).cuda_stream), "plip_similarity_topk")
    return idx, val


def sgd_shuffle_permutation(n: int, seed: int) -> np.ndarray:
    """The permutation scikit-learn's ``dataset.shuffle(seed)`` applies to the sample order every epoch (its
    Fisher-Yates with ``our_rand_r``): int32 ``[n]``, ``new_order[i] = old_order[sigma[i]]``.  Host only."""
    if not 1 <= int(n) < 2 ** 31:
        raise ValueError(f"n = {n} is outside 1..2^31-1")
    out = np.empty(int(n), np.int32)
    check(lib().plip_sgd_shuffle_permutation(int(n), int(seed) & 0xFFFFFFFF, out.ctypes.data),
          "plip_sgd_shuffle_permutation")
    return out


def probe_widths() -> str:
    """The accepted probe widths as an error message names them: ``"512 or 1024"``."""
    return " or ".join(map(str, PROBE_DIMS))


def _device_embeddings(x: torch.Tensor, what: str) -> Tuple[int, int]:
    if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.is_contiguous()
            and x.shape[1] in PROBE_DIMS):
        raise ValueError(f"{what} must be a contiguous CUDA float32 [n, d] tensor, d = {probe_widths()}")
    return int(x.shape[0]), int(x.shape[1])


@torch.no_grad()
def sgd_fit(x: torch.Tensor, class_ids, n_classes: int, problems, sigma, max_iter: int = 10000, tol: float = 1e-3,
            n_iter_no_change: int = 5):
    """scikit-learn's SGD logistic regression for many binary problems in one launch (``plip_sgd_fit``; needs no
    engine).  ``x``: CUDA float32 ``[n, d]``, ``d`` in ``PROBE_DIMS`` (512 or 1024); ``class_ids``: int ``[n]`` in
    ``0..n_classes-1``; ``problems``: one ``(alpha, pos_class, pos_weight, neg_weight, sigma_index)`` per problem;
    ``sigma``: int32 ``[n_sigma, n]`` epoch permutations (``sgd_shuffle_permutation``).  Returns device tensors
    ``(coef f32 [P, d], intercept f64 [P], n_iter int32 [P], overflow int32 [P])``; bad arguments raise ``ValueError`` before anything is launched."""
    n, d = _device_embeddings(x, "x")
    cls = np.ascontiguousarray(np.asarray(class_ids), dtype=np.int32)
    sig = np.ascontiguousarray(np.asarray(sigma), dtype=np.int32)
    if cls.shape != (n,) or sig.ndim != 2 or sig.shape[1] != n:
        raise ValueError(f"class ids {cls.shape} and sigma {sig.shape} do not match n = {n}")
    table = (_SgdProblem * len(problems))(*[_SgdProblem(float(a), float(wp), float(wn), int(pc), int(si))
                                            for a, pc, wp, wn, si in problems])
    p = len(problems)
    L = lib()
    need = C.c_uint64(0)
    _check_args(L.plip_sgd_workspace_bytes(n, int(sig.shape[0]), p, C.byref(need)), "plip_sgd_workspace_bytes")
    dev = x.device
    ws = torch.empty(int(need.value), dtype=torch.uint8, device=dev)
    coef = torch.empty(p, d, dtype=torch.float32, device=dev)
    intercept = torch.empty(p, dtype=torch.float64, device=dev)
    n_iter = torch.empty(p, dtype=torch.int32, device=dev)
    overflow = torch.empty(p, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _check_args(L.plip_sgd_fit(x.data_ptr(), n, d, cls.ctypes.data, int(n_classes), table, p, sig.ctypes.data,
                                   int(sig.shape[0]), int(max_iter), C.c_double(tol), int(n_iter_no_change),
                                   coef.data_ptr(), intercept.data_ptr(), n_iter.data_ptr(), overflow.data_ptr(),
                                   ws.data_ptr(), ws.numel(), torch.cuda.current_stream(dev).cuda_stream), "plip_sgd_fit")
    return coef, intercept, n_iter, overflow


@torch.no_grad()
def linear_decision(x: torch.Tensor, coef: torch.Tensor, intercept: torch.Tensor):
    """``decision_function`` and the predicted index of a linear classifier (``plip_linear_decision``; needs no engine):
    ``x`` CUDA float32 ``[n, d]``, ``coef`` float32 ``[C, d]`` (``d`` 512 or 1024), ``intercept`` ``[C]`` on the same
    device.  Returns ``(scores f32 [n, C], pred int32 [n])``: the first arg-max for ``C > 1``, ``score > 0`` for
    ``C == 1``."""
    n, d = _device_embeddings(x, "x")
    c, dc = _device_embeddings(coef, "coef")
    b = intercept.to(device=x.device, dtype=torch.float64).contiguous()
    if coef.device != x.device or dc != d or b.shape != (c,):
        raise ValueError(f"coef {tuple(coef.shape)} on {coef.device} and intercept {tuple(intercept.shape)} do not "
                         f"match x on {x.device}")
    scores = torch.empty(n, c, dtype=torch.float32, device=x.device)
    pred = torch.empty(n, dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device):
        _check_args(lib().plip_linear_decision(x.data_ptr(), n, d, coef.data_ptr(), b.data_ptr(), c, scores.data_ptr(),
                                               pred.data_ptr(), torch.cuda.current_stream(x.device).cuda_stream),
                    "plip_linear_decision")
    return scores, pred


def _device_embeddings_f64(x: torch.Tensor, what: str) -> Tuple[int, int]:
    if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float64 and x.dim() == 2 and x.is_contiguous()
            and x.shape[1] in PROBE_DIMS):
        raise ValueError(f"{what} must be a contiguous CUDA float64 [n, d] tensor, d = {probe_widths()}")
    return int(x.shape[0]), int(x.shape[1])


@torch.no_grad()
def sgd_fit_f64(x: torch.Tensor, class_ids, n_classes: int, problems, sigma, max_iter: int = 10000,
                tol: float = 1e-3, n_iter_no_change: int = 5):
    """``sgd_fit`` in scikit-learn's 64-bit instantiation (``plip_sgd_fit_f64``), the one it runs on float16 and
    float64 input: ``x`` CUDA float64 ``[n, d]`` (widen float16 exactly first), the other arguments as ``sgd_fit``.
    Returns device tensors ``(coef f64 [P, d], intercept f64 [P], n_iter int32 [P], overflow int32 [P])``."""
    n, d = _device_embeddings_f64(x, "x")
    cls = np.ascontiguousarray(np.asarray(class_ids), dtype=np.int32)
    sig = np.ascontiguousarray(np.asarray(sigma), dtype=np.int32)
    if cls.shape != (n,) or sig.ndim != 2 or sig.shape[1] != n:
        raise ValueError(f"class ids {cls.shape} and sigma {sig.shape} do not match n = {n}")
    table = (_SgdProblem * len(problems))(*[_SgdProblem(float(a), float(wp), float(wn), int(pc), int(si))
                                            for a, pc, wp, wn, si in problems])
    p = len(problems)
    L = lib()
    need = C.c_uint64(0)
    _check_args(L.plip_sgd_workspace_bytes(n, int(sig.shape[0]), p, C.byref(need)), "plip_sgd_workspace_bytes")
    dev = x.device
    ws = torch.empty(int(need.value), dtype=torch.uint8, device=dev)
    coef = torch.empty(p, d, dtype=torch.float64, device=dev)
    intercept = torch.empty(p, dtype=torch.float64, device=dev)
    n_iter = torch.empty(p, dtype=torch.int32, device=dev)
    overflow = torch.empty(p, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _check_args(L.plip_sgd_fit_f64(x.data_ptr(), n, d, cls.ctypes.data, int(n_classes), table, p, sig.ctypes.data,
                                       int(sig.shape[0]), int(max_iter), C.c_double(tol), int(n_iter_no_change),
                                       coef.data_ptr(), intercept.data_ptr(), n_iter.data_ptr(), overflow.data_ptr(),
                                       ws.data_ptr(), ws.numel(), torch.cuda.current_stream(dev).cuda_stream),
                    "plip_sgd_fit_f64")
    return coef, intercept, n_iter, overflow


@torch.no_grad()
def linear_decision_f64(x: torch.Tensor, coef: torch.Tensor, intercept: torch.Tensor):
    """``linear_decision`` in float64 (``plip_linear_decision_f64``): ``x`` CUDA float64 ``[n, d]``, ``coef`` float64
    ``[C, d]``, ``intercept`` ``[C]`` on the same device.  Returns ``(scores f64 [n, C], pred int32 [n])``."""
    n, d = _device_embeddings_f64(x, "x")
    c, dc = _device_embeddings_f64(coef, "coef")
    b = intercept.to(device=x.device, dtype=torch.float64).contiguous()
    if coef.device != x.device or dc != d or b.shape != (c,):
        raise ValueError(f"coef {tuple(coef.shape)} on {coef.device} and intercept {tuple(intercept.shape)} do not "
                         f"match x on {x.device}")
    scores = torch.empty(n, c, dtype=torch.float64, device=x.device)
    pred = torch.empty(n, dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device):
        _check_args(lib().plip_linear_decision_f64(x.data_ptr(), n, d, coef.data_ptr(), b.data_ptr(), c,
                                                   scores.data_ptr(), pred.data_ptr(),
                                                   torch.cuda.current_stream(x.device).cuda_stream),
                    "plip_linear_decision_f64")
    return scores, pred


class Engine:
    """One engine per CUDA device: packed bf16/fp32 weights + workspace for ``max_micro_batch``."""

    def __init__(self, state_dict: Mapping[str, torch.Tensor], device: Union[int, str, torch.device, None] = None,
                 max_micro_batch: int = 1024, operand_dtype="bf16"):
        """``operand_dtype``: 16-bit format of the GEMM / attention operands — ``"bf16"`` (default, BASELINE's dtype) or
        ``"fp16"`` (same speed, 3 more significand bits: 6-8x smaller end-to-end logits error, 65504 range; what the
        reference's OpenAI-clip flavour runs on a GPU).  Accumulation / residual stream / softmax are fp32 in both."""
        if not torch.cuda.is_available():
            raise RuntimeError("plip_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self._L = lib()
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError(f"plip_b200 runs on CUDA devices only, got {dev}")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        fmt, _ = operand_format(operand_dtype)
        self.operand_dtype = "fp16" if fmt == 1 else "bf16"
        patch = vision_patch(state_dict)                   # 32: ViT-B/32 (PLIP), 16: ViT-B/16
        blob, scale = pack_state_dict(state_dict, self.operand_dtype)
        self.logit_scale_exp = float(scale)
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            torch.cuda.init()
            check(self._L.plip_create_patch(blob.data_ptr(), blob.numel(), C.c_float(scale), self.device.index,
                                            int(max_micro_batch), fmt, patch, C.byref(h)), "plip_create_patch")
        self._h = h
        self.max_micro_batch = int(max_micro_batch)
        self.vision_patch = int(self._L.plip_vision_patch(h))

    def set_text_pooling(self, no_eos_argmax: bool) -> None:
        """Captions without an eos token: pool position 0 (HF, ``eos_token_id == 49407``; default) or the first argmax
        of the ids (legacy HF configs with ``eos_token_id == 2``, OpenAI clip).  See ``plip_set_text_pooling``."""
        check(self._L.plip_set_text_pooling(self._h, int(bool(no_eos_argmax))), "plip_set_text_pooling")

    def set_last_layer_pruning(self, on: bool) -> None:
        """Embedding calls run the last encoder layer's out_proj / LayerNorm 2 / MLP on the pooled rows only (CLS, first
        eos) — same embeddings, less work; hidden-state requests are never pruned.  See ``plip_set_last_layer_pruning``."""
        check(self._L.plip_set_last_layer_pruning(self._h, int(bool(on))), "plip_set_last_layer_pruning")

    def vision_seq_len(self, height: int = IMAGE_SIZE, width: int = IMAGE_SIZE) -> int:
        """Tokens of one ``height x width`` image at this engine's patch size (50 or 197 at 224 x 224)."""
        return vision_seq_len(height, width, self.vision_patch)

    def _pixel_format(self, t, interpolate_pos_encoding: bool = False) -> int:
        return _pixel_format(t, interpolate_pos_encoding, self.vision_patch)

    @property
    def last_layer_pruning(self) -> bool:
        return bool(self._L.plip_last_layer_pruning(self._h))

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._L.plip_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- helpers ---------------------------------------------------------------------------
    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _dev(self, t: torch.Tensor) -> torch.Tensor:
        if t.device != self.device:
            t = t.to(self.device, non_blocking=True)
        return t.contiguous()

    def upload_async(self, t: torch.Tensor):
        """Start copying a host tensor to the device on the engine's copy stream; returns ``(device tensor, event)``.
        The consumer stream must ``wait_event(event)`` before the first use (pinned sources overlap with compute)."""
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        cur = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self._copy_stream):
            d = t.contiguous().to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        d.record_stream(cur)
        return d, ev

    # ---- device-tensor API -------------------------------------------------------------------
    @torch.no_grad()
    def encode_images(self, pixels: torch.Tensor, normalize: bool = False,
                      interpolate_pos_encoding: bool = False) -> torch.Tensor:
        """``get_image_features``: ``[n,3,224,224]`` f32/bf16 or ``[n,224,224,3]`` u8 -> ``[n,512]`` f32 (device).

        ``interpolate_pos_encoding=True``: any ``[n,3,H,W]`` / ``[n,H,W,3]`` with ``P <= H, W`` and at most 32 patches
        of ``P = vision_patch`` pixels per side; the position table is resized bicubically to the patch grid, as HF
        does (``plip_encode_images_hw``).  An image's ``(H // P) * (W // P) + 1`` tokens must fit the workspace's
        ``50 * max_micro_batch`` token rows."""
        fmt = self._pixel_format(pixels, interpolate_pos_encoding)
        n = int(pixels.shape[0])
        if n == 0:
            return torch.empty(0, EMBED_DIM, device=self.device)
        pixels = self._dev(pixels)
        out = torch.empty(n, EMBED_DIM, device=self.device, dtype=torch.float32)
        h, w = _pixel_hw(pixels, fmt)
        with torch.cuda.device(self.device):
            check(self._L.plip_encode_images_hw(self._h, pixels.data_ptr(), fmt, n, h, w, out.data_ptr(),
                                                int(normalize), self._stream()), "plip_encode_images_hw")
        return out

    @torch.no_grad()
    def encode_windows(self, region: torch.Tensor, origins, normalize: bool = False) -> torch.Tensor:
        """224 x 224 windows of one uint8 RGB region ``[H, W, 3]`` on this engine's device (a row-strided view is fine)
        at ``origins`` (``[n, 2]`` (row, col), host or device) -> ``[n, 512]`` f32 (device), in window order: bit for
        bit what ``encode_images`` returns for the same windows cut out as uint8 tiles, without cutting them out
        (``plip_encode_windows``)."""
        h, w, pitch = _device_region(region)
        o = check_origins(origins, h, w)
        n = int(o.shape[0])
        out = torch.empty(n, EMBED_DIM, device=self.device, dtype=torch.float32)
        if n:
            if region.device != self.device:
                raise ValueError(f"the region is on {region.device}, the engine on {self.device}")
            with torch.cuda.device(self.device):
                check(self._L.plip_encode_windows(self._h, region.data_ptr(), h, w, pitch, o.ctypes.data, n,
                                                  out.data_ptr(), int(normalize), self._stream()), "plip_encode_windows")
        return out

    def window_background_counts(self, region: torch.Tensor, origins, threshold: int = 200) -> torch.Tensor:
        """See the module-level :func:`window_background_counts`."""
        return window_background_counts(region, origins, threshold)

    @torch.no_grad()
    def encode_text(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                    normalize: bool = False, prefix_len: Optional[int] = None) -> torch.Tensor:
        """``get_text_features``: ids ``[n,<=77]`` int32/int64 (+ optional mask) -> ``[n,512]`` f32 (device).

        ``prefix_len``: process only the first ``prefix_len`` positions of every row.  Exact whenever every
        caption's first eos lies inside the prefix (causal attention); the host path (``encode_text_host``)
        finds the longest caption itself, a device caller can pass it to avoid a sync."""
        n, s = _check_ids(input_ids, attention_mask)
        p_len = s if prefix_len is None else int(prefix_len)
        if not 1 <= p_len <= s:
            raise ValueError(f"prefix_len {p_len} out of [1, {s}]")
        if n == 0:
            return torch.empty(0, EMBED_DIM, device=self.device)
        idt = _ids_dtype(input_ids.dtype)
        ids = self._dev(input_ids)
        mask = None
        if attention_mask is not None:
            mask = self._dev(attention_mask.to(input_ids.dtype))
        out = torch.empty(n, EMBED_DIM, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(self._L.plip_encode_text_prefix(self._h, ids.data_ptr(), idt,
                                                  mask.data_ptr() if mask is not None else None, n, s, p_len,
                                                  out.data_ptr(), int(normalize), self._stream()), "plip_encode_text")
        return out

    @torch.no_grad()
    def encode_pair(self, pixels: torch.Tensor, input_ids: torch.Tensor,
                    attention_mask: Optional[torch.Tensor] = None, normalize: bool = True):
        """``(encode_images(pixels), encode_text(input_ids, attention_mask))`` for 224 x 224 images, bit for bit
        (``plip_encode_pair``): when each side fits one micro-batch, the text tower runs on the engine's own stream at
        the same time as the vision tower, each filling the SMs the other leaves idle.  Needs a second, text-only
        workspace (about 0.9 GB at ``max_micro_batch`` 1024), allocated on the first such call."""
        fmt = self._pixel_format(pixels)
        n_img = int(pixels.shape[0])
        n_txt, s = _check_ids(input_ids, attention_mask)
        if n_img == 0 or n_txt == 0:
            return (self.encode_images(pixels, normalize=normalize),
                    self.encode_text(input_ids, attention_mask, normalize=normalize))
        pixels = self._dev(pixels)
        ids = self._dev(input_ids)
        mask = None if attention_mask is None else self._dev(attention_mask.to(input_ids.dtype))
        img = torch.empty(n_img, EMBED_DIM, device=self.device, dtype=torch.float32)
        txt = torch.empty(n_txt, EMBED_DIM, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(self._L.plip_encode_pair(self._h, pixels.data_ptr(), fmt, n_img, ids.data_ptr(),
                                           _ids_dtype(input_ids.dtype), mask.data_ptr() if mask is not None else None,
                                           n_txt, s, img.data_ptr(), txt.data_ptr(), int(normalize), self._stream()),
                  "plip_encode_pair")
        return img, txt

    @torch.no_grad()
    def similarity(self, image_embeds: torch.Tensor, text_embeds: torch.Tensor, scale: Optional[float] = None,
                   normalize_image: bool = True, normalize_text: bool = True) -> torch.Tensor:
        """``logits_per_image[n,m] = scale * norm(image) @ norm(text).T`` (TF:923-930), fp32."""
        a = self._dev(image_embeds.to(torch.float32))
        b = self._dev(text_embeds.to(torch.float32))
        if a.shape[-1] != EMBED_DIM or b.shape[-1] != EMBED_DIM:
            raise ValueError("embeddings must have 512 columns")
        n, m = int(a.shape[0]), int(b.shape[0])
        ld = (m + 127) // 128 * 128          # the tensor-core path writes whole 128-column tiles
        out = torch.empty(n, ld, device=self.device, dtype=torch.float32)
        if n == 0 or m == 0:
            return out[:, :m]
        s = self.logit_scale_exp if scale is None else float(scale)
        with torch.cuda.device(self.device):
            check(self._L.plip_similarity(a.data_ptr(), n, b.data_ptr(), m, C.c_float(s), int(normalize_image),
                                          int(normalize_text), out.data_ptr(), ld, self._stream()), "plip_similarity")
        return out[:, :m]

    @torch.no_grad()
    def similarity_topk(self, query: torch.Tensor, space: torch.Tensor, k: int, scale: float = 1.0,
                        normalize_query: bool = True, normalize_space: bool = False):
        """Fused scores + top-k over ``space`` rows: returns ``(idx int32 [n,k], val f32 [n,k])``, descending."""
        return similarity_topk(query, space, k, scale, normalize_query, normalize_space, device=self.device)

    @torch.no_grad()
    def l2_normalize_(self, x: torch.Tensor) -> torch.Tensor:
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        if x.shape[0]:
            with torch.cuda.device(self.device):
                check(self._L.plip_l2_normalize(x.data_ptr(), int(x.shape[0]), int(x.shape[1]), self._stream()),
                      "plip_l2_normalize")
        return x

    @torch.no_grad()
    def resize_crop(self, src: torch.Tensor, descs: np.ndarray, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Packed RGB uint8 images on the device + host descriptors (``preprocess.pack_rgb``) -> uint8 tiles
        ``[n,224,224,3]``; Pillow-exact bicubic resize and crop (``plip_resize_crop_u8``)."""
        return resize_crop(src, descs, out)

    # ---- per-token outputs (output_hidden_states / output_attentions) ----------------------------------------------
    def _outputs(self, n: int, S: int, D: int, heads: int, output_hidden_states: bool, output_attentions: bool,
                 last_hidden_from_hidden: bool):
        """Allocate the buffers of one outputs call; returns ``(ctypes struct, dict of tensors)``."""
        from ._lib import TowerOutputs
        f32 = dict(device=self.device, dtype=torch.float32)
        out = {"embeds": torch.empty(n, EMBED_DIM, **f32), "pooler_output": torch.empty(n, D, **f32),
               "hidden": torch.empty(NUM_LAYERS + 1, n, S, D, **f32) if output_hidden_states else None,
               "attn": torch.empty(NUM_LAYERS, n, heads, S, S, **f32) if output_attentions else None}
        if last_hidden_from_hidden and out["hidden"] is not None:
            out["last_hidden_state"] = out["hidden"][NUM_LAYERS]
        else:
            out["last_hidden_state"] = torch.empty(n, S, D, **f32)
        own_last = out["hidden"] is None or not last_hidden_from_hidden
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        st = TowerOutputs(ptr(out["embeds"]), ptr(out["pooler_output"]),
                          ptr(out["last_hidden_state"]) if own_last else None, ptr(out["hidden"]), ptr(out["attn"]), 0)
        return st, out

    @staticmethod
    def _outputs_result(out) -> Dict[str, object]:
        hid, att = out.pop("hidden"), out.pop("attn")
        out["hidden_states"] = tuple(hid.unbind(0)) if hid is not None else None
        out["attentions"] = tuple(att.unbind(0)) if att is not None else None
        return out

    @torch.no_grad()
    def vision_outputs(self, pixels: torch.Tensor, output_hidden_states: bool = False, output_attentions: bool = False,
                       interpolate_pos_encoding: bool = False, normalize: bool = False) -> Dict[str, object]:
        """One vision tower pass that returns, as fp32 device tensors (``plip_vision_outputs``):

        - ``embeds`` ``[n,512]``: what ``encode_images`` returns (L2-normalised with ``normalize``), bit for bit;
        - ``pooler_output`` ``[n,768]``: ``post_layernorm`` of the CLS row, not projected;
        - ``last_hidden_state`` ``[n,S,768]``: the residual stream after the last layer, before ``post_layernorm``;
        - ``hidden_states``: 13 views ``[n,S,768]`` of one ``[13,n,S,768]`` tensor (``output_hidden_states``):
          ``[0]`` after ``pre_layrnorm``, ``[l]`` after layer ``l``; ``last_hidden_state`` is then ``hidden_states[12]``;
        - ``attentions``: 12 views ``[n,12,S,S]`` of one ``[12,n,12,S,S]`` tensor (``output_attentions``).

        ``S = self.vision_seq_len(H, W)`` (50 at 224 x 224, 197 on ViT-B/16).  The attentions take
        ``12 * 12 * S^2 * 4`` bytes per image (1.4 MB at 224 x 224, 605 MB at 1025 tokens)."""
        fmt = self._pixel_format(pixels, interpolate_pos_encoding)
        h, w = _pixel_hw(pixels, fmt)
        n, S = int(pixels.shape[0]), self.vision_seq_len(h, w)
        st, out = self._outputs(n, S, VISION_DIM, VISION_HEADS, output_hidden_states, output_attentions, True)
        st.normalize = int(bool(normalize))
        if n:
            pixels = self._dev(pixels)
            with torch.cuda.device(self.device):
                check(self._L.plip_vision_outputs(self._h, pixels.data_ptr(), fmt, n, h, w, C.byref(st),
                                                  self._stream()), "plip_vision_outputs")
        return self._outputs_result(out)

    @torch.no_grad()
    def text_outputs(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                     output_hidden_states: bool = False, output_attentions: bool = False,
                     normalize: bool = False) -> Dict[str, object]:
        """One text tower pass over all ``seq_len`` positions (``plip_text_outputs``); the keys of ``vision_outputs``:
        ``embeds`` (``encode_text``'s result, bit for bit), ``pooler_output`` ``[n,512]`` (the pooled row of
        ``last_hidden_state``), ``last_hidden_state`` ``[n,S,512]`` (``final_layer_norm`` of every row),
        ``hidden_states`` (13 x ``[n,S,512]``, ``[0]`` = token + position embeddings) and ``attentions``
        (12 x ``[n,8,S,S]``; masked keys are 0, a row with no visible key is all zeros)."""
        n, s = _check_ids(input_ids, attention_mask)
        idt = _ids_dtype(input_ids.dtype)
        st, out = self._outputs(n, s, TEXT_DIM, TEXT_HEADS, output_hidden_states, output_attentions, False)
        st.normalize = int(bool(normalize))
        if n:
            ids = self._dev(input_ids)
            mask = self._dev(attention_mask.to(input_ids.dtype)) if attention_mask is not None else None
            with torch.cuda.device(self.device):
                check(self._L.plip_text_outputs(self._h, ids.data_ptr(), idt,
                                                mask.data_ptr() if mask is not None else None, n, s, C.byref(st),
                                                self._stream()), "plip_text_outputs")
        return self._outputs_result(out)

    # ---- host-buffer API (copies inside the call) ------------------------------------------------
    def encode_images_host(self, pixels: Union[np.ndarray, torch.Tensor], normalize: bool = False,
                           out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Host array in, host ``[n,512]`` f32 tensor out; H2D/D2H pipelined inside the C call."""
        fmt = self._pixel_format(pixels)
        t = torch.from_numpy(np.ascontiguousarray(pixels)) if isinstance(pixels, np.ndarray) else pixels.contiguous()
        assert not t.is_cuda, "encode_images_host takes host memory; use encode_images for device tensors"
        n = int(t.shape[0])
        if out is None:
            out = torch.empty(n, EMBED_DIM, dtype=torch.float32)
        if n:
            check(self._L.plip_encode_images_host(self._h, t.data_ptr(), fmt, n, out.data_ptr(), int(normalize)),
                  "plip_encode_images_host")
        return out

    def encode_text_host(self, input_ids: Union[np.ndarray, torch.Tensor], attention_mask=None,
                         normalize: bool = False, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        ids = torch.from_numpy(np.ascontiguousarray(input_ids)) if isinstance(input_ids, np.ndarray) else input_ids.contiguous()
        n, s = _check_ids(ids, attention_mask)
        idt = _ids_dtype(ids.dtype)
        mask = None
        if attention_mask is not None:
            mask = (torch.from_numpy(np.ascontiguousarray(attention_mask)) if isinstance(attention_mask, np.ndarray)
                    else attention_mask).to(ids.dtype).contiguous()
        if out is None:
            out = torch.empty(n, EMBED_DIM, dtype=torch.float32)
        if n:
            check(self._L.plip_encode_text_host(self._h, ids.data_ptr(), idt, mask.data_ptr() if mask is not None else None,
                                                n, s, out.data_ptr(), int(normalize)), "plip_encode_text_host")
        return out

    # ---- in-step kernel timing (bench.py) ------------------------------------------------------
    def profile(self, on: bool) -> None:
        """Bracket every kernel launch of the following tower calls with CUDA events (``plip_profile_enable``)."""
        check(self._L.plip_profile_enable(self._h, int(bool(on))), "plip_profile_enable")

    def profile_read(self):
        """Rows ``{name, launches, total_ms, flops, bytes}`` aggregated per (tower, kernel role) since ``profile(True)``."""
        from ._lib import KernelTime
        buf = (KernelTime * 64)()
        cnt = C.c_int(0)
        check(self._L.plip_profile_read(self._h, buf, 64, C.byref(cnt)), "plip_profile_read")
        return [{"name": buf[i].name.decode(), "launches": int(buf[i].launches), "total_ms": float(buf[i].total_ms),
                 "flops": float(buf[i].flops), "bytes": float(buf[i].bytes)} for i in range(min(cnt.value, 64))]

    # ---- test hook ---------------------------------------------------------------------------
    @torch.no_grad()
    def hidden_states(self, tower: str, inputs: torch.Tensor, num_layers: int,
                      attention_mask: Optional[torch.Tensor] = None,
                      interpolate_pos_encoding: bool = False) -> torch.Tensor:
        """Residual stream after ``num_layers`` encoder layers (fp32), for layer-wise parity tests.  Vision with
        ``interpolate_pos_encoding``: any accepted image size, ``[n, S, 768]`` with ``S = self.vision_seq_len(H, W)``."""
        x = self._dev(inputs)
        n = int(x.shape[0])
        if tower == "vision":
            fmt = self._pixel_format(x, interpolate_pos_encoding)
            h, w = _pixel_hw(x, fmt)
            out = torch.empty((n, self.vision_seq_len(h, w), 768), device=self.device, dtype=torch.float32)
            with torch.cuda.device(self.device):
                check(self._L.plip_dbg_hidden_states_hw(self._h, x.data_ptr(), fmt, n, h, w, int(num_layers),
                                                        out.data_ptr(), self._stream()), "plip_dbg_hidden_states_hw")
            return out
        assert x.shape[1] == 77
        mask = self._dev(attention_mask.to(x.dtype)) if attention_mask is not None else None
        out = torch.empty((n, 77, 512), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(self._L.plip_dbg_hidden_states(self._h, 1, x.data_ptr(), _ids_dtype(x.dtype),
                                                 mask.data_ptr() if mask is not None else None, n, int(num_layers),
                                                 out.data_ptr(), self._stream()), "plip_dbg_hidden_states")
        return out
