"""Slide regions on the GPU: the reference's crop grid and background filter, windows read straight from the region.

The reference tiles a field of view in its data pipeline
(``reproducibility/generate_validation_datasets/preprocess/preprocess_DigestPath.py:28-100``, ``random_crop`` /
``background_ratio``): 224-px windows on a grid with ``crop_overlap`` overlap, windows whose tissue ratio (share of
pixels not all-channels ``>= 200``) is below ``non_bg_threshold`` dropped, the rest kept with their tissue ratio.
:func:`encode_region` does the same with the counting and the encoding on the device: the background kernel counts
every grid window in place, and ``Engine.encode_windows`` encodes the kept ones without cutting crops out.  With
``downsample = 1`` (the reference's resize is then an identity) origins, tissue ratios and the kept set are the
reference's exactly.

The reference runs that loop at ``downsample_list = [2, 4, 8, 16, 32]`` (``preprocess_DigestPath.py:219``): each
level is the whole image resized with Pillow's bicubic filter, and a tumour mask resized with NEAREST gives every kept
window a ``tumor_to_patch_ratio`` and a ``tumor_to_tissue_ratio``.  :func:`encode_region_pyramid` does that with the
resize on the device (``engine.resize_region``, bit-identical to Pillow), so levels, origins and all three ratios are
the reference's exactly.  A host region crosses PCIe once for all levels, in bands.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .engine import (WINDOW, Engine, ResizeWorkspace, _packed_u8, check_region, resize_filter_bounds, resize_region,
                     resize_rows, window_background_counts, window_mask_counts)

WINDOW_PIXELS = WINDOW * WINDOW
BAND_BYTES = 1 << 28  # host regions: pixels uploaded per band (two bands are in flight)
DOWNSAMPLE_LIST = (2, 4, 8, 16, 32)  # the reference's levels (preprocess_DigestPath.py:219)
MASK_THRESHOLD = 10  # the reference's mask binarisation, msk_np > 10 (preprocess_DigestPath.py:58-62)


class WindowGrid(NamedTuple):
    """Origins ``[n, 2]`` int32 (row, col) in row-major order (rows outer), and the row / column starts they combine."""
    origins: np.ndarray
    row_starts: np.ndarray
    col_starts: np.ndarray


def _starts(dim: int, crop_overlap: float) -> np.ndarray:
    # the reference's start list, then its `x2 >= shape` skip: a window that ends exactly on the border is dropped too
    s = np.arange(0, dim, WINDOW * (1 - crop_overlap)).astype(int)
    return s[s + WINDOW < dim].astype(np.int64)


def window_grid(height: int, width: int, crop_overlap: float = 0.1) -> WindowGrid:
    """The reference's window grid over a ``height x width`` region.

    Starts per axis are ``np.arange(0, dim, 224 * (1 - crop_overlap)).astype(int)``, and a window is dropped when its
    end is ``>=`` the region's size, as the reference does: a window ending exactly on the last row or column is
    dropped, so a 224 x 224 region has no window and a 225 x 225 one has one.  This is kept as is so that the crops
    match the reference's; callers who want another grid pass their own origins to ``Engine.encode_windows``.
    The reference's ``x`` is axis 0 (rows), so the order is rows outer, columns inner."""
    if not crop_overlap < 1:
        raise ValueError(f"crop_overlap must be < 1 (the grid step is 224 * (1 - crop_overlap)), got {crop_overlap}")
    rows, cols = _starts(int(height), crop_overlap), _starts(int(width), crop_overlap)
    rr, cc = np.meshgrid(rows, cols, indexing="ij")
    origins = np.stack([rr.ravel(), cc.ravel()], axis=1).astype(np.int32).reshape(-1, 2)
    return WindowGrid(origins, rows, cols)


def keep_windows(counts: np.ndarray, non_bg_threshold: float = 0.5) -> Tuple[np.ndarray, np.ndarray]:
    """``(keep, tissue_ratio)`` from per-window background pixel counts: the reference's ``1 - count / 50176`` in float64
    and its ``tissue_ratio < non_bg_threshold`` skip, so the decision is the reference's bit for bit."""
    tissue = 1 - np.asarray(counts, dtype=np.int64) / WINDOW_PIXELS
    return ~(tissue < non_bg_threshold), tissue


def plan_bands(row_starts: np.ndarray, width: int, budget: int = BAND_BYTES) -> List[Tuple[int, int]]:
    """Host regions are uploaded in horizontal bands of whole window rows: ``[(i0, i1)]`` ranges of ``row_starts``,
    each band's pixel rows ``row_starts[i0] .. row_starts[i1 - 1] + 224`` at most ``budget`` bytes (at least one
    window row per band)."""
    bands, i0, n = [], 0, len(row_starts)
    row_bytes = 3 * int(width)
    while i0 < n:
        i1 = i0 + 1
        while i1 < n and (int(row_starts[i1]) + WINDOW - int(row_starts[i0])) * row_bytes <= budget:
            i1 += 1
        bands.append((i0, i1))
        i0 = i1
    return bands


@dataclass
class RegionEncoding:
    """What :func:`encode_region` returns.  ``embeddings`` ``[k, 512]`` f32 (device) of the kept windows, in grid order;
    ``origins`` ``[k, 2]`` int32 (row, col); ``tissue_ratio`` ``[k]`` float64; ``row_starts`` / ``col_starts`` the
    grid's; ``grid_index`` ``[k]``: window ``i`` sits at grid cell ``divmod(grid_index[i], len(col_starts))``.
    ``downsample`` and ``level_size`` ``(height, width)`` name the level the origins refer to; ``tumor_to_patch_ratio`` /
    ``tumor_to_tissue_ratio`` ``[k]`` float64 are the reference's (zeros without a mask)."""
    engine: Engine
    embeddings: torch.Tensor
    origins: np.ndarray
    tissue_ratio: np.ndarray
    row_starts: np.ndarray
    col_starts: np.ndarray
    grid_index: np.ndarray
    downsample: float = 1
    level_size: Optional[Tuple[int, int]] = None
    tumor_to_patch_ratio: Optional[np.ndarray] = None
    tumor_to_tissue_ratio: Optional[np.ndarray] = None

    @torch.no_grad()
    def score_map(self, text_embeds: torch.Tensor) -> torch.Tensor:
        """Cosine score of every kept window against ``P`` text embeddings: ``[P, n_rows, n_cols]`` float32 on the
        engine's device, NaN at grid cells whose window was dropped (``Engine.similarity`` with scale 1)."""
        p = int(text_embeds.shape[0])
        nr, nc = len(self.row_starts), len(self.col_starts)
        out = torch.full((p, nr * nc), float("nan"), device=self.engine.device, dtype=torch.float32)
        if len(self.grid_index) and p:
            s = self.engine.similarity(self.embeddings, text_embeds, scale=1.0)  # [k, P]
            idx = torch.as_tensor(self.grid_index, dtype=torch.int64).to(out.device)
            out[:, idx] = s.t().to(out.device)
        return out.view(p, nr, nc)


def _as_host_array(region) -> np.ndarray:
    if torch.is_tensor(region):
        return region.numpy()
    return np.asarray(region)


@torch.no_grad()
def encode_region(engine: Engine, region: Union[torch.Tensor, np.ndarray], crop_overlap: float = 0.1,
                  non_bg_threshold: float = 0.5, bg_threshold: int = 200, normalize: bool = False,
                  band_bytes: int = BAND_BYTES, downsample: float = 1, mask=None,
                  mask_threshold: int = MASK_THRESHOLD) -> RegionEncoding:
    """The reference's ``random_crop`` on the GPU: the :func:`window_grid` of the region, the background count of every
    window on the device, the :func:`keep_windows` decision on the host, and ``Engine.encode_windows`` on the kept
    windows.

    ``region``: uint8 RGB ``[H, W, 3]``.  A CUDA tensor (packed pixels, rows may be strided) is read in place.  A host
    array (numpy or CPU tensor, any strides) is streamed in horizontal bands of whole window rows of at most
    ``band_bytes``, each uploaded once through pinned memory while the previous band is computed; its embeddings can
    differ from the device path's in the last bits, since a band changes the micro-batches the windows share.

    ``downsample != 1``: the region is first resized to :func:`level_size` on the device, bit-identical to Pillow's
    ``img.resize(new_size)``, and the grid runs on that level (:func:`encode_region_pyramid` with one level; host and
    device regions then give the same bits).  A level under 224 px in either dimension gives an empty result.
    ``mask``: a uint8 ``[h, w]`` or ``[h, w, 3]`` tumour mask (host or CUDA), resized with Pillow's NEAREST rule to the
    level's size (:func:`nearest_index`); each kept window then gets the reference's tumour ratios from the count of
    its mask elements ``> mask_threshold``."""
    if downsample != 1:
        return encode_region_pyramid(engine, region, mask, [downsample], crop_overlap, non_bg_threshold, bg_threshold,
                                     mask_threshold, normalize, band_bytes)[0]
    on_device = torch.is_tensor(region) and region.is_cuda
    if not on_device:
        region = _as_host_array(region)
    h, w, _ = check_region(region) if on_device else _check_host_region(region)
    if mask is not None:
        _check_mask(mask)
    grid = window_grid(h, w, crop_overlap)
    if on_device:
        counts = window_background_counts(region, grid.origins, bg_threshold).cpu().numpy()
        keep, tissue = keep_windows(counts, non_bg_threshold)
        emb = engine.encode_windows(region, grid.origins[keep], normalize=normalize)
    else:
        keep, tissue, emb = _encode_host_region(engine, region, grid, non_bg_threshold, bg_threshold, normalize,
                                                band_bytes)
    origins = grid.origins[keep]
    counts = None if mask is None else _mask_counts(engine, mask, h, w, origins, mask_threshold)
    return RegionEncoding(engine, emb, origins, tissue[keep], grid.row_starts, grid.col_starts, np.flatnonzero(keep),
                          downsample, (h, w), *tumor_ratios(counts, tissue[keep]))


def level_size(h: int, w: int, downsample: float) -> Tuple[int, int]:
    """``(height, width)`` of the reference's level: ``new_size = (int(np.round(W / ds)), int(np.round(H / ds)))``
    (Pillow's ``(width, height)``); ``np.round`` rounds halves to even, so 4999 and 5001 both give 2500 at ``ds = 2``."""
    return int(np.round(h / downsample)), int(np.round(w / downsample))


def nearest_index(in_size: int, out_size: int) -> np.ndarray:
    """The source index of every output index of Pillow's NEAREST resize along one axis: ``int(x)`` of the running sum
    ``x = a * 0.5, x += a`` with ``a = in_size / out_size`` in double, as Pillow's ``ImagingScaleAffine`` steps it (not
    ``int((i + 0.5) * a)``, which differs for some sizes).  int64 ``[out_size]``."""
    a = in_size / out_size
    steps = np.full(out_size, a)
    steps[0] = a * 0.5
    return np.minimum(np.cumsum(steps).astype(np.int64), in_size - 1)   # cumsum adds in order, as Pillow does


def tumor_ratios(counts: Optional[np.ndarray], tissue: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """The reference's ``tumor_to_patch_ratio = count / (224 * 224)`` and ``tumor_to_tissue_ratio = count / (224 * 224
    * tissue_ratio)`` in float64, in its operation order; zeros without a mask (``counts is None``), as it sets them.
    The denominator is 224 * 224 whatever the mask's channel count, so an RGB mask (every channel counted) can give a
    ratio above 1, as in the reference."""
    if counts is None:
        return np.zeros(len(tissue)), np.zeros(len(tissue))
    c = np.asarray(counts, dtype=np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):   # tissue 0 only if non_bg_threshold <= 0: inf / nan as there
        return c / WINDOW_PIXELS, c / (WINDOW_PIXELS * np.asarray(tissue, dtype=np.float64))


def _check_mask(mask) -> None:
    if torch.is_tensor(mask) and mask.is_cuda:
        _packed_u8(mask, "a mask", (1, 3))
        return
    m = _as_host_array(mask)
    if m.dtype != np.uint8 or m.ndim not in (2, 3) or (m.ndim == 3 and m.shape[2] != 3) or 0 in m.shape[:2]:
        raise ValueError(f"a mask must be uint8 [H, W] or [H, W, 3], got {m.dtype} {m.shape}")


def level_mask(mask, height: int, width: int):
    """``mask`` resized to ``height x width`` with Pillow's NEAREST rule (:func:`nearest_index` per axis), from the
    mask's own size even where it differs from the image's, as the reference does.  A CUDA mask is gathered on its
    device, a host mask (numpy or CPU tensor) with numpy; a mask already at that size is returned as it is."""
    if tuple(mask.shape[:2]) == (height, width):
        return mask
    rows, cols = nearest_index(int(mask.shape[0]), height), nearest_index(int(mask.shape[1]), width)
    if torch.is_tensor(mask) and mask.is_cuda:
        r, c = (torch.from_numpy(x).to(mask.device) for x in (rows, cols))
        return mask.index_select(0, r).index_select(1, c)
    return np.ascontiguousarray(_as_host_array(mask)[rows][:, cols])


def _mask_counts(engine: Engine, mask, height: int, width: int, origins: np.ndarray, threshold: int) -> np.ndarray:
    """Per window at ``origins`` of a ``height x width`` level, the level mask's elements ``> threshold``, counted on
    the device (a host mask is gathered to the level's size first, then uploaded)."""
    m = level_mask(mask, height, width)
    if not (torch.is_tensor(m) and m.is_cuda):
        m = torch.from_numpy(np.ascontiguousarray(_as_host_array(m))).to(engine.device)
    return window_mask_counts(m, origins, threshold).cpu().numpy()


@torch.no_grad()
def encode_region_pyramid(engine: Engine, region: Union[torch.Tensor, np.ndarray], mask=None,
                          downsample_list: Sequence[float] = DOWNSAMPLE_LIST, crop_overlap: float = 0.1,
                          non_bg_threshold: float = 0.5, bg_threshold: int = 200,
                          mask_threshold: int = MASK_THRESHOLD, normalize: bool = False,
                          band_bytes: int = BAND_BYTES) -> List[RegionEncoding]:
    """The reference's step 1 for one image (``preprocess_DigestPath.py:117-140``): ``random_crop`` at every
    ``downsample`` of ``downsample_list``, one :class:`RegionEncoding` per level in list order.  A level under 224 px in
    either dimension, or one with no kept window, gives an empty encoding (the reference's ``None``), not a missing one.

    Each level is the region resized to :func:`level_size` on the device (``resize_region``: Pillow's bicubic, bit for
    bit), then counted, kept and encoded in place as a device region; the mask is resized per level with
    :func:`level_mask`.  A CUDA region is resized whole for each level.  A host region is uploaded once for all levels
    in bands of at most ``band_bytes`` (never less than the tallest vertical filter window), through the pinned double
    buffer of :func:`encode_region`; consecutive bands share the rows of that window.  Each band produces every level's
    output rows whose filter window it holds (:func:`plan_pyramid_bands`), so host and device regions give the same
    levels and the same embeddings, bit for bit."""
    on_device = torch.is_tensor(region) and region.is_cuda
    if not on_device:
        region = _as_host_array(region)
    h, w = _packed_u8(region, "a region", (3,))[:2] if on_device else _check_host_region(region, 1)[:2]
    if mask is not None:
        _check_mask(mask)
    window_grid(0, 0, crop_overlap)   # rejects a crop_overlap >= 1 before any work
    levels = []
    for ds in downsample_list:
        if not (np.isfinite(ds) and ds > 0):
            raise ValueError(f"downsample must be a positive number, got {ds}")
        levels.append((ds,) + level_size(h, w, ds))
    active = [i for i, (_, lh, lw) in enumerate(levels) if lh >= WINDOW and lw >= WINDOW]
    images = {}
    if not on_device:
        images = dict(zip(active, _resize_host_levels(engine, region, [levels[i][1:] for i in active], band_bytes)))
    out = []
    for i, (ds, lh, lw) in enumerate(levels):
        level = None
        if i in active:
            level = images.pop(i) if not on_device else resize_region(region, lh, lw)
        out.append(_encode_level(engine, level, ds, lh, lw, mask, crop_overlap, non_bg_threshold, bg_threshold,
                                 mask_threshold, normalize))
    return out


def _encode_level(engine: Engine, level: Optional[torch.Tensor], ds: float, lh: int, lw: int, mask, crop_overlap: float,
                  non_bg_threshold: float, bg_threshold: int, mask_threshold: int, normalize: bool) -> RegionEncoding:
    """One level of :func:`encode_region_pyramid`: ``level`` is the ``lh x lw`` device image, or None when it is under
    one window (its grid is then empty too)."""
    grid = window_grid(lh, lw, crop_overlap)
    keep, tissue = np.zeros(len(grid.origins), bool), np.zeros(len(grid.origins))
    if level is not None and len(grid.origins):
        keep, tissue = keep_windows(window_background_counts(level, grid.origins, bg_threshold).cpu().numpy(),
                                    non_bg_threshold)
    origins = grid.origins[keep]
    if len(origins):
        emb = engine.encode_windows(level, origins, normalize=normalize)
    else:
        emb = torch.empty(0, 512, device=engine.device)
    counts = None
    if mask is not None:
        counts = _mask_counts(engine, mask, lh, lw, origins, mask_threshold) if len(origins) else np.zeros(0, np.int64)
    return RegionEncoding(engine, emb, origins, tissue[keep], grid.row_starts, grid.col_starts, np.flatnonzero(keep),
                          ds, (lh, lw), *tumor_ratios(counts, tissue[keep]))


def plan_pyramid_bands(bounds: Sequence[np.ndarray], height: int, row_bytes: int,
                       budget: int = BAND_BYTES) -> List[Tuple[int, int, List[Tuple[int, int]]]]:
    """Source bands of a host region for several levels at once: ``[(r0, r1, [(o0, o1) per level])]``.

    ``bounds[l]`` is level ``l``'s vertical filter windows, int ``[new_h, 2]`` (first source row, count), from the
    library (``engine.resize_filter_bounds``).  A band holds at most ``budget`` bytes of ``row_bytes`` rows, but never
    fewer rows than the tallest window.  Each band produces, per level, the next output rows whose whole window lies
    in it; the next band starts at the first row a pending output row still needs, so consecutive bands overlap by
    less than one window and every output row is produced exactly once."""
    win = max(int(b[:, 1].max()) for b in bounds)
    cap = max(int(budget) // int(row_bytes), win)
    ends = [b[:, 0].astype(np.int64) + b[:, 1] for b in bounds]
    nxt = [0] * len(bounds)
    bands, r0 = [], 0
    while any(nxt[i] < len(b) for i, b in enumerate(bounds)):
        r1 = min(height, r0 + cap)
        ranges = []
        for i in range(len(bounds)):
            o1 = max(nxt[i], int(np.searchsorted(ends[i], r1, side="right")))
            ranges.append((nxt[i], o1))
            nxt[i] = o1
        bands.append((r0, r1, ranges))
        pending = [int(bounds[i][nxt[i], 0]) for i in range(len(bounds)) if nxt[i] < len(bounds[i])]
        if pending:
            if min(pending) <= r0 and all(a == b for a, b in ranges):
                raise RuntimeError("band plan made no progress")   # cannot happen: cap >= every window
            r0 = min(pending)
    return bands


def _resize_host_levels(engine: Engine, region: np.ndarray, sizes: List[Tuple[int, int]],
                        band_bytes: int) -> List[torch.Tensor]:
    """Every ``(height, width)`` level of a host region on the device, from one banded upload of the region."""
    if not sizes:
        return []
    h, w = int(region.shape[0]), int(region.shape[1])
    bounds = [resize_filter_bounds(h, lh) for lh, _ in sizes]
    bands = plan_pyramid_bands(bounds, h, 3 * w, band_bytes)
    outs = [torch.empty((lh, lw, 3), dtype=torch.uint8, device=engine.device) for lh, lw in sizes]
    ws = ResizeWorkspace(engine.device)
    for (r0, _, ranges), dev in zip(bands, _upload_bands(engine, region, [(r0, r1) for r0, r1, _ in bands])):
        for (lh, lw), out, (o0, o1) in zip(sizes, outs, ranges):
            if o1 > o0:
                resize_rows(dev, r0, h, lh, lw, (o0, o1), out[o0:o1], ws)
    return outs
def _check_host_region(region: np.ndarray, min_size: int = WINDOW) -> Tuple[int, int, int]:
    if region.dtype != np.uint8 or region.ndim != 3 or region.shape[2] != 3:
        raise ValueError(f"a region must be uint8 RGB [H, W, 3], got {region.dtype} {region.shape}")
    h, w = int(region.shape[0]), int(region.shape[1])
    if h < min_size or w < min_size:
        raise ValueError(f"region {h}x{w} is smaller than one {min_size}x{min_size} window" if min_size == WINDOW
                         else f"region {h}x{w} is empty")
    return h, w, 3 * w


def _upload_bands(engine: Engine, region: np.ndarray, ranges: List[Tuple[int, int]]):
    """Yield the host row ranges ``[r0, r1)`` of ``region`` as device tensors, each uploaded once through a pinned
    double buffer: the host copy and upload of range ``k + 1`` overlap the work queued on range ``k``.  The current
    stream waits for each upload before its tensor is yielded."""
    if not ranges:
        return
    rows_max = max(r1 - r0 for r0, r1 in ranges)
    stage = [torch.empty((rows_max,) + region.shape[1:], dtype=torch.uint8, pin_memory=True)
             for _ in range(min(2, len(ranges)))]
    uploads = [None] * len(stage)  # copy event of the range each staging buffer last held

    def start(k):
        r0, r1 = ranges[k]
        b = k % len(stage)
        if uploads[b] is not None:
            uploads[b].synchronize()  # the copy out of this staging buffer is done
        buf = stage[b][:r1 - r0]
        buf.numpy()[...] = region[r0:r1]
        dev, ev = engine.upload_async(buf)
        uploads[b] = ev
        return dev, ev

    cur = torch.cuda.current_stream(engine.device)
    pending = start(0)
    for k in range(len(ranges)):
        dev, ev = pending
        cur.wait_event(ev)
        if k + 1 < len(ranges):
            pending = start(k + 1)  # host copy + upload of the next range overlap this one's compute
        yield dev


def _encode_host_region(engine: Engine, region: np.ndarray, grid: WindowGrid, non_bg_threshold: float,
                        bg_threshold: int, normalize: bool, band_bytes: int):
    n_cols = len(grid.col_starts)
    bands = plan_bands(grid.row_starts, region.shape[1], band_bytes)
    keep = np.zeros(len(grid.origins), dtype=bool)
    tissue = np.zeros(len(grid.origins), dtype=np.float64)
    embs = []
    if not bands:
        return keep, tissue, torch.empty(0, 512, device=engine.device)
    rows = [(int(grid.row_starts[i0]), int(grid.row_starts[i1 - 1]) + WINDOW) for i0, i1 in bands]
    for (i0, i1), (r0, _), dev in zip(bands, rows, _upload_bands(engine, region, rows)):
        sel = slice(i0 * n_cols, i1 * n_cols)  # the band's windows: whole grid rows
        rel = grid.origins[sel] - np.array([r0, 0], dtype=np.int32)
        counts = window_background_counts(dev, rel, bg_threshold).cpu().numpy()
        keep[sel], tissue[sel] = keep_windows(counts, non_bg_threshold)
        embs.append(engine.encode_windows(dev, rel[keep[sel]], normalize=normalize))
    return keep, tissue, torch.cat(embs)
