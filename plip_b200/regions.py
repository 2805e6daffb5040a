"""Slide regions on the GPU: the reference's crop grid and background filter, windows read straight from the region.

The reference tiles a field of view in its data pipeline
(``reproducibility/generate_validation_datasets/preprocess/preprocess_DigestPath.py:28-100``, ``random_crop`` /
``background_ratio``): 224-px windows on a grid with ``crop_overlap`` overlap, windows whose tissue ratio (share of
pixels not all-channels ``>= 200``) is below ``non_bg_threshold`` dropped, the rest kept with their tissue ratio.
:func:`encode_region` does the same with the counting and the encoding on the device: the background kernel counts
every grid window in place, and ``Engine.encode_windows`` encodes the kept ones without cutting crops out.  With
``downsample = 1`` (the reference's resize is then an identity) origins, tissue ratios and the kept set are the
reference's exactly.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, NamedTuple, Tuple, Union

import numpy as np
import torch

from .engine import WINDOW, Engine, check_region, window_background_counts

WINDOW_PIXELS = WINDOW * WINDOW
BAND_BYTES = 1 << 28  # host regions: pixels uploaded per band (two bands are in flight)


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
    grid's; ``grid_index`` ``[k]``: window ``i`` sits at grid cell ``divmod(grid_index[i], len(col_starts))``."""
    engine: Engine
    embeddings: torch.Tensor
    origins: np.ndarray
    tissue_ratio: np.ndarray
    row_starts: np.ndarray
    col_starts: np.ndarray
    grid_index: np.ndarray

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
                  band_bytes: int = BAND_BYTES) -> RegionEncoding:
    """The reference's ``random_crop`` (``downsample = 1``) on the GPU: the :func:`window_grid` of the region, the
    background count of every window on the device, the :func:`keep_windows` decision on the host, and
    ``Engine.encode_windows`` on the kept windows.

    ``region``: uint8 RGB ``[H, W, 3]``.  A CUDA tensor (packed pixels, rows may be strided) is read in place.  A host
    array (numpy or CPU tensor, any strides) is streamed in horizontal bands of whole window rows of at most
    ``band_bytes``, each uploaded once through pinned memory while the previous band is computed; its embeddings can
    differ from the device path's in the last bits, since a band changes the micro-batches the windows share."""
    on_device = torch.is_tensor(region) and region.is_cuda
    if not on_device:
        region = _as_host_array(region)
    h, w, _ = check_region(region) if on_device else _check_host_region(region)
    grid = window_grid(h, w, crop_overlap)
    if on_device:
        counts = window_background_counts(region, grid.origins, bg_threshold).cpu().numpy()
        keep, tissue = keep_windows(counts, non_bg_threshold)
        emb = engine.encode_windows(region, grid.origins[keep], normalize=normalize)
    else:
        keep, tissue, emb = _encode_host_region(engine, region, grid, non_bg_threshold, bg_threshold, normalize,
                                                band_bytes)
    return RegionEncoding(engine, emb, grid.origins[keep], tissue[keep], grid.row_starts, grid.col_starts,
                          np.flatnonzero(keep))


def _check_host_region(region: np.ndarray) -> Tuple[int, int, int]:
    if region.dtype != np.uint8 or region.ndim != 3 or region.shape[2] != 3:
        raise ValueError(f"a region must be uint8 RGB [H, W, 3], got {region.dtype} {region.shape}")
    h, w = int(region.shape[0]), int(region.shape[1])
    if h < WINDOW or w < WINDOW:
        raise ValueError(f"region {h}x{w} is smaller than one {WINDOW}x{WINDOW} window")
    return h, w, 3 * w


def _encode_host_region(engine: Engine, region: np.ndarray, grid: WindowGrid, non_bg_threshold: float,
                        bg_threshold: int, normalize: bool, band_bytes: int):
    n_cols = len(grid.col_starts)
    bands = plan_bands(grid.row_starts, region.shape[1], band_bytes)
    keep = np.zeros(len(grid.origins), dtype=bool)
    tissue = np.zeros(len(grid.origins), dtype=np.float64)
    embs = []
    if not bands:
        return keep, tissue, torch.empty(0, 512, device=engine.device)
    rows_max = max(int(grid.row_starts[i1 - 1]) + WINDOW - int(grid.row_starts[i0]) for i0, i1 in bands)
    stage = [torch.empty((rows_max,) + region.shape[1:], dtype=torch.uint8, pin_memory=True)
             for _ in range(min(2, len(bands)))]
    uploads = [None] * len(stage)  # copy event of the band each staging buffer last held

    def start(k):
        i0, i1 = bands[k]
        r0, r1 = int(grid.row_starts[i0]), int(grid.row_starts[i1 - 1]) + WINDOW
        b = k % len(stage)
        if uploads[b] is not None:
            uploads[b].synchronize()  # the copy out of this staging buffer is done
        buf = stage[b][:r1 - r0]
        buf.numpy()[...] = region[r0:r1]
        dev, ev = engine.upload_async(buf)
        uploads[b] = ev
        return dev, ev, r0

    cur = torch.cuda.current_stream(engine.device)
    pending = start(0)
    for k, (i0, i1) in enumerate(bands):
        dev, ev, r0 = pending
        cur.wait_event(ev)
        if k + 1 < len(bands):
            pending = start(k + 1)  # host copy + upload of the next band overlap this band's compute
        sel = slice(i0 * n_cols, i1 * n_cols)  # the band's windows: whole grid rows
        rel = grid.origins[sel] - np.array([r0, 0], dtype=np.int32)
        counts = window_background_counts(dev, rel, bg_threshold).cpu().numpy()
        keep[sel], tissue[sel] = keep_windows(counts, non_bg_threshold)
        embs.append(engine.encode_windows(dev, rel[keep[sel]], normalize=normalize))
    return keep, tissue, torch.cat(embs)
