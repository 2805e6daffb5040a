"""Test oracle for slide regions: the reference's crop loop and background ratio
(``reproducibility/generate_validation_datasets/preprocess/preprocess_DigestPath.py:28-100``, ``random_crop`` with
``downsample = 1`` and no mask, ``background_ratio``) restated in plain numpy, one window at a time.  The engine's
``plip_b200.regions`` is checked against it; nothing here runs on the device."""
import numpy as np

CROP = 224


def background_ratio(rgb: np.ndarray, threshold: int = 200) -> float:
    """Share of the pixels of ``rgb [h, w, 3]`` whose three channels are all ``>= threshold``."""
    bg = (rgb[..., 0] >= threshold) & (rgb[..., 1] >= threshold) & (rgb[..., 2] >= threshold)
    return np.sum(bg) / (rgb.shape[0] * rgb.shape[1])


def crops(img: np.ndarray, crop_overlap: float = 0.1, non_bg_threshold: float = 0.5):
    """The crops the reference keeps from ``img [H, W, 3]`` uint8: ``(crops [k, 224, 224, 3], origins [(row, col)],
    tissue ratios [k])``.  ``non_bg_threshold=-np.inf`` keeps every window of the grid."""
    if img.shape[0] < CROP or img.shape[1] < CROP:
        return np.zeros((0, CROP, CROP, 3), np.uint8), [], []
    step = CROP * (1 - crop_overlap)
    out, origins, tissue = [], [], []
    for r in np.arange(0, img.shape[0], step).astype(int):          # the reference's x: axis 0
        for c in np.arange(0, img.shape[1], step).astype(int):
            if r + CROP >= img.shape[0] or c + CROP >= img.shape[1]:
                continue
            patch = img[r:r + CROP, c:c + CROP, :]
            t = 1 - background_ratio(patch)
            if t < non_bg_threshold:
                continue
            out.append(patch)
            origins.append((int(r), int(c)))
            tissue.append(t)
    stacked = np.stack(out) if out else np.zeros((0, CROP, CROP, 3), np.uint8)
    return stacked, origins, tissue


def region_with_blocks(h: int, w: int, seed: int, blocks: int = 6, white: int = 230) -> np.ndarray:
    """Random tissue-like pixels with a few planted near-white (background) rectangles of random size, so that windows
    fall on both sides of the tissue threshold, some exactly at the boundary values."""
    g = np.random.default_rng(seed)
    img = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
    for _ in range(blocks):
        bh, bw = int(g.integers(50, max(51, h // 2))), int(g.integers(50, max(51, w // 2)))
        r, c = int(g.integers(0, h - min(bh, h) + 1)), int(g.integers(0, w - min(bw, w) + 1))
        img[r:r + bh, c:c + bw] = g.integers(white, 256, (min(bh, h - r), min(bw, w - c), 3), dtype=np.uint8)
    return img
