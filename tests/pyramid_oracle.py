"""Test oracle for region pyramids: the reference's ``random_crop``
(``reproducibility/generate_validation_datasets/preprocess/preprocess_DigestPath.py:36-108``) with ``downsample`` and a
tumour mask, through PIL's own resize, and a JPEG-like tumour mask generator.  The crop loop and ``background_ratio``
are those of ``region_oracle``.  ``plip_b200.regions.encode_region_pyramid`` is checked against it; nothing here runs
on the device."""
import numpy as np

from region_oracle import CROP, background_ratio


def random_crop(img: np.ndarray, msk=None, downsample=1, crop_overlap: float = 0.1, non_bg_threshold: float = 0.5):
    """The reference's ``random_crop`` (``preprocess_DigestPath.py:36-108``) with ``downsample`` and a mask: the image
    resized with PIL's default (BICUBIC) to ``new_size``, the mask with NEAREST from its own size, binarised ``> 10``,
    then the crop loop with the tumour ratios in the reference's expressions.  ``img`` uint8 ``[H, W, 3]``; ``msk``
    uint8 ``[h, w]`` or ``[h, w, 3]`` or None.  Returns None where the reference returns ``(None, None)``, else a dict
    ``crops [k,224,224,3]``, ``origins [(row, col)]``, ``tissue``, ``t2p``, ``t2t`` (lists of floats), ``level`` (the
    resized image)."""
    from PIL import Image
    pil = Image.fromarray(img)
    new_size = (int(np.round(pil.size[0] / downsample)), int(np.round(pil.size[1] / downsample)))
    pil = pil.resize(new_size)
    if pil.size[0] < CROP or pil.size[1] < CROP:
        return None
    img_np = np.array(pil)
    if msk is not None:
        msk_np = (np.array(Image.fromarray(msk).resize(new_size, Image.Resampling.NEAREST)) > 10).astype(int)
    step = CROP * (1 - crop_overlap)
    out = {"crops": [], "origins": [], "tissue": [], "t2p": [], "t2t": [], "level": img_np}
    for x1 in np.arange(0, img_np.shape[0], step).astype(int):
        for y1 in np.arange(0, img_np.shape[1], step).astype(int):
            x2, y2 = x1 + CROP, y1 + CROP
            if x2 >= img_np.shape[0] or y2 >= img_np.shape[1]:
                continue
            patch = img_np[x1:x2, y1:y2, :]
            tissue_ratio = 1 - background_ratio(patch)
            if tissue_ratio < non_bg_threshold:
                continue
            if msk is not None:
                mp = msk_np[x1:x2, y1:y2]
                t2p = np.sum(mp > 0) / (mp.shape[0] * mp.shape[1])
                t2t = np.sum(mp > 0) / (mp.shape[0] * mp.shape[1] * tissue_ratio)
            else:
                t2p, t2t = 0, 0
            out["crops"].append(patch)
            out["origins"].append((int(x1), int(y1)))
            out["tissue"].append(tissue_ratio)
            out["t2p"].append(t2p)
            out["t2t"].append(t2t)
    if not out["crops"]:
        return None
    out["crops"] = np.stack(out["crops"])
    return out


def tumour_mask(h: int, w: int, seed: int, rgb: bool = False) -> np.ndarray:
    """A JPEG-like tumour mask: a few bright blobs over low noise (values on both sides of the > 10 cut)."""
    g = np.random.default_rng(seed)
    m = g.integers(0, 14, (h, w), dtype=np.uint8)
    for _ in range(4):
        bh, bw = int(g.integers(h // 8, h // 2)), int(g.integers(w // 8, w // 2))
        r, c = int(g.integers(0, h - bh)), int(g.integers(0, w - bw))
        m[r:r + bh, c:c + bw] = g.integers(8, 256, (bh, bw), dtype=np.uint8)
    if rgb:
        m = np.stack([m, np.roll(m, 7, 0), np.roll(m, 11, 1)], -1)
    return m
