"""Evaluation datasets on the device: the reference's 224-px evaluation tiles and its PanNuke benchmark.

``reproduce.sh`` evaluates on tiles that the reference's dataset scripts wrote to disk; the embedders then read those
files, and their own ``Resize(224)`` / ``CenterCrop(224)`` does nothing to a 224 x 224 tile.  This module rebuilds
those tiles and the PanNuke table from the raw inputs, bit for bit, without writing anything:

* :func:`evaluation_tiles` — ``resizeimg`` (``generate_validation_datasets/prepare_dataset_to_csv.py:40-63``), the
  resize every evaluation image goes through.  Its arithmetic is kept as it is (:func:`resizeimg_plan`): the new size
  is ``int(side * (224 / min_side))``, which is 223 for some short sides, and the centre-crop box of a non-square image
  is computed from the ORIGINAL size, so the window can reach past the resized image, where PIL fills zeros (a
  1000 x 800 image gives an all-black tile).  RGB images run through ``plip_resize_crop_fill_u8``.
* :func:`pannuke_binary` — ``preprocess/preprocess_PanNuke.py``: drop images without cells, count the nucleus
  instances of each channel (``len(np.unique(...)) - 1``) from the per-(image, channel) value sets of
  ``plip_mask_value_sets_u8``, label malignant (``n_neoplastic >= 10 and n_neoplastic / total > 0.3``) or benign
  (``n_neoplastic == 0``), name and caption the rows, and resize the kept images to their 224 x 224 tiles.
* :func:`split_pannuke` — ``_dataset_loader.py:182-233`` ``process_PanNuke``: caption parsing, the seeded shuffle and
  the per-tissue, per-label train / test split.

Tables are dicts of columns (numpy arrays, and a CUDA uint8 ``[n,224,224,3]`` tensor under ``"tiles"``), in the
reference's row order.  Example (PanNuke's three folds, as ``np.load`` returns them)::

    folds = [(np.load(f"fold{i}/images.npy", mmap_mode="r"), np.load(f"fold{i}/masks.npy", mmap_mode="r"),
              np.load(f"fold{i}/types.npy")) for i in (1, 2, 3)]
    train, test = split_pannuke(pannuke_binary(folds), seed=1, train_ratio=0.7)
    x_train = engine.encode_images(train["tiles"], normalize=True)     # CLIPEmbedder's rows for those files
    x_test = engine.encode_images(test["tiles"], normalize=True)
    results = linear_probe_sweep(x_train, train["label"].astype(np.int64), x_test, test["label"].astype(np.int64),
                                 alphas)
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np
import PIL.Image

from .preprocess import SIZE, ImageLike, RESIZE_DESC_DTYPE, pack_rgb, resize_fits_device

# PanNuke's nucleus channels: 0 neoplastic, 1 inflammatory, 2 connective, 3 dead, 4 epithelial; 5 background.
PANNUKE_CHANNELS = 6
MASK_CHUNK = 256  # images per pinned upload of pannuke_binary


def resizeimg_plan(width: int, height: int) -> Tuple[int, int, int, int]:
    """``(new_w, new_h, left, top)`` of the reference's ``resizeimg`` for a ``width x height`` image: the resize
    ``img.resize((new_w, new_h))`` and the 224 x 224 crop at ``(left, top)`` of the resized image, with the reference's
    Python float arithmetic and the ``round()`` (half to even) that ``Image.crop`` applies to its box.  ``left`` /
    ``top`` may be negative or past the resized image.  A square image gives ``(224, 224, 0, 0)``."""
    width, height = int(width), int(height)
    if width == height:
        return SIZE, SIZE, 0, 0
    scale = SIZE / min(width, height)
    left, top = (width - SIZE) / 2, (height - SIZE) / 2
    return int(width * scale), int(height * scale), int(round(left)), int(round(top))


def _open(img: ImageLike) -> PIL.Image.Image:
    if isinstance(img, str):
        return PIL.Image.open(img)
    if isinstance(img, np.ndarray):
        return PIL.Image.fromarray(img)
    return img


def _pil_tile(img: PIL.Image.Image) -> np.ndarray:
    """``resizeimg`` with PIL in the image's own mode (Pillow's default filter for it, alpha premultiplied, palette
    index 0 outside the image), then the RGB conversion the embedders apply when they read the saved tile."""
    nw, nh, left, top = resizeimg_plan(*img.size)
    tile = img.resize((nw, nh))
    if img.size[0] != img.size[1]:
        tile = tile.crop((left, top, left + SIZE, top + SIZE))
    return np.asarray(tile.convert("RGB"))


def evaluation_tiles(images: Sequence[ImageLike], device=None, num_workers: int = 0):
    """Paths / PIL images / arrays -> CUDA uint8 ``[n,224,224,3]``: the tiles ``resizeimg`` saves, as the embedders
    read them back (``_convert_image_to_rgb``).

    Images are opened as ``Image.open`` leaves them, without conversion.  RGB images the kernel's shared-memory plan
    takes are packed into one pinned buffer, uploaded once and resized + cropped by ``plip_resize_crop_fill_u8``;
    images in any other mode (P, L, RGBA, ...) and RGB images too large for the kernel are resized by PIL in their
    own mode with the same plan, then converted to RGB.  ``num_workers`` host threads decode (and run PIL).

    For lossless sources (PNG, TIFF: Kather, PanNuke, DigestPath, WSSS4LUAD) the tiles equal the files the reference
    writes.  For JPEG sources (KIMIA Path24) the reference re-encodes its tile as JPEG, so its files differ from these
    tiles by that encoding."""
    import torch

    from .engine import resize_crop_fill
    device = torch.device(device if device is not None else "cuda")
    images = list(images)

    def _decode(img):
        im = _open(img)
        if im.mode == "RGB" and resize_fits_device(*im.size, *resizeimg_plan(*im.size)[:2]):
            return np.asarray(im), True
        return _pil_tile(im), False

    if num_workers > 1 and len(images) > 1:
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=int(num_workers)) as ex:
            decoded = list(ex.map(_decode, images))
    else:
        decoded = [_decode(im) for im in images]
    out = torch.empty((len(images), SIZE, SIZE, 3), dtype=torch.uint8, device=device)
    dev = [i for i, (_, on_device) in enumerate(decoded) if on_device]
    host = [i for i, (_, on_device) in enumerate(decoded) if not on_device]
    if dev:
        arrays = [decoded[i][0] for i in dev]
        plan = np.zeros(len(arrays), dtype=RESIZE_DESC_DTYPE)
        for k, a in enumerate(arrays):
            plan[k]["new_width"], plan[k]["new_height"], plan[k]["left"], plan[k]["top"] = \
                resizeimg_plan(a.shape[1], a.shape[0])
        buf, descs = pack_rgb(arrays, pinned=True, plan=plan)
        tiles = resize_crop_fill(buf.to(device, non_blocking=True), descs)
        if len(dev) == len(images):
            return tiles
        out[torch.as_tensor(dev, device=device)] = tiles
    if host:
        pinned = torch.from_numpy(np.stack([decoded[i][0] for i in host])).pin_memory()
        out[torch.as_tensor(host, device=device)] = pinned.to(device, non_blocking=True)
    return out


def _tissue(t) -> str:
    return str(t).lower().replace("_", " ")


def pannuke_rows(sets: np.ndarray, types: np.ndarray) -> Dict[str, np.ndarray]:
    """The rows of ``PanNuke_all_binary.csv`` from the value sets of the masks (uint32 ``[n, c >= 6, 8]``, as
    ``plip_mask_value_sets_u8`` returns them) and the tissue types ``[n]``, in the reference's order: malignant images,
    then benign ones, each in source order.  Columns ``image`` (file name), ``caption``, ``source_index``.

    An image is dropped when channels 0..4 are all zero (each set is exactly ``{0}``).  A channel's instance count is
    its set's popcount minus 1, as ``len(np.unique(...)) - 1`` counts it (one too few for a channel without a zero).
    The tumour rule runs in float64 with the total over channels 0..5; an image whose counts are all 0 is benign here
    (its ratio is NaN), where the reference's object-dtype division stops with ZeroDivisionError."""
    sets = np.asarray(sets).view(np.uint32)
    if sets.ndim != 3 or sets.shape[1] < PANNUKE_CHANNELS or sets.shape[2] != 8:
        raise ValueError(f"sets must be [n, c >= {PANNUKE_CHANNELS}, 8], got {sets.shape}")
    types = np.asarray(types)
    if types.shape[0] != sets.shape[0]:
        raise ValueError(f"{sets.shape[0]} images but {types.shape[0]} types")
    only_zero = (sets[:, :5, 0] == 1) & np.all(sets[:, :5, 1:] == 0, axis=2)
    kept = np.flatnonzero(~np.all(only_zero, axis=1))
    bits = np.unpackbits(sets[kept, :PANNUKE_CHANNELS].view(np.uint8), axis=2)
    counts = bits.sum(axis=2, dtype=np.int64) - 1
    n0, total = counts[:, 0], counts.sum(axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = n0.astype(np.float64) / total.astype(np.float64)
    groups = (("malignant", kept[(n0 >= 10) & (ratio > 0.3)]), ("benign", kept[n0 == 0]))
    image: List[str] = []
    caption: List[str] = []
    for label, idx in groups:
        for i, src in enumerate(idx):
            tissue = _tissue(types[src])
            image.append("%s_%s_%04d.png" % (tissue, label, i))
            caption.append("An H&E image of %s %s tissue." % (label, tissue))
    return {"image": np.array(image, dtype=object), "caption": np.array(caption, dtype=object),
            "source_index": np.concatenate([idx for _, idx in groups]).astype(np.int64)}


def pannuke_binary(folds, device=None) -> Dict[str, object]:
    """PanNuke's malignant / benign table, ``preprocess/preprocess_PanNuke.py``, on the device.

    ``folds``: a sequence of ``(images, masks, types)`` per fold as ``np.load`` returns them (any dtype;
    ``mmap_mode="r"`` works): images ``[n, h, h, 3]``, masks ``[n, h, w, c >= 6]``, types ``[n]``.  The arrays are cast
    chunk by chunk with numpy's ``.astype(np.uint8)`` on the host, as the reference casts them (instance ids of 256 and
    more wrap there), uploaded through a pinned buffer, and each mask chunk's per-(image, channel) value sets come from
    ``plip_mask_value_sets_u8``.  Returns the columns of :func:`pannuke_rows` plus ``tiles``: the kept images'
    224 x 224 tiles, ``resizeimg``'s square branch (``img.resize((224, 224))``, bicubic), by ``plip_resize_crop_u8``.
    Nothing is written to disk."""
    import torch

    from .engine import mask_value_sets
    device = torch.device(device if device is not None else "cuda")
    folds = [tuple(f) for f in folds]
    shapes = set()
    for k, (images, masks, types) in enumerate(folds):
        if not (len(images) == len(masks) == len(types)):
            raise ValueError(f"fold {k}: {len(images)} images, {len(masks)} masks, {len(types)} types")
        if masks.ndim != 4 or not PANNUKE_CHANNELS <= masks.shape[3] <= 8:
            raise ValueError(f"fold {k}: masks must be [n, h, w, 6..8], got {masks.shape}")
        if images.ndim != 4 or images.shape[3] != 3 or images.shape[1] != images.shape[2]:
            raise ValueError(f"fold {k}: images must be square RGB [n, h, h, 3], got {images.shape}")
        shapes.add(masks.shape[1:])
    if len(shapes) > 1:
        raise ValueError(f"the folds' masks differ in shape: {sorted(shapes)}")
    n = sum(len(f[0]) for f in folds)
    c = shapes.pop()[2] if shapes else PANNUKE_CHANNELS
    sets = torch.empty((n, c, 8), dtype=torch.int32, device=device)
    base = 0
    for _, masks, _ in folds:   # pinned blocks return to torch's host cache once their upload has run
        for i in range(0, len(masks), MASK_CHUNK):
            chunk = torch.from_numpy(np.asarray(masks[i:i + MASK_CHUNK]).astype(np.uint8)).pin_memory()
            mask_value_sets(chunk.to(device, non_blocking=True), out=sets[base + i:base + i + len(chunk)])
        base += len(masks)
    types = np.concatenate([np.asarray(f[2]) for f in folds]) if folds else np.zeros(0, dtype=str)
    table = pannuke_rows(sets.cpu().numpy(), types)
    table["tiles"] = _pannuke_tiles(folds, table["source_index"], device)
    return table


def _pannuke_tiles(folds, source_index: np.ndarray, device):
    """224 x 224 tiles of the listed images (indices into the concatenated folds), in that order."""
    import torch

    from .engine import resize_crop
    out = torch.empty((len(source_index), SIZE, SIZE, 3), dtype=torch.uint8, device=device)
    starts = np.cumsum([0] + [len(f[0]) for f in folds])
    for r in range(0, len(source_index), MASK_CHUNK):
        idx = source_index[r:r + MASK_CHUNK]
        arrays = []
        for s in idx:
            f = int(np.searchsorted(starts, s, side="right")) - 1
            arrays.append(np.asarray(folds[f][0][s - starts[f]]).astype(np.uint8))
        plan = np.zeros(len(arrays), dtype=RESIZE_DESC_DTYPE)
        plan["new_width"] = plan["new_height"] = SIZE
        buf, descs = pack_rgb(arrays, pinned=True, plan=plan)
        resize_crop(buf.to(device, non_blocking=True), descs, out=out[r:r + len(arrays)])
    return out


def split_pannuke(table: Dict[str, object], seed: int = 1, train_ratio: float = 0.7):
    """``process_PanNuke`` (``_dataset_loader.py:182-233``): ``table`` (from :func:`pannuke_binary` or
    :func:`pannuke_rows`) -> ``(train, test)``.

    Each caption gives ``tissue``, ``label`` (1.0 malignant, 0.0 benign; float64, as the CSV holds it),
    ``label_text``, ``label_tissue`` and ``caption_no_tissue``.  The rows are shuffled with
    ``RandomState(seed).permutation`` (what ``df.sample(frac=1, random_state=seed)`` draws); then for each tissue in
    order of first appearance and each label (benign, then malignant) the subset is shuffled again the same way and its
    first ``int(len * train_ratio)`` rows go to train, the rest to test.  Columns: ``image, label, label_text,
    text_style_0`` (label + tissue), ``text_style_1`` (caption), ``text_style_4`` (caption without the tissue), and
    ``source_index`` / ``tiles`` carried along when present."""
    captions = [str(c) for c in table["caption"]]
    n = len(captions)
    tissue, label, label_text, label_tissue, no_tissue = [], [], [], [], []
    for cap in captions:
        for word, value in (("malignant", 1.0), ("benign", 0.0)):
            if word in cap:
                t = cap.split(word + " ")[1].split(" tissue")[0]
                break
        else:
            raise ValueError(f"caption {cap!r} names neither malignant nor benign")
        tissue.append(t)
        label.append(value)
        label_text.append(word)
        label_tissue.append("%s %s" % (word, t))
        no_tissue.append(cap.replace(t + " ", ""))
    tissue_a = np.array(tissue, dtype=object)
    text_a = np.array(label_text, dtype=object)
    order = np.random.RandomState(seed).permutation(n)
    seen = dict.fromkeys(tissue_a[order])
    train_rows: List[np.ndarray] = []
    test_rows: List[np.ndarray] = []
    for t in seen:
        for lt in ("benign", "malignant"):
            subset = order[(tissue_a[order] == t) & (text_a[order] == lt)]
            subset = subset[np.random.RandomState(seed).permutation(len(subset))]
            k = int(len(subset) * train_ratio)
            train_rows.append(subset[:k])
            test_rows.append(subset[k:])
    cols = {"image": np.array([str(x) for x in table["image"]], dtype=object),
            "label": np.array(label, dtype=np.float64), "label_text": text_a,
            "text_style_0": np.array(label_tissue, dtype=object), "text_style_1": np.array(captions, dtype=object),
            "text_style_4": np.array(no_tissue, dtype=object)}

    def _take(rows):
        rows = np.concatenate(rows).astype(np.int64) if rows else np.zeros(0, dtype=np.int64)
        out = {k: v[rows] for k, v in cols.items()}
        if "source_index" in table:
            out["source_index"] = np.asarray(table["source_index"])[rows]
        if "tiles" in table:
            import torch
            tiles = table["tiles"]
            out["tiles"] = tiles[torch.as_tensor(rows, device=tiles.device)]
        return out

    return _take(train_rows), _take(test_rows)
