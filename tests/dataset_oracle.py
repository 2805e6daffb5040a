"""Plain numpy / PIL / pandas restatement of the reference's evaluation-dataset steps, for the dataset tests:
``resizeimg`` (generate_validation_datasets/prepare_dataset_to_csv.py:40-63), the PanNuke labelling
(preprocess/preprocess_PanNuke.py) and ``process_PanNuke`` (_dataset_loader.py:182-233).  Written from their
behaviour, step by step, with the same library calls; pandas is imported only where the reference uses it."""
import os

import numpy as np
import PIL.Image

NEWSIZE = 224


def resizeimg_box(width, height):
    """The reference's resize size and (float) crop box of a non-square image."""
    scale = NEWSIZE / min(width, height)
    left, top = (width - NEWSIZE) / 2, (height - NEWSIZE) / 2
    return (int(width * scale), int(height * scale)), (left, top, left + NEWSIZE, top + NEWSIZE)


def resizeimg(img):
    """The tile ``resizeimg`` saves for a PIL image (before any file format)."""
    if img.size[0] != img.size[1]:
        size, box = resizeimg_box(*img.size)
        return img.resize(size).crop(box)
    return img.resize((NEWSIZE, NEWSIZE))


def saved_tile(img, path):
    """``resizeimg`` saved as PNG, then read back as the embedders read it (``Image.open(...).convert("RGB")``)."""
    resizeimg(img).save(path)
    with PIL.Image.open(path) as im:
        return np.asarray(im.convert("RGB"))


def unique_counts(masks_u8):
    """``len(np.unique(masks[i, ..., j])) - 1`` for every image and channel (the reference's loop)."""
    n, c = masks_u8.shape[0], masks_u8.shape[3]
    out = np.zeros((n, c), dtype=np.int64)
    for i in range(n):
        for j in range(c):
            out[i, j] = len(np.unique(masks_u8[..., j].reshape(n, -1)[i, :])) - 1
    return out


def value_sets(masks_u8):
    """The 256-bit value set of every (image, channel), uint32 [n, c, 8], from np.unique."""
    n, c = masks_u8.shape[0], masks_u8.shape[3]
    out = np.zeros((n, c, 8), dtype=np.uint32)
    for i in range(n):
        for j in range(c):
            for v in np.unique(masks_u8[i, ..., j]):
                out[i, j, v >> 5] |= np.uint32(1 << (int(v) & 31))
    return out


def pannuke_table(folds, savedir="images"):
    """``PanNuke_all_binary.csv`` as the reference builds it (a pandas DataFrame with the file paths under
    ``savedir``), plus the source index of every row and the uint8 images, in row order."""
    import pandas as pd
    imgs = np.concatenate([f[0].astype(np.uint8) for f in folds], axis=0)
    msks = np.concatenate([f[1].astype(np.uint8) for f in folds], axis=0)
    typs = np.concatenate([f[2] for f in folds], axis=0)
    src = np.arange(len(imgs))
    idx = np.sum(msks[..., 0:5].reshape(len(msks), -1), axis=1) == 0
    imgs, msks, typs, src = imgs[~idx], msks[~idx], typs[~idx], src[~idx]
    stat = pd.DataFrame(index=np.arange(len(imgs)), columns=np.arange(6))
    counts = unique_counts(msks[..., :6])
    for i in range(len(imgs)):
        for j in range(6):
            stat.loc[i, j] = int(counts[i, j])
    total = stat.sum(axis=1)
    tumor = (stat[0] >= 10) & (stat[0] / total > 0.3)
    benign = stat[0] == 0
    df = pd.DataFrame()
    rows_src, rows_img = [], []
    for label, sel in (("malignant", tumor.to_numpy(dtype=bool)), ("benign", benign.to_numpy(dtype=bool))):
        for i, k in enumerate(np.flatnonzero(sel)):
            tissue = str(typs[k]).lower().replace("_", " ")
            fname = "%s_%s_%04d.png" % (tissue, label, i)
            row = pd.DataFrame({"image": os.path.join(savedir, fname),
                                "caption": "An H&E image of %s %s tissue." % (label, tissue)}, index=[i])
            df = pd.concat([df, row], axis=0)
            rows_src.append(src[k])
            rows_img.append(imgs[k])
    return df, np.array(rows_src, dtype=np.int64), rows_img


def process_pannuke(df, seed=1, train_ratio=0.7):
    """``process_PanNuke`` on the table (after its CSV round trip: a fresh 0..n-1 index)."""
    import pandas as pd
    df = df.reset_index(drop=True)
    for i in df.index:
        caption = df.loc[i, "caption"]
        for word, value in (("malignant", 1), ("benign", 0)):
            if word in caption:
                tissue = caption.split(word + " ")[1].split(" tissue")[0]
                df.loc[i, "tissue"] = tissue
                df.loc[i, "label"] = value
                df.loc[i, "label_text"] = word
                df.loc[i, "label_tissue"] = "%s %s" % (word, tissue)
                df.loc[i, "caption_no_tissue"] = caption.replace(tissue + " ", "")
                break
    df = df.sample(frac=1, random_state=seed).reset_index(drop=True)
    train, test = pd.DataFrame(), pd.DataFrame()
    for tissue in df["tissue"].unique():
        for label_text in ["benign", "malignant"]:
            sub = df.loc[(df["tissue"] == tissue) & (df["label_text"] == label_text)]
            sub = sub.sample(frac=1, random_state=seed).reset_index(drop=True)
            k = int(len(sub) * train_ratio)
            train = pd.concat([train, sub.iloc[:k, :].reset_index(drop=True)], axis=0)
            test = pd.concat([test, sub.iloc[k:, :].reset_index(drop=True)], axis=0)
    cols = ["image", "label", "label_text", "label_tissue", "caption", "caption_no_tissue"]
    names = ["image", "label", "label_text", "text_style_0", "text_style_1", "text_style_4"]
    out = []
    for part in (train.reset_index(drop=True), test.reset_index(drop=True)):
        part = part[cols]
        part.columns = names
        out.append(part)
    return tuple(out)
