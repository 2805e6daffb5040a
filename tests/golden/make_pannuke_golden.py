"""Generate tests/golden/pannuke_golden.npz: the PanNuke benchmark of seeded synthetic folds, frozen.

Run once in the build container:  python tests/golden/make_pannuke_golden.py

The folds come from ``plip_b200.synthetic.make_pannuke_folds(SEED)``.  The table and the split are built by
``tests/dataset_oracle.py`` with pandas and PIL (np.unique per image and channel, the reference's DataFrame steps,
``Image.fromarray(...).save`` as PNG and ``resizeimg`` on the file read back).  Only outputs are stored: the rows of
``PanNuke_all_binary.csv`` (file name, caption, source index, SHA-256 of the 224 x 224 tile the embedders read), the
train / test rows in order with their labels and text columns, and the library versions used."""
import hashlib
import os
import sys
import tempfile

import numpy as np
import PIL
import PIL.Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

SEED = 0
SPLIT_SEED, TRAIN_RATIO = 1, 0.7
TEXT = ("image", "label_text", "text_style_0", "text_style_1", "text_style_4")


def sha(tile):
    return hashlib.sha256(np.ascontiguousarray(tile, dtype=np.uint8).tobytes()).hexdigest()


def build():
    """The golden arrays, computed with the oracle (pandas + PIL)."""
    import pandas as pd

    import dataset_oracle as O
    from plip_b200.synthetic import make_pannuke_folds
    folds = make_pannuke_folds(SEED)
    df, src, imgs = O.pannuke_table(folds)
    with tempfile.TemporaryDirectory() as tmp:
        tiles = []
        for name, img in zip(df["image"], imgs):
            png = os.path.join(tmp, os.path.basename(name))
            PIL.Image.fromarray(img).save(png)
            with PIL.Image.open(png) as im:
                tiles.append(O.saved_tile(im, os.path.join(tmp, "tile_" + os.path.basename(name))))
    sha_of = {os.path.basename(n): sha(t) for n, t in zip(df["image"], tiles)}
    train, test = O.process_pannuke(df, SPLIT_SEED, TRAIN_RATIO)
    out = {"table_image": np.array([os.path.basename(x) for x in df["image"]]),
           "table_caption": np.array(list(df["caption"])), "table_source_index": src,
           "table_tile_sha256": np.array([sha_of[os.path.basename(x)] for x in df["image"]]),
           "versions": np.array([f"numpy {np.__version__}", f"Pillow {PIL.__version__}", f"pandas {pd.__version__}"])}
    for part, frame in (("train", train), ("test", test)):
        names = [os.path.basename(x) for x in frame["image"]]
        out[f"{part}_image"] = np.array(names)
        out[f"{part}_label"] = frame["label"].to_numpy(dtype=np.float64)
        assert frame["label"].dtype == np.float64
        for col in TEXT[1:]:
            out[f"{part}_{col}"] = np.array(list(frame[col]))
        out[f"{part}_tile_sha256"] = np.array([sha_of[x] for x in names])
    return out


def main():
    out = build()
    path = os.path.join(HERE, "pannuke_golden.npz")
    np.savez_compressed(path, **out)
    print(path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
