"""The dataset builders of plip_b200.datasets on one GPU, against the reference's CPU path on the same host, in one call:

  - ``plip_mask_value_sets_u8`` on PanNuke-sized masks (7,901 x 256 x 256 x 6 uint8, already in device memory):
    kernel time (CUDA events) and GB/s against the H100 SXM's 3.35 TB/s;
  - the host-to-device upload of those masks from pinned memory;
  - ``pannuke_binary`` + ``split_pannuke`` from host arrays, wall clock around a device synchronise, and the
    reference's CPU path (np.unique per image and channel, PIL's 256 -> 224 resize) on a subset, per image;
  - ``plip_resize_crop_fill_u8`` tiles/s on WSSS4LUAD-like RGB sizes (150..400 px per side, sources in device memory)
    against ``resizeimg`` with PIL on the host's threads.

The folds are seeded synthetic ones (``make_pannuke_folds``, uint8): 256 distinct images repeated to PanNuke's 7,901.
Prints the card name and power limit with the numbers.  GPU only.

    python tools/dataset_probe.py [out.json] [--images 7901] [--threads 16]
"""
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import PIL.Image
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

from densenet_probe import timed  # noqa: E402
from region_probe import card  # noqa: E402

HBM = 3.35e12


def folds_of(n, seed=0):
    """Three folds of n images in all: 256 distinct synthetic images, repeated."""
    from plip_b200.synthetic import make_pannuke_folds
    (img, msk, typ), = make_pannuke_folds(seed, sizes=(256,), dtype=np.uint8)
    idx = np.arange(n) % len(img)
    parts = np.array_split(idx, 3)
    return [(img[p], msk[p], typ[p]) for p in parts]


def oracle_cpu(folds, n):
    """The reference's per-image work on the first n images: np.unique per channel, and the saved tile's resize."""
    imgs = np.concatenate([f[0] for f in folds])[:n]
    msks = np.concatenate([f[1] for f in folds])[:n]
    t0 = time.perf_counter()
    for i in range(n):
        for j in range(6):
            len(np.unique(msks[..., j].reshape(n, -1)[i, :]))
    t1 = time.perf_counter()
    for i in range(n):
        PIL.Image.fromarray(imgs[i]).resize((224, 224))
    t2 = time.perf_counter()
    return t1 - t0, t2 - t1


def main():
    if not torch.cuda.is_available():
        sys.exit("dataset_probe: needs a CUDA device")
    args = sys.argv[1:]
    n = int(args[args.index("--images") + 1]) if "--images" in args else 7901
    threads = int(args[args.index("--threads") + 1]) if "--threads" in args else min(16, os.cpu_count() or 1)
    out_path = args[0] if args and not args[0].startswith("--") else None
    from plip_b200.datasets import pannuke_binary, resizeimg_plan, split_pannuke
    from plip_b200.engine import mask_value_sets, resize_crop_fill
    from plip_b200.preprocess import RESIZE_DESC_DTYPE, pack_rgb
    res = {"card": card(), "images": n, "host_threads": threads}
    print(res["card"], flush=True)

    folds = folds_of(n)
    masks = np.concatenate([f[1] for f in folds])
    nbytes = masks.nbytes
    pinned = torch.from_numpy(masks).pin_memory()
    dev = torch.empty_like(pinned, device="cuda")
    t_up = timed(lambda: dev.copy_(pinned, non_blocking=True), 2.0)
    sets = torch.empty((n, 6, 8), dtype=torch.int32, device="cuda")
    t_k = timed(lambda: mask_value_sets(dev, out=sets), 2.0)
    res["mask_value_sets"] = {"bytes": nbytes, "ms": t_k * 1e3, "GB_s": nbytes / t_k / 1e9,
                              "share_of_3.35TB_s": nbytes / t_k / HBM}
    res["upload"] = {"bytes": nbytes, "ms": t_up * 1e3, "GB_s": nbytes / t_up / 1e9}
    del dev, pinned
    print("mask_value_sets", res["mask_value_sets"], "upload", res["upload"], flush=True)

    def pipeline():
        table = pannuke_binary(folds)
        train, test = split_pannuke(table)
        torch.cuda.synchronize()
        return table, train, test

    pipeline()                                                     # warm-up (module loads, allocator)
    walls = []
    for _ in range(3):
        t0 = time.perf_counter()
        table, train, test = pipeline()
        walls.append(time.perf_counter() - t0)
    sub = min(n, 600)
    t_unique, t_pil = oracle_cpu(folds, sub)
    res["pannuke"] = {"rows": len(table["image"]), "train": len(train["image"]), "test": len(test["image"]),
                      "wall_s": min(walls), "wall_s_all": walls,
                      "oracle_subset_images": sub, "oracle_unique_s_per_image": t_unique / sub,
                      "oracle_pil_resize_s_per_image": t_pil / sub}
    print("pannuke", res["pannuke"], flush=True)

    rng = np.random.default_rng(1)
    arrays = [rng.integers(0, 256, (int(h), int(w), 3), dtype=np.uint8) for w, h in rng.integers(150, 401, (2048, 2))]
    plan = np.zeros(len(arrays), dtype=RESIZE_DESC_DTYPE)
    for k, a in enumerate(arrays):
        plan[k]["new_width"], plan[k]["new_height"], plan[k]["left"], plan[k]["top"] = resizeimg_plan(a.shape[1],
                                                                                                      a.shape[0])
    buf, descs = pack_rgb(arrays, plan=plan)
    src = buf.cuda()
    tiles = torch.empty((len(arrays), 224, 224, 3), dtype=torch.uint8, device="cuda")
    t_a = timed(lambda: resize_crop_fill(src, descs, out=tiles), 2.0)

    def pil_one(a):
        w, h = a.shape[1], a.shape[0]
        nw, nh, left, top = resizeimg_plan(w, h)
        im = PIL.Image.fromarray(a).resize((nw, nh))
        return im.crop((left, top, left + 224, top + 224)) if w != h else im

    with ThreadPoolExecutor(max_workers=threads) as ex:
        list(ex.map(pil_one, arrays[:64]))
        t0 = time.perf_counter()
        list(ex.map(pil_one, arrays))
        t_pil = time.perf_counter() - t0
    res["resize_crop_fill"] = {"images": len(arrays), "ms": t_a * 1e3, "tiles_s": len(arrays) / t_a,
                               "pil_host_threads_tiles_s": len(arrays) / t_pil}
    print("resize_crop_fill", res["resize_crop_fill"], flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
