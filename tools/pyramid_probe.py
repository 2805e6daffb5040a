"""Region pyramids on one GPU, on an 8192 x 8192 region with white blocks at the reference's levels (2, 4, 8, 16, 32):
per-level time and GB/s of the whole-image resize against the HBM bound (source read, intermediate write and read,
level write), kept windows/s of ``regions.encode_region_pyramid`` on a device and on a host region, and the CPU route
of the same work (PIL resize, the crop loop in numpy, ``encode_images`` on the crops).  Checks the device levels
against PIL bit for bit.  Prints the card name and power limit with the numbers.  GPU only.

    python tools/pyramid_probe.py [out.json]
"""
import json
import os
import sys
import time

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from oracle import weights  # noqa: E402
from plip_b200.engine import Engine, resize_region  # noqa: E402
from plip_b200.regions import (DOWNSAMPLE_LIST, encode_region_pyramid, keep_windows, level_size,  # noqa: E402
                               window_grid)
from region_probe import card, make_region, timed  # noqa: E402

SIDE = 8192
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet (700 W)


def cpu_route(eng, host):
    """The reference's way: PIL resize per level, the crop loop in numpy, encode_images on the kept crops."""
    t0 = time.perf_counter()
    kept, t_resize = 0, 0.0
    for ds in DOWNSAMPLE_LIST:
        h, w = level_size(SIDE, SIDE, ds)
        r0 = time.perf_counter()
        lv = np.asarray(Image.fromarray(host).resize((w, h)))
        t_resize += time.perf_counter() - r0
        if h < 224 or w < 224:
            continue
        g = window_grid(h, w)
        crops = np.stack([lv[r:r + 224, c:c + 224] for r, c in g.origins]) if len(g.origins) else None
        if crops is None:
            continue
        counts = (crops >= 200).all(-1).reshape(len(crops), -1).sum(1)
        keep, _ = keep_windows(counts)
        if keep.any():
            eng.encode_images(torch.from_numpy(np.ascontiguousarray(crops[keep])).cuda())
            kept += int(keep.sum())
    torch.cuda.synchronize()
    return time.perf_counter() - t0, t_resize, kept


def main():
    if not torch.cuda.is_available():
        sys.exit("pyramid_probe: needs a CUDA device")
    torch.set_grad_enabled(False)
    eng = Engine(weights.make_state_dict(0, "rich"), max_micro_batch=1024)
    region = make_region(SIDE)
    host = region.cpu().numpy()
    report = {"card": card(), "region": f"{SIDE}x{SIDE}", "levels": list(DOWNSAMPLE_LIST), "max_micro_batch": 1024,
              "hbm_bound_bytes_per_s": HBM_BYTES_PER_S}

    # per-level resize: bytes the two passes must move at least, over the call time (three launches)
    src_bytes = SIDE * SIDE * 3
    levels = []
    for ds in DOWNSAMPLE_LIST:
        h, w = level_size(SIDE, SIDE, ds)
        out = torch.empty((h, w, 3), dtype=torch.uint8, device="cuda")
        ms = timed(lambda: resize_region(region, h, w, out=out), 2, 10)
        nbytes = src_bytes + 2 * SIDE * w * 3 + h * w * 3
        same = np.array_equal(out.cpu().numpy(), np.asarray(Image.fromarray(host).resize((w, h))))
        levels.append({"downsample": ds, "size": [h, w], "resize_ms": round(ms, 4), "bytes": nbytes,
                       "GB_per_s": round(nbytes / ms / 1e6, 1),
                       "share_of_hbm_bound": round(nbytes / HBM_BYTES_PER_S * 1e3 / ms, 3),
                       "bit_identical_to_pil": bool(same)})
    report["resize"] = levels

    dev = encode_region_pyramid(eng, region)
    kept = sum(len(lv.origins) for lv in dev)
    report["grid_windows"] = [len(window_grid(*level_size(SIDE, SIDE, ds)).origins) for ds in DOWNSAMPLE_LIST]
    report["kept_windows"] = [len(lv.origins) for lv in dev]
    ms_dev = timed(lambda: encode_region_pyramid(eng, region), 1, 5)
    ms_host = timed(lambda: encode_region_pyramid(eng, host), 1, 3)
    hres = encode_region_pyramid(eng, host)
    same = all(torch.equal(a.embeddings, b.embeddings) for a, b in zip(hres, dev))
    report["device_region"] = {"ms": round(ms_dev, 3), "kept_windows_per_s": round(kept / ms_dev * 1e3, 1)}
    report["host_region"] = {"ms": round(ms_host, 3), "kept_windows_per_s": round(kept / ms_host * 1e3, 1),
                             "bit_identical_to_device": bool(same)}
    cpu_route(eng, host)                                   # warm the encode shapes once
    s, s_resize, k_cpu = cpu_route(eng, host)
    report["cpu_route"] = {"ms": round(s * 1e3, 1), "pil_resize_ms": round(s_resize * 1e3, 1),
                           "kept_windows": k_cpu, "kept_windows_per_s": round(k_cpu / s, 1)}
    eng.close()
    out = json.dumps(report)
    print(out)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()
