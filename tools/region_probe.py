"""Slide regions on one GPU: windows/s of ``regions.encode_region`` on an 8192 x 8192 device region with white blocks
against torch crops + ``Engine.encode_images`` on the same kept windows; GB/s of the background kernel and of the
window gather next to the tile im2col of the same run; windows/s of the host-region (band) path against host crops +
``encode_images_host``.  Prints the card name and power limit with the numbers.  GPU only.

    python tools/region_probe.py [out.json]
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import weights  # noqa: E402
from plip_b200.engine import Engine, window_background_counts  # noqa: E402
from plip_b200.regions import encode_region, window_grid  # noqa: E402

SIDE = 8192
WINDOW_BYTES = 224 * 224 * 3


def timed(fn, warmup=2, iters=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as ex:  # the numbers below stay valid; the card line says what could not be read
        info["power_limit"] = f"unknown ({ex})"
    return info


def make_region(side, seed=0):
    """Random tissue-like pixels with white (background) blocks covering about a third of the region."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = torch.randint(0, 256, (side, side, 3), generator=g, device="cuda", dtype=torch.uint8)
    gh = np.random.default_rng(seed)
    for _ in range(24):
        h, w = int(gh.integers(300, side // 4)), int(gh.integers(300, side // 4))
        y, x = int(gh.integers(0, side - h)), int(gh.integers(0, side - w))
        r[y:y + h, x:x + w] = 240
    return r


def device_crops(region, origins):
    """The kept windows cut out on the device with one advanced-index gather: [k, 224, 224, 3]."""
    o = torch.from_numpy(origins).to(region.device, torch.int64)
    ar = torch.arange(224, device=region.device)
    return region[(o[:, 0, None] + ar)[:, :, None], (o[:, 1, None] + ar)[:, None, :]]


def im2col_gbs(eng, fn):
    eng.profile(True)
    fn()
    rows = {r["name"]: r for r in eng.profile_read()}
    eng.profile(False)
    r = rows["vision/im2col"]
    return round(r["bytes"] / r["total_ms"] / 1e6, 1), round(r["total_ms"], 4)


def main():
    if not torch.cuda.is_available():
        sys.exit("region_probe: needs a CUDA device")
    torch.set_grad_enabled(False)
    eng = Engine(weights.make_state_dict(0, "rich"), max_micro_batch=1024)
    region = make_region(SIDE)
    grid = window_grid(SIDE, SIDE)
    report = {"card": card(), "region": f"{SIDE}x{SIDE}", "grid_windows": len(grid.origins), "max_micro_batch": 1024}

    # device region: encode_region (count + keep + encode) vs torch crops + encode_images of the kept windows
    res = encode_region(eng, region)
    kept = res.origins
    crops = device_crops(region, kept)
    same = torch.equal(res.embeddings, eng.encode_images(crops))
    ms_region = timed(lambda: encode_region(eng, region))
    ms_crops = timed(lambda: eng.encode_images(device_crops(region, kept)))
    report["device_region"] = {
        "kept_windows": len(kept), "encode_region_ms": round(ms_region, 3),
        "encode_region_windows_per_s": round(len(kept) / ms_region * 1e3, 1),
        "torch_crops_encode_images_ms": round(ms_crops, 3),
        "torch_crops_encode_images_windows_per_s": round(len(kept) / ms_crops * 1e3, 1),
        "embeddings_bit_identical": bool(same)}

    # background kernel over every grid window: algorithmic bytes n * 150528 read
    n = len(grid.origins)
    ms_bg = timed(lambda: window_background_counts(region, grid.origins), 3, 20)
    # window gather vs tile im2col inside the same encode (profile role "vision/im2col"), one pass of 1024 windows
    o1k = kept[:1024]
    gbs_win, ms_win = im2col_gbs(eng, lambda: eng.encode_windows(region, o1k))
    tiles = device_crops(region, o1k).contiguous()
    gbs_tile, ms_tile = im2col_gbs(eng, lambda: eng.encode_images(tiles))
    report["kernels"] = {
        "background_ms": round(ms_bg, 4), "background_GB_per_s": round(n * WINDOW_BYTES / ms_bg / 1e6, 1),
        "window_gather_ms_1024": ms_win, "window_gather_GB_per_s": gbs_win,
        "tile_im2col_ms_1024": ms_tile, "tile_im2col_GB_per_s": gbs_tile}

    # host region: bands through pinned memory vs host crops + encode_images_host of the same kept windows
    host = region.cpu().numpy()
    hres = encode_region(eng, host)
    cos = torch.nn.functional.cosine_similarity(hres.embeddings, res.embeddings).min().item()
    pinned = torch.empty((len(kept), 224, 224, 3), dtype=torch.uint8).pin_memory()

    def host_crops():
        v = pinned.numpy()
        for i, (r, c) in enumerate(kept.tolist()):
            v[i] = host[r:r + 224, c:c + 224]
        return eng.encode_images_host(pinned)

    ms_hregion = timed(lambda: encode_region(eng, host), 1, 3)
    ms_hcrops = timed(host_crops, 1, 3)
    report["host_region"] = {
        "encode_region_ms": round(ms_hregion, 3), "encode_region_windows_per_s": round(len(kept) / ms_hregion * 1e3, 1),
        "host_crops_encode_images_host_ms": round(ms_hcrops, 3),
        "host_crops_encode_images_host_windows_per_s": round(len(kept) / ms_hcrops * 1e3, 1),
        "min_cos_vs_device_path": cos}
    eng.close()
    out = json.dumps(report)
    print(out)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()
