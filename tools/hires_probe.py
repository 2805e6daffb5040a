"""Vision tower at 224^2, 448^2, 512^2 and 1024^2 (interpolate_pos_encoding): images/s with bf16 pixels resident on the
device, the in-call kernel profile (the long-sequence attention kernel against the roofline its S puts it under, GEMM
TFLOP/s next to the 224 tower's), transformers.CLIPModel in bf16 on the same GPU as context, and 1 - cos against the
golden vectors / the fp32 oracle.  GPU only: without CUDA it exits with an error.

    python tools/hires_probe.py [out.json]
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import hires_oracle as HO  # noqa: E402
from oracle import clip_oracle as O  # noqa: E402
from oracle import weights  # noqa: E402
from plip_b200.engine import Engine, vision_seq_len  # noqa: E402
from plip_b200.synthetic import pixel_values_hw  # noqa: E402

SIZES = (224, 448, 512, 1024)
WARMUP, TIMED = 3, 20
PEAK_TFLOPS, PEAK_GBS = 989.0, 3350.0  # H100 SXM data sheet (dense BF16, HBM3), 700 W


def timed(fn, warmup, iters):
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


def main():
    if not torch.cuda.is_available():
        sys.exit("hires_probe: needs a CUDA device")
    torch.set_grad_enabled(False)
    sd = weights.make_state_dict(0, "rich")
    golden = dict(np.load(os.path.join(ROOT, "tests", "golden", "hires_golden.npz")))
    eng = Engine(sd, max_micro_batch=1024)
    from transformers import CLIPConfig, CLIPModel
    hf = CLIPModel(CLIPConfig()).eval()
    hf.load_state_dict(sd, strict=True)
    hf = hf.to("cuda", torch.bfloat16)
    report = {"card": card(), "max_micro_batch": 1024, "operand_format": "bf16", "sizes": {}}
    for s in SIZES:
        S = vision_seq_len(s, s)
        n = min(1024, 50 * 1024 // S)           # one full token budget: one pass
        px = pixel_values_hw(n, s, s, seed=s).to(torch.bfloat16).cuda()
        ipe = s != 224
        ms = timed(lambda: eng.encode_images(px, interpolate_pos_encoding=ipe), WARMUP, TIMED)
        eng.profile(True)
        eng.encode_images(px, interpolate_pos_encoding=ipe)
        rows = eng.profile_read()
        eng.profile(False)
        prof = {}
        for r in rows:
            d = {"launches": r["launches"], "ms": round(r["total_ms"], 4)}
            if r["total_ms"] > 0 and r["flops"] > 0:
                d["TFLOP/s"] = round(r["flops"] / r["total_ms"] / 1e9, 1)
            if r["total_ms"] > 0 and r["bytes"] > 0:
                d["GB/s"] = round(r["bytes"] / r["total_ms"] / 1e6, 1)
            if "attention" in r["name"] and r["total_ms"] > 0:
                t_min = max(r["flops"] / (PEAK_TFLOPS * 1e12), r["bytes"] / (PEAK_GBS * 1e9)) * 1e3
                d["bound"] = "tensor" if r["flops"] / (PEAK_TFLOPS * 1e12) > r["bytes"] / (PEAK_GBS * 1e9) else "HBM"
                d["share_of_datasheet_bound"] = round(t_min / r["total_ms"], 3)
            prof[r["name"]] = d
        # accuracy: 2 fp32 images against the live-transformers golden (or the fp32 oracle where none is stored)
        px2 = pixel_values_hw(2, s, s)
        key = f"image_features_{HO.size_key(s, s)}"
        if key in golden:
            ref, against = torch.from_numpy(golden[key]), "golden"
        else:
            ref, against = HO.get_image_features(sd, px2, interpolate_pos_encoding=True), "oracle"
        cos = (1 - O.cosine(eng.encode_images(px2.cuda(), interpolate_pos_encoding=True).cpu(), ref)).max().item()
        # context: transformers in bf16 on the same GPU, same inputs
        hf_ms = timed(lambda: hf.get_image_features(pixel_values=px, interpolate_pos_encoding=ipe), 2, 5)
        report["sizes"][f"{s}x{s}"] = {
            "tokens_per_image": S, "images_per_call": n, "ms_per_call": round(ms, 3),
            "images_per_s": round(n / ms * 1e3, 1), "transformers_bf16_images_per_s": round(n / hf_ms * 1e3, 1),
            "one_minus_cos": cos, "cos_against": against, "profile": prof}
        print(json.dumps({f"{s}x{s}": report["sizes"][f"{s}x{s}"]}), flush=True)
        del px
        torch.cuda.empty_cache()
    eng.close()
    out = json.dumps(report)
    print(out)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()
