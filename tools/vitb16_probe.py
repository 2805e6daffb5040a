"""CLIP ViT-B/16 vision tower at 224^2 on uint8 device tiles, batch 1024: images/s of the engine with bf16 and fp16
operands and of transformers.CLIPModel(patch_size=16) in bf16 in the same process, three timed repeats each after a
warm-up (spread reported), the in-call kernel profile, and the achieved TFLOP/s from the shapes.  The card's name and
power limit are read in the same run.  GPU only: without CUDA it exits with an error.

    python tools/vitb16_probe.py [out.json]
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import vitb16_oracle as V  # noqa: E402
from hires_probe import card, timed  # noqa: E402
from oracle import clip_oracle as O  # noqa: E402
from plip_b200.engine import Engine  # noqa: E402
from plip_b200.synthetic import make_state_dict  # noqa: E402

N, MB = 1024, 1024
WARMUP, TIMED, REPEATS = 3, 10, 3
D, FF, S, P = 768, 3072, 197, 196


def flops_per_image(patch=16):
    """GEMM + attention FLOPs of one image's vision tower (the projection head aside): per layer QKV, QK^T, PV,
    out_proj, fc1, fc2; plus the patch GEMM."""
    s, p, k = (224 // patch) ** 2 + 1, (224 // patch) ** 2, 3 * patch * patch
    layer = 2 * s * D * 3 * D + 2 * 2 * s * s * D + 2 * s * D * D + 2 * 2 * s * D * FF
    return 12 * layer + 2 * p * k * D, layer, 2 * p * k * D


def spread(xs):
    return {"median": round(float(np.median(xs)), 1), "min": round(min(xs), 1), "max": round(max(xs), 1),
            "runs": [round(x, 1) for x in xs]}


def main():
    if not torch.cuda.is_available():
        sys.exit("vitb16_probe: needs a CUDA device")
    torch.set_grad_enabled(False)
    sd = make_state_dict(0, "rich", patch=16)
    tiles = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (N, 224, 224, 3), dtype=np.uint8)).cuda()
    f_img, f_layer, f_patch = flops_per_image(16)
    report = {"card": card(), "images": N, "max_micro_batch": MB,
              "gflop_per_image": round(f_img / 1e9, 3), "gflop_per_layer": round(f_layer / 1e9, 3),
              "gflop_patch_gemm": round(f_patch / 1e9, 3), "gflop_per_image_b32": round(flops_per_image(32)[0] / 1e9, 3),
              "engine": {}}
    # accuracy of the timed configuration: 2 tiles against the fp32 oracle
    ref = V.get_image_features(sd, O.preprocess_u8(tiles[:2].cpu()))
    engines = {dt: Engine(sd, max_micro_batch=MB, operand_dtype=dt) for dt in ("bf16", "fp16")}
    from transformers import CLIPConfig, CLIPModel
    hf = CLIPModel(CLIPConfig(vision_config={"patch_size": 16, "hidden_act": "quick_gelu"})).eval()
    hf.load_state_dict(sd, strict=True)
    hf = hf.to("cuda", torch.bfloat16)
    px_hf = O.preprocess_u8(tiles.cpu()).to("cuda", torch.bfloat16)  # transformers takes normalised pixels
    runs = {k: [] for k in ("bf16", "fp16", "transformers_bf16")}
    for dt, eng in engines.items():                                    # warm-up of every timed configuration
        timed(lambda: eng.encode_images(tiles), WARMUP, 1)
    timed(lambda: hf.get_image_features(pixel_values=px_hf), 1, 1)
    for _ in range(REPEATS):                                           # alternate the three, repeat
        for dt, eng in engines.items():
            runs[dt].append(N / timed(lambda: eng.encode_images(tiles), 1, TIMED) * 1e3)
        runs["transformers_bf16"].append(N / timed(lambda: hf.get_image_features(pixel_values=px_hf), 1, 3) * 1e3)
    for dt, eng in engines.items():
        eng.profile(True)
        eng.encode_images(tiles)
        rows = eng.profile_read()
        eng.profile(False)
        prof = {}
        for r in rows:
            d = {"launches": r["launches"], "ms": round(r["total_ms"], 4)}
            if r["total_ms"] > 0 and r["flops"] > 0:
                d["TFLOP/s"] = round(r["flops"] / r["total_ms"] / 1e9, 1)
            if r["total_ms"] > 0 and r["bytes"] > 0:
                d["GB/s"] = round(r["bytes"] / r["total_ms"] / 1e6, 1)
            prof[r["name"]] = d
        ips = float(np.median(runs[dt]))
        report["engine"][dt] = {
            "images_per_s": spread(runs[dt]), "achieved_TFLOP_s": round(ips * f_img / 1e12, 1),
            "one_minus_cos_vs_oracle": (1 - O.cosine(eng.encode_images(tiles[:2]).cpu(), ref)).max().item(),
            "profile": prof}
    report["transformers_bf16"] = {"images_per_s": spread(runs["transformers_bf16"]),
                                   "achieved_TFLOP_s": round(float(np.median(runs["transformers_bf16"])) * f_img / 1e12, 1)}
    for eng in engines.values():
        eng.close()
    out = json.dumps(report)
    print(out)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()
