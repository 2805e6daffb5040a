"""The MuDiPath DenseNet-121 embedder on one GPU: images/s of ``DenseNetEngine.encode_images`` on device-resident
uint8 224 x 224 tiles at a user-sized micro-batch, against two cuDNN arms on the same card in the same call:

  - the reference's own arm: the ``torch.nn.functional`` restatement of ``NoHeadDenseNet`` (``tests/densenet_oracle``)
    in fp32 with cuDNN's defaults (TF32 convolutions), which is what ``build_densenet(...).to("cuda")`` runs;
  - the same in bf16 with channels_last tensors, for context.

Every arm is warmed up and timed with CUDA events over at least a second of work.  Prints the card name and power
limit, the multiply-adds and compulsory HBM bytes per image computed from the shapes, the share of the data-sheet
BF16 rate reached, and 1 - cos of the engine against the fp32 arm.  Synthetic seeded weights (same shapes as the
MuDiPath checkpoint).  GPU only.

    python tools/densenet_probe.py [out.json] [--batch 256]
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import densenet_oracle as O  # noqa: E402
from plip_b200.densenet import DenseNetEngine  # noqa: E402
from region_probe import card  # noqa: E402

BF16_PEAK = 989e12      # H100 SXM data sheet, dense BF16, 700 W
HBM_PEAK = 3.35e12


def macs_per_image():
    """Multiply-adds of the engine's convolutions (the transitions pool before their 1x1 conv) and of the
    reference's order (conv, then pool), from the shapes."""
    stem = 112 * 112 * 64 * 147
    engine = ref = stem
    c, side = 64, 56
    for b, n in enumerate(O.BLOCKS):
        for j in range(n):
            layer = side * side * (128 * (c + 32 * j) + 32 * 1152)
            engine += layer
            ref += layer
        c += 32 * n
        if b < 3:
            engine += (side // 2) ** 2 * (c // 2) * c
            ref += side * side * (c // 2) * c
            c //= 2
            side //= 2
    return engine, ref


def timed(fn, min_seconds=1.0):
    """Mean seconds per call over >= min_seconds of back-to-back calls (after one warm-up call)."""
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps, total = 1, 0.0
    while True:
        start.record()
        for _ in range(reps):
            fn()
        end.record()
        end.synchronize()
        total = start.elapsed_time(end) / 1e3
        if total >= min_seconds:
            return total / reps
        reps = max(reps * 2, int(reps * min_seconds / max(total, 1e-6)) + 1)


def main():
    if not torch.cuda.is_available():
        sys.exit("densenet_probe: needs a CUDA device")
    args = sys.argv[1:]
    batch = int(args[args.index("--batch") + 1]) if "--batch" in args else 256
    out_path = next((a for i, a in enumerate(args) if not a.startswith("--") and (i == 0 or args[i - 1] != "--batch")),
                    None)
    torch.set_grad_enabled(False)
    sd = O.make_state_dict(0)
    eng = DenseNetEngine(sd, device="cuda:0", max_micro_batch=batch)
    g = torch.Generator(device="cuda").manual_seed(0)
    tiles = torch.randint(0, 256, (batch, 224, 224, 3), generator=g, device="cuda", dtype=torch.uint8)
    out = torch.empty(batch, 1024, device="cuda")
    res = {"card": card(), "batch": batch}
    macs, macs_ref = macs_per_image()
    comp_bytes = 224 * 224 * 3 + 1024 * 4
    res["macs_per_image"], res["macs_per_image_conv_then_pool"] = macs, macs_ref
    res["compulsory_bytes_per_image"] = comp_bytes
    res["weight_bytes"] = int(eng._L.plip_densenet_blob_bytes())

    t = timed(lambda: eng.encode_images(tiles, out=out))
    res["engine_img_s"] = batch / t
    res["engine_tflops"] = 2 * macs * batch / t / 1e12
    res["engine_share_of_bf16_peak"] = 2 * macs * batch / t / BF16_PEAK
    res["bound_img_s_flops"] = BF16_PEAK / (2 * macs)
    res["bound_img_s_bytes"] = HBM_PEAK / comp_bytes

    sdc = {k: v.cuda() for k, v in sd.items()}
    x = O.normalize_u8(tiles)
    torch.backends.cudnn.benchmark = False
    ref_out = O.forward(sdc, x)
    t = timed(lambda: O.forward(sdc, x))
    res["cudnn_fp32_tf32_img_s"] = batch / t
    sdb = {k: (v.to(torch.bfloat16) if v.is_floating_point() else v) for k, v in sdc.items()}
    xb = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    sdb = {k: (v.contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v) for k, v in sdb.items()}
    t = timed(lambda: O.forward(sdb, xb))
    res["cudnn_bf16_channels_last_img_s"] = batch / t

    eng.encode_images(tiles, out=out)
    torch.cuda.synchronize()
    res["engine_vs_fp32_arm_1mcos_max"] = O.cosine_gap(out, ref_out).max().item()
    res["speedup_vs_fp32_arm"] = res["engine_img_s"] / res["cudnn_fp32_tf32_img_s"]
    res["speedup_vs_bf16_arm"] = res["engine_img_s"] / res["cudnn_bf16_channels_last_img_s"]
    print(json.dumps(res, indent=1))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
