"""Cost of the per-token outputs (``output_hidden_states`` / ``output_attentions``) on the GPU: ``get_image_features``
against ``vision_model`` with each flag and with both, at 1024 x 224^2 and at one full pass of 448^2 (259 images), the
same for ``text_model`` at 1024 x 77 tokens, and the attention-probabilities kernel per launch (in-call profile: its
time, GB/s and share of the HBM bound).  Records the card name and power limit.  GPU only.

    python tools/outputs_probe.py [out.json]
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from hires_probe import PEAK_GBS, card, timed  # noqa: E402
from oracle import synth, weights  # noqa: E402
from plip_b200.engine import Engine, vision_seq_len  # noqa: E402
from plip_b200.synthetic import pixel_values_hw  # noqa: E402

WARMUP, TIMED = 2, 5
VARIANTS = {"hidden_states": (True, False), "attentions": (False, True), "both": (True, True)}


def probs_profile(eng, call):
    """The probabilities kernel inside one outputs call: per-launch ms, GB/s, share of the HBM bound."""
    eng.profile(True)
    call()
    rows = eng.profile_read()
    eng.profile(False)
    r = next(r for r in rows if r["name"].endswith("attention[probs]"))
    ms = r["total_ms"] / r["launches"]
    return {"launches": r["launches"], "ms_per_launch": round(ms, 4),
            "MB_per_launch": round(r["bytes"] / r["launches"] / 1e6, 2),
            "GB/s": round(r["bytes"] / r["total_ms"] / 1e6, 1),
            "share_of_hbm_bound": round(r["bytes"] / (PEAK_GBS * 1e9) * 1e3 / r["total_ms"], 3)}


def compare(eng, features, outputs):
    base = timed(features, WARMUP, TIMED)
    res = {"features_ms": round(base, 3)}
    for name, (h, a) in VARIANTS.items():
        ms = timed(lambda: outputs(h, a), WARMUP, TIMED)
        res[f"{name}_ms"] = round(ms, 3)
        res[f"{name}_extra_ms"] = round(ms - base, 3)
    res["probs_kernel"] = probs_profile(eng, lambda: outputs(False, True))
    torch.cuda.empty_cache()
    return res


def main():
    if not torch.cuda.is_available():
        sys.exit("outputs_probe: needs a CUDA device")
    torch.set_grad_enabled(False)
    eng = Engine(weights.make_state_dict(0, "rich"), max_micro_batch=1024)
    report = {"card": card(), "max_micro_batch": 1024, "operand_format": "bf16", "cases": {}}
    for size, n in ((224, 1024), (448, 50 * 1024 // vision_seq_len(448, 448))):
        px = pixel_values_hw(n, size, size, seed=size).to(torch.bfloat16).cuda()
        ipe = size != 224
        res = compare(eng, lambda: eng.encode_images(px, interpolate_pos_encoding=ipe),
                      lambda h, a: eng.vision_outputs(px, h, a, interpolate_pos_encoding=ipe))
        res.update(images=n, tokens=vision_seq_len(size, size))
        report["cases"][f"vision_{size}"] = res
        print(json.dumps({f"vision_{size}": res}), flush=True)
        del px
    ids, mask = synth.token_ids(1024)
    ids, mask = ids.cuda(), mask.cuda()
    res = compare(eng, lambda: eng.encode_text(ids, mask),
                  lambda h, a: eng.text_outputs(ids, mask, h, a))
    res.update(captions=1024, tokens=77)
    report["cases"]["text_77"] = res
    print(json.dumps({"text_77": res}), flush=True)
    eng.close()
    out = json.dumps(report)
    print(out)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()
