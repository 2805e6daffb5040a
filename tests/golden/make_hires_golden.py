"""Generate tests/golden/hires_golden.npz from the live ``transformers.CLIPModel`` (fp32, CPU):

    python tests/golden/make_hires_golden.py

``get_image_features(pixel_values, interpolate_pos_encoding=True)`` on ``make_state_dict(0, "rich")`` weights, for 2
seeded images (``plip_b200.synthetic.pixel_values_hw(2, H, W)``) at each size of ``tests/hires_oracle.HIRES_SIZES``,
and the first 5 / last 5 tokens of the first image's vision hidden states at layers 0, 1 and 12.  Only outputs are stored: weights
and inputs are regenerated from their seeds at test time.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from hires_oracle import HIRES_SIZES, size_key  # noqa: E402
from oracle import weights  # noqa: E402
from plip_b200.synthetic import pixel_values_hw  # noqa: E402

LAYERS = (0, 1, 12)


def main():
    import transformers
    from transformers import CLIPConfig, CLIPModel

    torch.set_grad_enabled(False)
    sd = weights.make_state_dict(0, "rich")
    hf = CLIPModel(CLIPConfig()).eval()
    hf.load_state_dict(sd, strict=True)
    out = {"transformers_version": np.array(transformers.__version__), "torch_version": np.array(torch.__version__)}
    for h, w in HIRES_SIZES:
        k = size_key(h, w)
        px = pixel_values_hw(2, h, w)
        out[f"image_features_{k}"] = hf.get_image_features(pixel_values=px, interpolate_pos_encoding=True).pooler_output.numpy()
        vo = hf.vision_model(pixel_values=px, output_hidden_states=True, interpolate_pos_encoding=True)
        for l in LAYERS:
            hs = vo.hidden_states[l]
            out[f"vision_hidden_{l}_{k}"] = torch.cat([hs[:1, :5], hs[:1, -5:]], dim=1).numpy()  # first image
        print(k, "S =", vo.hidden_states[0].shape[1])
    path = os.path.join(ROOT, "tests", "golden", "hires_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
