"""Generate tests/golden/vitb16_golden.npz from the live ``transformers.CLIPModel`` with ``patch_size=16`` (fp32, CPU):

    python tests/golden/make_vitb16_golden.py

``CLIPModel(CLIPConfig(vision_config={"patch_size": 16, "hidden_act": "quick_gelu"}))`` loaded with
``make_state_dict(0, "rich", patch=16)`` weights.  For 2 seeded images (``plip_b200.synthetic.pixel_values_hw(2, H, W)``)
at each size of ``tests/vitb16_oracle.SIZES``: ``get_image_features`` (with ``interpolate_pos_encoding`` off the 224
grid), and at 224 x 224 and 320 x 448 the first 5 / last 5 tokens of the first image's hidden states at layers 0, 1 and
12 and the first 4 query rows of its layer-0 and layer-11 attentions (all heads).  Only outputs are stored: weights and
inputs are regenerated from their seeds at test time.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from vitb16_oracle import SIZES, size_key  # noqa: E402
from plip_b200.synthetic import make_state_dict, pixel_values_hw  # noqa: E402

LAYERS = (0, 1, 12)
ATTN_LAYERS = (0, 11)
DETAIL_SIZES = SIZES[:2]


def main():
    import transformers
    from transformers import CLIPConfig, CLIPModel

    torch.set_grad_enabled(False)
    sd = make_state_dict(0, "rich", patch=16)
    cfg = CLIPConfig(vision_config={"patch_size": 16, "hidden_act": "quick_gelu"})
    hf = CLIPModel(cfg).eval()
    hf.config._attn_implementation = "eager"
    hf.load_state_dict(sd, strict=True)
    out = {"transformers_version": np.array(transformers.__version__), "torch_version": np.array(torch.__version__)}
    for h, w in SIZES:
        k = size_key(h, w)
        px = pixel_values_hw(2, h, w)
        ipe = (h, w) != (224, 224)
        out[f"image_features_{k}"] = hf.get_image_features(pixel_values=px, interpolate_pos_encoding=ipe).pooler_output.numpy()
        if (h, w) not in DETAIL_SIZES:
            continue
        vo = hf.vision_model(pixel_values=px, output_hidden_states=True, output_attentions=True,
                             interpolate_pos_encoding=ipe)
        for l in LAYERS:
            hs = vo.hidden_states[l]
            out[f"vision_hidden_{l}_{k}"] = torch.cat([hs[:1, :5], hs[:1, -5:]], dim=1).numpy()  # first image
        for l in ATTN_LAYERS:
            out[f"vision_attn_{l}_{k}"] = vo.attentions[l][:1, :, :4].numpy()                     # [1, 12, 4, S]
        print(k, "S =", vo.hidden_states[0].shape[1])
    path = os.path.join(ROOT, "tests", "golden", "vitb16_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
