"""Generate tests/golden/outputs_golden.npz from the live ``transformers.CLIPModel`` (fp32, CPU, eager attention):

    python tests/golden/make_outputs_golden.py

``vision_model`` / ``text_model`` with ``output_hidden_states=True, output_attentions=True`` on ``make_state_dict(0,
"rich")`` weights, for the cases of ``tests/outputs_oracle.py``: 2 images at 224 x 224, 1 image at 448 x 448
(``interpolate_pos_encoding``, ``plip_b200.synthetic.pixel_values_hw``) and 3 captions (``golden_text_inputs``: one
padding mask with a hole).  To stay small it keeps selected layers and rows:

- ``hidden_<l>``: layers ``GOLDEN_HIDDEN_LAYERS``, first image / all captions, the first and last rows
  (``golden_rows``: 5 for vision, 2 for text);
- ``last_hidden_state``: the same rows of every sequence; ``pooler_output`` in full;
- ``attn_<l>``: layers ``GOLDEN_ATTN_LAYERS``, every sequence and head, query rows ``golden_rows(S, 1)`` (vision: the
  CLS row and the last patch) or ``golden_rows(S, 2)`` (text), all keys.

Only outputs are stored: weights and inputs are regenerated from their seeds at test time.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import outputs_oracle as OO  # noqa: E402
from oracle import weights  # noqa: E402
from plip_b200.synthetic import pixel_values_hw  # noqa: E402


def _select(out, key, S, hidden_rows, attn_rows):
    hs, at = out.hidden_states, out.attentions
    sel = {}
    for l in OO.GOLDEN_HIDDEN_LAYERS:
        sel[f"{key}_hidden_{l}"] = hs[l][:, hidden_rows].numpy() if key == "text" else hs[l][:1, hidden_rows].numpy()
    sel[f"{key}_last_hidden_state"] = out.last_hidden_state[:, hidden_rows].numpy()
    sel[f"{key}_pooler_output"] = out.pooler_output.numpy()
    for l in OO.GOLDEN_ATTN_LAYERS:
        sel[f"{key}_attn_{l}"] = at[l][:, :, attn_rows].numpy()
    return sel


def main():
    import transformers
    from transformers import CLIPConfig, CLIPModel

    torch.set_grad_enabled(False)
    sd = weights.make_state_dict(0, "rich")
    hf = CLIPModel._from_config(CLIPConfig(), attn_implementation="eager").eval()
    hf.load_state_dict(sd, strict=True)
    out = {"transformers_version": np.array(transformers.__version__), "torch_version": np.array(torch.__version__)}
    for key, (n, size) in OO.GOLDEN_CASES.items():
        px = pixel_values_hw(n, size, size)
        vo = hf.vision_model(pixel_values=px, output_hidden_states=True, output_attentions=True,
                             interpolate_pos_encoding=size != 224)
        S = vo.last_hidden_state.shape[1]
        out.update(_select(vo, key, S, OO.golden_rows(S, 5), OO.golden_rows(S, 1)))
        print(key, "S =", S)
    ids, mask = OO.golden_text_inputs()
    to = hf.text_model(input_ids=ids, attention_mask=mask, output_hidden_states=True, output_attentions=True)
    out.update(_select(to, "text", 77, OO.golden_rows(77, 2), OO.golden_rows(77, 2)))
    path = os.path.join(ROOT, "tests", "golden", "outputs_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
