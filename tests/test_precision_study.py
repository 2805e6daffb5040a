"""The CPU emulation behind DESIGN.md §2 stays runnable and keeps telling the same
story on a tiny sample: fp16 operands beat bf16 by ~an order of magnitude in logits error, the 3-term split is exact
to ~1e-5, and the LayerNorm fold does not cost accuracy on the outlier weights."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_precision_study_tool(tmp_path):
    out = tmp_path / "ps.json"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "precision_study.py"), "--images", "4", "--captions", "4",
                        "--modes", "outlier", "--out", str(out)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    rows = {x["config"]: x for x in json.load(open(out))["outlier"]["rows"]}
    bf_fold = rows["act=bf16 wgt=bf16 attn=bf16 fold=True"]
    bf_plain = rows["act=bf16 wgt=bf16 attn=bf16 fold=False"]
    fp = rows["act=fp16 wgt=fp16 attn=fp16 fold=True"]
    split3 = rows["act=fp16x2 wgt=fp16x2 attn=fp16x2 fold=True"]
    assert bf_fold["one_minus_cos_image_max"] < 1e-4 and bf_fold["one_minus_cos_text_max"] < 1e-4        # north_star cosine bar
    assert bf_fold["one_minus_cos_image_max"] < 3 * bf_plain["one_minus_cos_image_max"] + 1e-7            # the fold is free
    assert fp["dlogits_mean"] < 0.5 * bf_fold["dlogits_mean"]
    assert split3["dlogits_max"] < 1e-4 < bf_fold["dlogits_max"]
