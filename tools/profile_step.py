"""Run a few vision (and text) forwards at batch 1024 for a profiler to attach to (no timing here)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import weights
from plip_b200.engine import Engine

which = sys.argv[1] if len(sys.argv) > 1 else "vision"
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 3
sd = weights.make_state_dict(0)
eng = Engine(sd, max_micro_batch=1024)
if which == "vision":
    x = torch.randn(1024, 3, 224, 224, device="cuda", dtype=torch.bfloat16)
    for _ in range(iters):
        eng.encode_images(x)
else:
    from oracle import synth
    ids, _ = synth.token_ids(1024, full_length=True)
    ids = ids.cuda()
    for _ in range(iters):
        eng.encode_text(ids)
torch.cuda.synchronize()
print("done")
