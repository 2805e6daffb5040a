"""Time plip_similarity_topk on a cfg5-rank-sized problem (10,000 queries x 125,000 gallery rows, k = 50; the
tensor-core score chunks + row merge), and check the result against torch."""
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from plip_b200.engine import similarity_topk  # noqa: E402

n, m, k = int(sys.argv[1]) if len(sys.argv) > 1 else 10000, int(sys.argv[2]) if len(sys.argv) > 2 else 125000, 50
g = torch.Generator().manual_seed(0)
q = torch.randn(n, 512, generator=g).cuda()
s = torch.randn(m, 512, generator=g).cuda()
q = q / q.norm(dim=1, keepdim=True)
s = s / s.norm(dim=1, keepdim=True)
if os.environ.get("TOPK_DUP"):      # a gallery drawn cyclically from 8192 distinct rows (what bench.py --config cfg5 uses): exact ties
    s = s[:8192].repeat((m + 8191) // 8192, 1)[:m].contiguous()
for _ in range(2):
    idx, val = similarity_topk(q, s, k, normalize_query=False)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(3):
    idx, val = similarity_topk(q, s, k, normalize_query=False)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 3
ref = (q[:64].double() @ s.double().t()).topk(k, dim=1)
ok_v = (val[:64].double() - ref.values).abs().max().item()
mism = (idx[:64].long() != ref.indices).float().mean().item()
print(f"similarity_topk n={n} m={m} k={k}: {ms:.2f} ms  |dval| {ok_v:.2e}  index mismatch rate {mism:.4f}")
