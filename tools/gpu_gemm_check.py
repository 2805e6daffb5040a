"""GPU bring-up check of the wgmma GEMM.  Each case runs in its own
subprocess under a timeout so a trap / hang in one configuration cannot take the others down."""
import json
import subprocess
import sys
import time

CASES = [
    # cg, bn, epi, M, N, K
    (1, 128, 4, 128, 128, 64),
    (1, 128, 4, 256, 256, 256),
    (1, 256, 4, 300, 512, 768),
    (2, 128, 4, 256, 128, 64),
    (2, 256, 4, 512, 512, 768),
    (2, 256, 4, 1000, 768, 3072),
    (1, 256, 0, 1000, 768, 768),
    (2, 256, 1, 1000, 3072, 768),
    (2, 256, 2, 1000, 768, 3072),
    (2, 256, 3, 980, 768, 3072),
    (1, 256, 4, 51200, 768, 768),
    (2, 256, 4, 51200, 768, 768),
    (1, 256, 0, 51200, 2304, 768),
    (2, 256, 0, 51200, 2304, 768),
    (2, 256, 1, 51200, 3072, 768),
    (2, 256, 2, 51200, 768, 3072),
    (1, 256, 2, 51200, 768, 3072),
    (2, 128, 2, 51200, 768, 3072),
]


def run_case(cg, bn, epi, M, N, K):
    import torch
    from plip_b200._lib import lib, check
    L = lib(strict=False)
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(1)
    A = (torch.randn(M, K, generator=g) * 0.5).to(dev).to(torch.bfloat16)
    W = (torch.randn(N, K, generator=g) * 0.05).to(dev).to(torch.bfloat16)
    bias = torch.randn(N, generator=g).to(dev)
    pos = torch.randn(50, N, generator=g).to(dev)
    ref = A.float() @ W.float().t()
    if epi in (0, 1, 2):
        ref = ref + bias
    if epi == 1:
        ref = ref * torch.sigmoid(1.702 * ref)
    if epi in (0, 1):
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    elif epi == 2:
        x0 = torch.randn(M, N, generator=g).to(dev)
        out = x0.clone()
        ref = ref + x0
    elif epi == 3:
        nb = M // 49
        out = torch.zeros(nb * 50, N, device=dev)
        r = torch.zeros(nb * 50, N, device=dev)
        r.view(nb, 50, N)[:, 1:, :] = ref.view(nb, 49, N) + pos[1:]
        ref = r
    else:
        out = torch.zeros(M, N, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def call():
        check(L.plip_dbg_gemm(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(), out.data_ptr(), N,
                              pos.data_ptr(), epi, cg, bn, None, None, 0, None, None, stream), "gemm")
    call()
    torch.cuda.synchronize()
    err = 0.0 if epi == 7 else (out.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    res = {"cg": cg, "bn": bn, "epi": epi, "M": M, "N": N, "K": K, "max_abs_err": err, "ref_max": scale}
    if M >= 10000 and epi != 2:
        for _ in range(3):
            call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 20
        res["ms"] = ms
        res["tflops"] = 2.0 * M * N * K / ms / 1e9
    elif M >= 10000:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        res["ms"] = ms
        res["tflops"] = 2.0 * M * N * K / ms / 1e9
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1:
        run_case(*map(int, sys.argv[1:]))
        sys.exit(0)
    for c in CASES:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, __file__, *map(str, c)], capture_output=True, text=True, timeout=120)
            out = (r.stdout.strip().splitlines() or ["<no output>"])[-1]
            tail = r.stderr.strip().splitlines()[-3:] if r.returncode != 0 else []
            print(f"case {c} rc={r.returncode} {time.time()-t0:.1f}s: {out} {' | '.join(tail)}", flush=True)
        except subprocess.TimeoutExpired:
            print(f"case {c} TIMEOUT", flush=True)
