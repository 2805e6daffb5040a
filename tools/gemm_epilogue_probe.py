"""Where the layer GEMMs of the default benchmark step spend their time: each of the 8 shapes (vision M = 51 200,
D = 768; text M = 78 848, D = 512; QKV, out_proj, fc1, fc2) timed through plip_dbg_gemm with its real epilogue and
with EPI_NULL (main loop only, accumulators dropped).  The difference is the epilogue time the main loop does not
hide.  CUDA events over short bursts (best of several, as bench.py's kernel_bursts); TFLOP/s, and GB/s by the byte
rule of the in-step profile (engine.cu: A + W + the output, 8 bytes per fp32 residual element, + the 16-bit copy).
GPU only: without CUDA it exits with an error.

    python tools/gemm_epilogue_probe.py [--root DIR] [--json out.json]

--root DIR imports plip_b200 (and its built library) from another tree, e.g. a build of an earlier commit, so two
builds can be compared in one run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

EPI_RESID, EPI_LN, EPI_LN_GELU, EPI_NULL = 2, 5, 6, 7
SHAPES = [  # (tower, role, epilogue, M, N, K)
    ("vision", "ln1+qkv", EPI_LN, 51200, 2304, 768),
    ("vision", "out_proj+resid", EPI_RESID, 51200, 768, 768),
    ("vision", "ln2+fc1+gelu", EPI_LN_GELU, 51200, 3072, 768),
    ("vision", "fc2+resid", EPI_RESID, 51200, 768, 3072),
    ("text", "ln1+qkv", EPI_LN, 78848, 1536, 512),
    ("text", "out_proj+resid", EPI_RESID, 78848, 512, 512),
    ("text", "ln2+fc1+gelu", EPI_LN_GELU, 78848, 2048, 512),
    ("text", "fc2+resid", EPI_RESID, 78848, 512, 2048),
]
BURSTS, PER_BURST = 8, 5


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as ex:  # the timings stay valid; the card line says what could not be read
        info["power_limit"] = f"unknown ({ex})"
    return info


def bursts(call):
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    res = []
    for _ in range(BURSTS):
        time.sleep(0.03)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(PER_BURST):
            call()
        e1.record()
        torch.cuda.synchronize()
        res.append(e0.elapsed_time(e1) / PER_BURST * 1e3)
    return min(res), statistics.median(res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_epilogue_probe: needs a CUDA device")
    sys.path.insert(0, os.path.abspath(args.root))
    from plip_b200._lib import check, lib
    L = lib(strict=True)
    torch.manual_seed(0)
    stream = torch.cuda.current_stream().cuda_stream
    report = {"card": card(), "root": os.path.abspath(args.root), "shapes": []}
    print(json.dumps({"card": report["card"]}), flush=True)
    for tower, role, epi, M, N, K in SHAPES:
        A = torch.randn(M, K, device="cuda").to(torch.bfloat16)
        W = (torch.randn(N, K, device="cuda") * 0.03).to(torch.bfloat16)
        bias = torch.randn(N, device="cuda") * 0.1
        colsum = W.float().sum(1).contiguous()
        stats = torch.zeros(M, 8, 2, device="cuda")
        stats[:, 0, 1] = float(K)                        # mean 0, var 1 -> rstd ~ 1
        resid = epi == EPI_RESID
        out = torch.randn(M, N, device="cuda") if resid else torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        xb = torch.empty(M, N, device="cuda", dtype=torch.bfloat16) if resid else None
        st_out = torch.empty(M, 8, 2, device="cuda") if resid else None
        ln = epi in (EPI_LN, EPI_LN_GELU)

        def call(e):
            real = e != EPI_NULL
            check(L.plip_dbg_gemm(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(), out.data_ptr(), N, None, e,
                                  0, 0, colsum.data_ptr() if ln else None, stats.data_ptr() if ln else None,
                                  1 if ln else 0, xb.data_ptr() if real and resid else None,
                                  st_out.data_ptr() if real and resid else None, stream), "gemm")

        us, us_med = bursts(lambda: call(epi))
        us_null, us_null_med = bursts(lambda: call(EPI_NULL))
        out_elem = 8 if resid else 2
        nbytes = M * K * 2 + N * K * 2 + M * N * out_elem + (M * N * 2 if resid else 0)
        row = {"tower": tower, "role": role, "epi": epi, "M": M, "N": N, "K": K,
               "us": round(us, 1), "us_median": round(us_med, 1), "us_main_loop": round(us_null, 1),
               "us_main_loop_median": round(us_null_med, 1), "us_exposed_epilogue": round(us - us_null, 1),
               "tflops": round(2.0 * M * N * K / us / 1e6, 1), "GBps": round(nbytes / us / 1e3, 1),
               "tflops_main_loop": round(2.0 * M * N * K / us_null / 1e6, 1)}
        report["shapes"].append(row)
        print(json.dumps(row), flush=True)
        del A, W, out, xb, st_out, stats
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            f.write(json.dumps(report) + "\n")


if __name__ == "__main__":
    main()
