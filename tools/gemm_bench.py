"""Micro-benchmark of the wgmma GEMM: operand majors x shapes against cuBLAS, on one GPU (same clocks); then the FeedForward's
two GELU epilogues against the plain bias epilogue at the same shape and majors (the difference is what the fusion costs).

    python tools/gemm_bench.py [--epilogues-only]      (B200_LIB_PATH=<other build> times another build of the library)
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import _cabi, ops  # noqa: E402

dev = "cuda"


def timeit(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def majors_sweep():
    shapes = [(50432, 2304, 768), (50432, 768, 768), (50432, 3072, 768), (50432, 768, 3072)]
    for (M, N, K) in shapes:
        a = torch.randn(M, K, device=dev).to(torch.bfloat16)
        b = (torch.randn(N, K, device=dev) * 0.02).to(torch.bfloat16)
        at, bt = a.t().contiguous(), b.t().contiguous()
        bias = torch.zeros(N, device=dev, dtype=torch.bfloat16)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        res = []
        for a_mn, b_mn in ((0, 0), (0, 1), (1, 0), (1, 1)):
            ms = timeit(lambda: ops.gemm(at if a_mn else a, bt if b_mn else b, a_mn_major=bool(a_mn), b_mn_major=bool(b_mn), bias=bias, out0=out))
            res.append(f"A{'mn' if a_mn else 'k'}B{'mn' if b_mn else 'k'} {ms*1e3:6.1f}us {2*M*N*K/ms/1e9:6.0f}TF")
        ref = timeit(lambda: torch.matmul(a, b.t()))
        print(f"{M}x{N}x{K}: " + " | ".join(res) + f" | cuBLAS {ref*1e3:6.1f}us {2*M*N*K/ref/1e9:6.0f}TF", flush=True)


def gelu_epilogues(reps=50):
    # ViT-B/16 at batch 256: FF1 forward (majors (0,0), bias + GELU with the dual output) and the FF2 dgrad through GELU
    # (majors (0,1), dGELU on aux = h).  Inputs are scaled like the step's (h ~ N(0, 1)), and plain and fused alternate.
    M, N, K = 50432, 3072, 768
    a = torch.randn(M, K, device=dev).to(torch.bfloat16)
    w = (torch.randn(N, K, device=dev) / K ** 0.5).to(torch.bfloat16)
    wt = w.t().contiguous()
    bias = (torch.randn(N, device=dev) * 0.02).to(torch.bfloat16)
    h = torch.randn(M, N, device=dev).to(torch.bfloat16)
    out0 = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    out1 = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    rows = {
        "ff1 (0,0)": (lambda: ops.gemm(a, w, bias=bias, out0=out0),
                      lambda: ops.gemm(a, w, bias=bias, epilogue=ops.EPI_BIAS_GELU_BF16, out0=out0, out1=out1), "bias+GELU dual"),
        "ff2-dgrad (0,1)": (lambda: ops.gemm(a, wt, b_mn_major=True, out0=out0),
                            lambda: ops.gemm(a, wt, b_mn_major=True, epilogue=ops.EPI_DGELU_BF16, out0=out0, aux=h), "dGELU"),
    }
    for name, (plain, fused, what) in rows.items():
        tp, tf = [], []
        for _ in range(3):
            tp.append(timeit(plain, reps))
            tf.append(timeit(fused, reps))
        p, f = sorted(tp)[1], sorted(tf)[1]
        fl = 2.0 * M * N * K
        print(f"{M}x{N}x{K} {name}: plain {p*1e3:6.1f}us {fl/p/1e9:4.0f}TF | {what} {f*1e3:6.1f}us {fl/f/1e9:4.0f}TF | "
              f"fused - plain {(f-p)*1e3:6.1f}us ({f/p:.3f}x)   [medians of 3 x {reps} launches]", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epilogues-only", action="store_true", help="skip the operand-majors sweep")
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    print(f"card: {smi.stdout.strip()}; library {_cabi.LIB_PATH}", flush=True)
    if not args.epilogues_only:
        majors_sweep()
    gelu_epilogues()


if __name__ == "__main__":
    main()
