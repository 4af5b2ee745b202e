"""The SD-v1.5 UNet's attention shapes (512 px, batch 8, 8 heads) on one GPU: ops.cross_attention_fwd/_bwd against torch's flash SDPA.

    python tools/unet_attn_bench.py [--reps 30] [--batch 8]

Self-attention at (T, Dh) = (4096, 40), (1024, 80), (256, 160), (64, 160), and cross-attention at the same Tq with a 77-token
context.  Both sides get contiguous [B*H, T, Dh] operands (ours reads them as B*H images of one head, SDPA as
[B, H, T, Dh]).  Prints one JSON line per shape with the card's name, power limit and median SM clock read during that measurement.  FLOP conventions are bench.py's:
forward 4 B H Tq Tk Dh, backward 10 B H Tq Tk Dh.
"""
from __future__ import annotations

import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from torch.nn.attention import SDPBackend, sdpa_kernel  # noqa: E402

from bench import ClockSampler  # noqa: E402
from long_seq_bench import emit, time_ms  # noqa: E402

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import ops  # noqa: E402

DEV = torch.device("cuda", 0)
LEVELS = [(4096, 40), (1024, 80), (256, 160), (64, 160)]
CONTEXT = 77


def bench(B: int, H: int, Tq: int, Tk: int, Dh: int, reps: int) -> None:
    BH = B * H
    g = torch.Generator(device="cpu").manual_seed(Tq + Tk + Dh)
    q, k, v = (torch.randn(BH, t, Dh, generator=g).to(torch.bfloat16).to(DEV) for t in (Tq, Tk, Tk))
    dout = torch.randn(BH, Tq, Dh, generator=g).to(torch.bfloat16).to(DEV)
    q2, k2, v2, do2 = q.view(BH * Tq, Dh), k.view(BH * Tk, Dh), v.view(BH * Tk, Dh), dout.view(BH * Tq, Dh)
    dq, dk, dv = torch.empty_like(q2), torch.empty_like(k2), torch.empty_like(v2)
    sampler = ClockSampler(DEV.index)
    sampler.start()
    out, lse = ops.cross_attention_fwd(q2, k2, v2, BH, 1)
    f_ours = time_ms(lambda: ops.cross_attention_fwd(q2, k2, v2, BH, 1), reps)
    b_ours = time_ms(lambda: ops.cross_attention_bwd(q2, k2, v2, out, do2, lse, BH, 1, dq=dq, dk=dk, dv=dv), reps)
    # the same bytes as [B, H, T, Dh] (torch's flash kernel takes 4-D operands)
    qs, ks, vs = (t.view(B, H, -1, Dh).clone().requires_grad_(True) for t in (q, k, v))
    do4 = dout.view(B, H, Tq, Dh)
    with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
        f_sdpa = time_ms(lambda: F.scaled_dot_product_attention(qs, ks, vs), reps)
        o = F.scaled_dot_product_attention(qs, ks, vs)
        b_sdpa = time_ms(lambda: torch.autograd.grad(o, (qs, ks, vs), do4, retain_graph=True), reps)
    clocks = sampler.stop()
    ff, fb = 4.0 * BH * Tq * Tk * Dh, 10.0 * BH * Tq * Tk * Dh
    tf = lambda flop, ms: round(flop / (ms * 1e-3) / 1e12, 1)  # noqa: E731
    emit({"run": "unet_attention", "kind": "self" if Tq == Tk else "cross", "B": B, "H": H, "Tq": Tq, "Tk": Tk, "Dh": Dh,
          "fwd_ms": {"ours": round(f_ours, 4), "sdpa_flash": round(f_sdpa, 4)},
          "bwd_ms": {"ours": round(b_ours, 4), "sdpa_flash": round(b_sdpa, 4)},
          "fwd_tflops": {"ours": tf(ff, f_ours), "sdpa_flash": tf(ff, f_sdpa)},
          "bwd_tflops": {"ours": tf(fb, b_ours), "sdpa_flash": tf(fb, b_sdpa)},
          "note": "CUDA events over the launches; sdpa bwd is autograd.grad of its flash forward (includes the grad allocations)"},
         clocks)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--batch", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unet_attn_bench needs a GPU")
    for T, Dh in LEVELS:
        for Tk in (T, CONTEXT):
            bench(args.batch, 8, T, Tk, Dh, args.reps)


if __name__ == "__main__":
    main()
