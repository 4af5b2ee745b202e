"""The SD-v1.5 UNet's SpatialTransformer (512 px, batch 8, 77 x 768 context) on one GPU: SpatialTransformerB200 against eager bf16
autocast of the same math (oracle/unet_oracle.py::spatial_transformer, whose attention is torch's SDPA), and the GEGLU GEMM alone
against the plain bias GEMM followed by torch's chunk / gelu / mul.

    python tools/spatial_transformer_bench.py [--reps 20] [--batch 8]

Shapes: C 320 at 64x64 (Dh 40), C 640 at 32x32 (Dh 80), C 1280 at 16x16 (Dh 160) and the middle block, C 1280 at 8x8; 8 heads,
one block each.  Prints one JSON line per measurement with the card's name, power limit and median SM clock.  FLOPs count the
GEMMs (2 M N K each) and attention (4 B H Tq Tk Dh forward); forward + backward is 3x the forward.
"""
from __future__ import annotations

import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench import ClockSampler  # noqa: E402
from long_seq_bench import emit, time_ms  # noqa: E402

import cflearn_b200  # noqa: F401,E402
import unet_oracle as uo  # noqa: E402
from cflearn_b200 import ops  # noqa: E402
from cflearn_b200.spatial_transformer import SpatialTransformerB200  # noqa: E402

DEV = torch.device("cuda", 0)
SHAPES = [(320, 64), (640, 32), (1280, 16), (1280, 8)]
CONTEXT, CONTEXT_DIM, HEADS = 77, 768, 8


def transformer_flops(B: int, C: int, side: int) -> float:
    M, T, F_ = B * side * side, side * side, 4 * C
    gemm = 2.0 * M * C * C * 2                       # to_latent, from_latent
    gemm += 2.0 * M * C * 3 * C + 2.0 * M * C * C     # attn1: qkv, out
    gemm += 2.0 * M * C * C * 2 + 2.0 * B * CONTEXT * CONTEXT_DIM * 2 * C  # attn2: q, out; kv of the context
    gemm += 2.0 * M * C * 2 * F_ + 2.0 * M * F_ * C   # GEGLU projection, FF2
    attn = 4.0 * B * C * T * (T + CONTEXT)            # 4 B H Tq Tk Dh for both attentions (H Dh = C)
    return gemm + attn


def bench_transformer(B: int, C: int, side: int, reps: int) -> None:
    m = SpatialTransformerB200(C, HEADS, C // HEADS, context_dim=CONTEXT_DIM).to(DEV)
    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=C + side)
    m.load_state_dict(sd, strict=True)
    sdd = {k: v.to(DEV).requires_grad_(True) for k, v in sd.items()}
    g = torch.Generator().manual_seed(1)
    net = torch.randn(B, C, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    ctx = torch.randn(B, CONTEXT, CONTEXT_DIM, generator=g).to(DEV)
    up = torch.randn(B, C, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    x = net.clone().requires_grad_(True)
    c = ctx.clone().requires_grad_(True)

    def ours_fwd():
        with torch.no_grad():
            m(net, ctx)

    def ours_step():
        m(x, c).backward(up)

    def eager_fwd():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            uo.spatial_transformer(sdd, "", net, ctx, HEADS)

    def eager_step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = uo.spatial_transformer(sdd, "", x, c, HEADS)
        y.backward(up)

    sampler = ClockSampler(DEV.index)
    sampler.start()
    t = {name: time_ms(fn, reps) for name, fn in (("ours_fwd", ours_fwd), ("eager_fwd", eager_fwd), ("ours_step", ours_step),
                                                  ("eager_step", eager_step))}
    clocks = sampler.stop()
    fl = transformer_flops(B, C, side)
    tf = lambda flop, ms: round(flop / (ms * 1e-3) / 1e12, 1)  # noqa: E731
    emit({"run": "spatial_transformer", "B": B, "C": C, "side": side, "Dh": C // HEADS,
          "fwd_ms": {"ours": round(t["ours_fwd"], 3), "eager_bf16": round(t["eager_fwd"], 3)},
          "fwd_bwd_ms": {"ours": round(t["ours_step"], 3), "eager_bf16": round(t["eager_step"], 3)},
          "fwd_tflops": {"ours": tf(fl, t["ours_fwd"]), "eager_bf16": tf(fl, t["eager_fwd"])},
          "fwd_bwd_tflops": {"ours": tf(3 * fl, t["ours_step"]), "eager_bf16": tf(3 * fl, t["eager_step"])},
          "speedup_fwd": round(t["eager_fwd"] / t["ours_fwd"], 2), "speedup_fwd_bwd": round(t["eager_step"] / t["ours_step"], 2),
          "note": "CUDA events; fwd without autograd; fwd_bwd includes parameter-gradient accumulation on both sides"}, clocks)


def bench_geglu(M: int, C: int, reps: int) -> None:
    F_ = 4 * C
    g = torch.Generator().manual_seed(2)
    x = torch.randn(M, C, generator=g).to(DEV).to(torch.bfloat16)
    w1 = (torch.randn(2 * F_, C, generator=g) * C ** -0.5).to(DEV).to(torch.bfloat16)
    b1 = (torch.randn(2 * F_, generator=g) * 0.02).to(DEV).to(torch.bfloat16)
    a = torch.empty(M, F_, dtype=torch.bfloat16, device=DEV)
    hg = torch.empty(M, 2 * F_, dtype=torch.bfloat16, device=DEV)

    def fused():
        ops.gemm(x, w1, bias=b1, epilogue=ops.EPI_BIAS_GEGLU_BF16, out0=hg, out1=a)

    def plain():
        ops.gemm(x, w1, bias=b1, out0=hg)

    def split():
        t = ops.gemm(x, w1, bias=b1, out0=hg)
        h, gate = t.chunk(2, dim=-1)
        return h * F.gelu(gate)

    sampler = ClockSampler(DEV.index)
    sampler.start()
    t = {name: time_ms(fn, reps) for name, fn in (("geglu_epilogue", fused), ("bias_gemm_alone", plain), ("bias_gemm+torch", split))}
    clocks = sampler.stop()
    fl = 2.0 * M * 2 * F_ * C
    emit({"run": "geglu_gemm", "M": M, "K": C, "N": 2 * F_,
          "ms": {k: round(v, 4) for k, v in t.items()},
          "tflops": {k: round(fl / (v * 1e-3) / 1e12, 1) for k, v in t.items()},
          "note": "CUDA events; tflops = the GEMM's 2 M N K over each variant's time"}, clocks)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spatial_transformer_bench needs a GPU")
    for C, side in SHAPES:
        bench_transformer(args.batch, C, side, args.reps)
    for C, side in SHAPES:
        bench_geglu(args.batch * side * side, C, max(args.reps, 50))


if __name__ == "__main__":
    main()
