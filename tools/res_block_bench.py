"""The SD-v1.5 UNet's ResBlock (512 px, batch 8, time width 1280) on one GPU: ResidualBlockWithTimeEmbeddingB200 against eager bf16
autocast of the same math (oracle/unet_oracle.py::res_block) run NCHW, as the reference runs it, and channels-last, cuDNN's strong
case; then each 3x3 convolution alone (forward, input gradient, weight gradient) against cuDNN on channels-last bf16.

    python tools/res_block_bench.py [--reps 20] [--batch 8]

Shapes cover the down path, the middle and the widest skip concatenations of the up path: 320->320 and 960->320 at 64x64,
320->640 and 1920->640 at 32x32, 640->1280 and 2560->1280 at 16x16, 1280->1280 and 2560->1280 at 8x8.  Prints one JSON line per
measurement with the card's name, power limit and median SM clock.  FLOPs count the two 3x3 convolutions and the 1x1 shortcut
(2 M N K each); forward + backward is 3x the forward.
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
from cflearn_b200.unet_blocks import ResidualBlockWithTimeEmbeddingB200  # noqa: E402

DEV = torch.device("cuda", 0)
SHAPES = [(320, 320, 64), (960, 320, 64), (320, 640, 32), (1920, 640, 32), (640, 1280, 16), (2560, 1280, 16), (1280, 1280, 8),
          (2560, 1280, 8)]
TDIM = 1280
CL = torch.channels_last


def block_flops(B: int, Cin: int, Cout: int, side: int) -> float:
    M = B * side * side
    fl = 2.0 * M * Cout * 9 * Cin + 2.0 * M * Cout * 9 * Cout
    return fl + (2.0 * M * Cout * Cin if Cin != Cout else 0.0)


def tflops(flop: float, ms: float) -> float:
    return round(flop / (ms * 1e-3) / 1e12, 1)


def bench_block(B: int, Cin: int, Cout: int, side: int, reps: int) -> None:
    m = ResidualBlockWithTimeEmbeddingB200(Cin, Cout, norm_eps=1e-5, time_embedding_channels=TDIM)
    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=Cin + Cout + side)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV)
    sdd = {k: v.to(DEV).requires_grad_(True) for k, v in sd.items()}
    g = torch.Generator().manual_seed(1)
    net = torch.randn(B, Cin, side, side, generator=g).to(DEV).to(torch.bfloat16)
    tn = torch.randn(B, TDIM, generator=g).to(DEV).to(torch.bfloat16)
    up = torch.randn(B, Cout, side, side, generator=g).to(DEV).to(torch.bfloat16)
    inputs = {"cl": (net.contiguous(memory_format=CL), up.contiguous(memory_format=CL)), "nchw": (net.contiguous(), up.contiguous())}
    leaves = {k: (x.clone().requires_grad_(True), tn.clone().requires_grad_(True)) for k, (x, _) in inputs.items()}

    def ours_fwd():
        with torch.no_grad():
            m(inputs["cl"][0], tn)

    def ours_step():
        x, t = leaves["cl"]
        m(x, t).backward(inputs["cl"][1])

    def eager(fmt, step):
        def run():
            x, t = leaves[fmt]
            if not step:
                with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                    uo.res_block(sdd, "", inputs[fmt][0], tn)
                return
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = uo.res_block(sdd, "", x, t)
            y.backward(inputs[fmt][1])
        return run

    fns = {"ours_fwd": ours_fwd, "eager_nchw_fwd": eager("nchw", False), "eager_cl_fwd": eager("cl", False),
           "ours_step": ours_step, "eager_nchw_step": eager("nchw", True), "eager_cl_step": eager("cl", True)}
    sampler = ClockSampler(DEV.index)
    sampler.start()
    t = {name: time_ms(fn, reps) for name, fn in fns.items()}
    clocks = sampler.stop()
    fl = block_flops(B, Cin, Cout, side)
    emit({"run": "res_block", "B": B, "Cin": Cin, "Cout": Cout, "side": side,
          "fwd_ms": {"ours": round(t["ours_fwd"], 3), "eager_nchw": round(t["eager_nchw_fwd"], 3), "eager_cl": round(t["eager_cl_fwd"], 3)},
          "fwd_bwd_ms": {"ours": round(t["ours_step"], 3), "eager_nchw": round(t["eager_nchw_step"], 3),
                         "eager_cl": round(t["eager_cl_step"], 3)},
          "fwd_tflops": {"ours": tflops(fl, t["ours_fwd"]), "eager_cl": tflops(fl, t["eager_cl_fwd"])},
          "fwd_bwd_tflops": {"ours": tflops(3 * fl, t["ours_step"]), "eager_cl": tflops(3 * fl, t["eager_cl_step"])},
          "note": "CUDA events; fwd without autograd; fwd_bwd includes parameter-gradient accumulation on both sides"}, clocks)


def bench_conv(B: int, Cin: int, Cout: int, side: int, reps: int) -> None:
    """conv1 of the block (Cin -> Cout) alone: ours vs F.conv2d / cuDNN's backward on channels-last bf16."""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(B, side, side, Cin, generator=g).to(DEV).to(torch.bfloat16)       # NHWC
    dy = torch.randn(B, side, side, Cout, generator=g).to(DEV).to(torch.bfloat16)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).to(DEV)
    b = (torch.randn(Cout, generator=g) * 0.02).to(DEV).to(torch.bfloat16)
    wp, wd = ops.pack_conv3x3_weight(w), ops.pack_conv3x3_weight_dgrad(w)
    wb = w.to(torch.bfloat16).contiguous(memory_format=CL)
    xc, dyc = x.permute(0, 3, 1, 2), dy.permute(0, 3, 1, 2)  # channels-last NCHW views of the same memory
    wpart = torch.empty(Cout, 9 * Cin, dtype=torch.float32, device=DEV)

    def cudnn_bwd(mask):
        return lambda: torch.ops.aten.convolution_backward(dyc, xc, wb, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, mask)

    fns = {"fwd_ours": lambda: ops.conv3x3(x, wp, b), "fwd_cudnn": lambda: F.conv2d(xc, wb, b, padding=1),
           "dgrad_ours": lambda: ops.conv3x3(dy, wd), "dgrad_cudnn": cudnn_bwd([True, False, False]),
           "wgrad_ours": lambda: ops.conv3x3_wgrad(dy, x, wpart), "wgrad_cudnn": cudnn_bwd([False, True, False])}
    sampler = ClockSampler(DEV.index)
    sampler.start()
    t = {name: time_ms(fn, reps) for name, fn in fns.items()}
    clocks = sampler.stop()
    fl = 2.0 * B * side * side * Cout * 9 * Cin
    emit({"run": "conv3x3", "B": B, "Cin": Cin, "Cout": Cout, "side": side,
          "ms": {k: round(v, 4) for k, v in t.items()}, "tflops": {k: tflops(fl, v) for k, v in t.items()},
          "note": "CUDA events; cuDNN on channels-last bf16 (F.conv2d / aten.convolution_backward); ours: the implicit-GEMM kernels; "
                  "wgrad_ours includes the split-K reduction"}, clocks)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("res_block_bench needs a GPU")
    torch.backends.cudnn.benchmark = True  # cuDNN picks its best algorithm per shape during the warm-up
    for Cin, Cout, side in SHAPES:
        bench_block(args.batch, Cin, Cout, side, args.reps)
    for Cin, Cout, side in SHAPES:
        bench_conv(args.batch, Cin, Cout, side, max(args.reps, 50))


if __name__ == "__main__":
    main()
