"""The SD-v1.5 UNet's six resampling layers (512 px, batch 8) on one GPU: forward, input gradient and weight gradient of ours against
cuDNN (eager bf16, NCHW and channels-last, cudnn.benchmark on), and the fused upsampling convolution against a nearest copy followed
by our stride-1 convolution.

    python tools/resample_bench.py [--reps 50] [--batch 8]

Down: ResDownsample at 64x64 / 320, 32x32 / 640, 16x16 / 1280 (input sizes).  Up: ResUpsample at 8x8 / 1280, 16x16 / 1280,
32x32 / 640 (input sizes).  Eager's upsampling layer is F.interpolate then F.conv2d; its input gradient the convolution's input
gradient then interpolate's backward; its weight gradient the convolution's on the upsampled input.  Ours: the fused forward
(conv3x3_up2), the stride-1 input gradient at 2H x 2W then sum2x2, the nearest copy then the stride-1 weight gradient.  One JSON
line per layer, with the card's name, power limit and median SM clock.
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

from bench import ClockSampler  # noqa: E402
from long_seq_bench import emit, time_ms  # noqa: E402

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import ops  # noqa: E402

DEV = torch.device("cuda", 0)
CL = torch.channels_last
LAYERS = [(False, 64, 320), (False, 32, 640), (False, 16, 1280), (True, 8, 1280), (True, 16, 1280), (True, 32, 640)]


def bench_layer(B: int, up: bool, side: int, C: int, reps: int) -> None:
    g = torch.Generator().manual_seed(side + C)
    so = 2 * side if up else side // 2                    # output side
    x = torch.randn(B, side, side, C, generator=g).to(DEV).to(torch.bfloat16)  # NHWC
    dy = torch.randn(B, so, so, C, generator=g).to(DEV).to(torch.bfloat16)
    w = (torch.randn(C, C, 3, 3, generator=g) * (9 * C) ** -0.5).to(DEV)
    b = (torch.randn(C, generator=g) * 0.02).to(DEV).to(torch.bfloat16)
    bias_rows = b.expand(B, C).contiguous()
    wp, wd = ops.pack_conv3x3_weight(w), ops.pack_conv3x3_weight_dgrad(w)
    wd2 = ops.pack_conv3x3_weight_s2_dgrad(w)
    wpart = torch.empty(C, 9 * C, dtype=torch.float32, device=DEV)
    epi = ops.EPI_BIAS_ADD_PER_IMAGE_BF16
    stride = [1, 1] if up else [2, 2]
    fmts = {"cl": (x.permute(0, 3, 1, 2), dy.permute(0, 3, 1, 2), w.to(torch.bfloat16).contiguous(memory_format=CL)),
            "nchw": (x.permute(0, 3, 1, 2).contiguous(), dy.permute(0, 3, 1, 2).contiguous(), w.to(torch.bfloat16).contiguous())}

    def eager(fmt, what):
        xe, dye, we = fmts[fmt]
        if what == "fwd":
            if up:
                return lambda: F.conv2d(F.interpolate(xe, scale_factor=2, mode="nearest"), we, b, padding=1)
            return lambda: F.conv2d(xe, we, b, stride=2, padding=1)
        mask = [what == "dgrad", what == "wgrad", False]
        if not up:
            return lambda: torch.ops.aten.convolution_backward(dye, xe, we, None, stride, [1, 1], [1, 1], False, [0, 0], 1, mask)
        if what == "wgrad":
            return lambda: torch.ops.aten.convolution_backward(dye, F.interpolate(xe, scale_factor=2, mode="nearest"), we, None, stride,
                                                               [1, 1], [1, 1], False, [0, 0], 1, mask)
        xu = F.interpolate(xe, scale_factor=2, mode="nearest")
        return lambda: torch.ops.aten.upsample_nearest2d_backward(
            torch.ops.aten.convolution_backward(dye, xu, we, None, stride, [1, 1], [1, 1], False, [0, 0], 1, mask)[0],
            [2 * side, 2 * side], list(xe.shape), 2.0, 2.0)

    if up:
        ours = {"fwd": lambda: ops.conv3x3_up2(x, wp, epilogue=epi, aux=bias_rows),
                "fwd_unfused": lambda: ops.conv3x3(ops.upsample_nearest2x(x), wp, epilogue=epi, aux=bias_rows),
                "dgrad": lambda: ops.sum2x2(ops.conv3x3(dy, wd)),
                "wgrad": lambda: ops.conv3x3_wgrad(dy, ops.upsample_nearest2x(x), wpart)}
    else:
        ours = {"fwd": lambda: ops.conv3x3_s2(x, wp, epilogue=epi, aux=bias_rows),
                "dgrad": lambda: ops.conv3x3_s2_dgrad(dy, wd2),
                "wgrad": lambda: ops.conv3x3_s2_wgrad(dy, x, wpart)}
    fns = {f"{k}_ours": fn for k, fn in ours.items()}
    for what in ("fwd", "dgrad", "wgrad"):
        for fmt in ("cl", "nchw"):
            fns[f"{what}_cudnn_{fmt}"] = eager(fmt, what)
    sampler = ClockSampler(DEV.index)
    sampler.start()
    t = {name: time_ms(fn, reps) for name, fn in fns.items()}
    # the fused / unfused decision: alternate the two, a second time, in the same process
    if up:
        t["fwd_ours_again"] = time_ms(ours["fwd"], reps)
        t["fwd_unfused_ours_again"] = time_ms(ours["fwd_unfused"], reps)
    clocks = sampler.stop()
    fl = 2.0 * B * so * so * C * 9 * C
    emit({"run": "resample", "layer": "up" if up else "down", "B": B, "side": side, "C": C,
          "ms": {k: round(v, 4) for k, v in t.items()}, "tflops": {k: round(fl / (v * 1e-3) / 1e12, 1) for k, v in t.items()},
          "note": "CUDA events; cuDNN bf16 via F.conv2d / aten.convolution_backward; ours' wgrad includes the split-K reduction"}, clocks)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--batch", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resample_bench needs a GPU")
    torch.backends.cudnn.benchmark = True  # cuDNN picks its best algorithm per shape during the warm-up
    for up, side, C in LAYERS:
        bench_layer(args.batch, up, side, C, args.reps)


if __name__ == "__main__":
    main()
