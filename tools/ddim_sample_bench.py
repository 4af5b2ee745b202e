"""DDIM sampling with the SD-v1.5 UNet on one GPU: DDPMB200.decode (one CUDA-graph replay per denoising step) against eager bf16
autocast of oracle/unet_oracle.py::forward driven by oracle/ddim_oracle.py's loop.  Synthetic weights, 64 x 64 latents (512 px),
a 77 x 768 context, classifier-free guidance 7.5 with equal token counts (one UNet forward at batch 2B per step), 50 steps.

    python tools/ddim_sample_bench.py [--batches 1 4 8] [--steps 50] [--reps 3]

Rows per batch, each the median of --reps sampling calls timed with CUDA events after one warm-up call (which, for the native
row, captures the graph), the rows alternating:
  native      DDPMB200.decode
  eager       the oracle loop on eager autocast
Each row reports ms_per_step, s_per_batch and peak_mib (torch.cuda.max_memory_allocated over one call, parameters included).
A separate torch.profiler run of one native call reports the step kernel's mean time (step_kernel_us).  Prints one JSON line per
row with the card's name, power limit and SM clock.
"""
from __future__ import annotations

import argparse
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from long_seq_bench import emit  # noqa: E402

import cflearn_b200  # noqa: F401,E402
import ddim_oracle  # noqa: E402
import unet_oracle as uo  # noqa: E402
from cflearn_b200.ddpm import DDPMB200  # noqa: E402

DEV = torch.device("cuda", 0)
MIB = 1 << 20
SIDE, CONTEXT, SCALE = 64, 77, 7.5


def timed_s(fn) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3


def peak_mib(fn) -> float:
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    fn()
    torch.cuda.synchronize()
    return round(torch.cuda.max_memory_allocated(DEV) / MIB, 1)


def step_kernel_us(fn) -> float:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "ddim_step_kernel" in e.name]
    return round(sum(times) / max(len(times), 1), 2)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ddim_sample_bench needs a GPU")
    cfg = uo.unet_config("sd_v1_5")
    m = DDPMB200(SIDE, cfg["in_channels"], cfg["out_channels"], use_spatial_transformer=True, num_heads=cfg["num_heads"],
                 context_dim=cfg["context_dim"], start_channels=cfg["start_channels"], num_res_blocks=cfg["num_res_blocks"],
                 attention_downsample_rates=cfg["attention_downsample_rates"], channel_multipliers=cfg["channel_multipliers"],
                 condition_model="identity")
    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.unet.state_dict().items()], seed=0)
    m.unet.load_state_dict(sd, strict=True)
    m = m.to(DEV)
    params = {k: v.to(DEV) for k, v in sd.items()}
    g = torch.Generator().manual_seed(1)
    uncond = torch.randn(1, CONTEXT, cfg["context_dim"], generator=g).to(DEV)
    m.switch_sampler("ddim", dict(unconditional_cond=uncond, unconditional_guidance_scale=SCALE))

    def eager_denoise(image, ts, cond):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            return uo.forward(params, image, ts, cond, cfg)

    for B in args.batches:
        z = torch.randn(B, cfg["in_channels"], SIDE, SIDE, generator=g).to(DEV)
        cond = torch.randn(B, CONTEXT, cfg["context_dim"], generator=g).to(DEV)
        rows = {
            "native": lambda: m.decode(z, cond=cond, num_steps=args.steps),
            "eager": lambda: ddim_oracle.sample(eager_denoise, m.alphas_cumprod, z, cond=cond, unconditional_cond=uncond,
                                                num_steps=args.steps, unconditional_guidance_scale=SCALE),
        }
        peaks = {}
        for name, fn in rows.items():
            fn()  # warm-up (the native row captures its graph here)
            peaks[name] = peak_mib(fn)
        kernel_us = step_kernel_us(rows["native"])
        clocks_sampler = ClockSampler(DEV.index)
        clocks_sampler.start()
        times = {name: [] for name in rows}
        for _ in range(args.reps):
            for name, fn in rows.items():
                times[name].append(timed_s(fn))
        clocks = clocks_sampler.stop()
        for name in rows:
            s = statistics.median(times[name])
            rec = {"run": "ddim_sd_v1_5", "row": name, "B": B, "side": SIDE, "steps": args.steps, "guidance": SCALE,
                   "ms_per_step": round(1e3 * s / args.steps, 2), "s_per_batch": round(s, 3), "peak_mib": peaks[name]}
            if name == "native":
                rec["step_kernel_us"] = kernel_us
            emit(rec, clocks)
        m.sampler.release()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
