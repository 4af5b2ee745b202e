"""The SD-v1.5 UNet's training step on one GPU: UNetDiffuserB200 + noise_prediction_loss against eager bf16 autocast of
oracle/unet_oracle.py::forward in NCHW (the reference's layout) with torch's mse_loss.  64 x 64 latents (512 px), a 77 x 768
context, batch 8 (the eager rows fall back to the largest batch that fits, and say so).

    python tools/unet_bench.py [--batch 8] [--reps 5]

Rows, each the median of three rounds of ``--reps`` calls timed with CUDA events after warm-up, the rounds alternating the rows:
  forward             UNetDiffuserB200 forward (autograd recording, as in training)
  step_stored         forward + loss + backward
  step_checkpoint     the same with use_checkpoint=True
  step_graphed        the stored step as one CUDA-graph replay
  eager_step          eager bf16 autocast forward + F.mse_loss + backward
Each row also reports peak_mib: torch.cuda.max_memory_allocated over one call, the parameters included; for the graphed row, over
the capture and one replay, as the graph's private pool keeps every buffer its capture allocated (a replay allocates nothing).
The eager row runs after ours is freed, so it is not alternated with them.  The
skip concatenation's bytes (torch.cat of bf16 channels-last tensors: both halves read and the result written in forward; the
two gradients of each skip read and their sum written in backward) are computed from the shapes.  Prints one JSON line per row with the card's name, power limit and SM clock.
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
import torch.nn.functional as F  # noqa: E402

from bench import ClockSampler  # noqa: E402
from long_seq_bench import emit, time_ms  # noqa: E402

import cflearn_b200  # noqa: F401,E402
import unet_oracle as uo  # noqa: E402
from cflearn_b200.unet import UNetDiffuserB200, noise_prediction_loss  # noqa: E402
from cflearn_b200.unet_blocks import ResUpsampleB200  # noqa: E402

DEV = torch.device("cuda", 0)
MIB = 1 << 20
SIDE, CONTEXT = 64, 77


def build(cfg: dict) -> tuple:
    m = UNetDiffuserB200(cfg["in_channels"], cfg["out_channels"], use_spatial_transformer=True, num_heads=cfg["num_heads"],
                         context_dim=cfg["context_dim"], start_channels=cfg["start_channels"], num_res_blocks=cfg["num_res_blocks"],
                         attention_downsample_rates=cfg["attention_downsample_rates"], channel_multipliers=cfg["channel_multipliers"])
    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=0)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def batch(cfg: dict, B: int) -> list:
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, cfg["in_channels"], SIDE, SIDE, generator=g)
    ts = torch.randint(0, 1000, (B,), generator=g)
    ctx = torch.randn(B, CONTEXT, cfg["context_dim"], generator=g)
    noise = torch.randn(B, cfg["out_channels"], SIDE, SIDE, generator=g)
    return [t.to(DEV) for t in (x, ts, ctx, noise)]


def cat_bytes(m: UNetDiffuserB200, B: int) -> dict:
    """HBM bytes of the skip concatenations: forward reads both halves and writes the result; backward slices the gradient (views)
    and adds each skip's two bf16 gradients (the concatenation's and the next down-path block's): two reads and one write."""
    side, c, fwd, bwd = SIDE >> (m.levels - 1), m.residual[-1].out_channels, 0, 0
    for blocks in m.output_blocks:
        cin = blocks[0].in_channels
        fwd += 2 * 2 * B * cin * side * side
        bwd += 3 * 2 * B * (cin - c) * side * side
        c = blocks[0].out_channels
        if isinstance(blocks[-1], ResUpsampleB200):
            side *= 2
    return {"cat_fwd_mb": round(fwd / 1e6, 1), "cat_bwd_mb": round(bwd / 1e6, 1)}


def peak_mib(fn) -> float:
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    fn()
    torch.cuda.synchronize()
    return round(torch.cuda.max_memory_allocated(DEV) / MIB, 1)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unet_bench needs a GPU")
    cfg = uo.unet_config("sd_v1_5")
    B = args.batch
    m, sd = build(cfg)
    x, ts, ctx, noise = batch(cfg, B)

    def set_checkpoint(flag: bool) -> None:
        for mod in m.modules():
            if hasattr(mod, "use_checkpoint"):
                mod.use_checkpoint = flag

    def forward():
        m.zero_grad(set_to_none=True)  # as the steps do: no previous step's gradients held
        m(x, timesteps=ts, context=ctx)

    def step():
        m.zero_grad(set_to_none=True)
        noise_prediction_loss(m(x, timesteps=ts, context=ctx), noise).backward()

    def step_ckpt():
        set_checkpoint(True)
        step()
        set_checkpoint(False)

    rows = {"forward": forward, "step_stored": step, "step_checkpoint": step_ckpt}
    step()  # warm-up: workspaces reach their size
    peaks = {name: peak_mib(fn) for name, fn in rows.items()}
    # one CUDA graph of the stored step: warm-up on a side stream, then capture with the gradients allocated in the graph's pool
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    m.zero_grad(set_to_none=True)
    # the graph keeps every buffer its capture allocated (its private pool) for as long as it lives: the peak across the capture,
    # from the parameters alone, is the graphed step's footprint (a replay allocates nothing)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        noise_prediction_loss(m(x, timesteps=ts, context=ctx), noise).backward()
    graph.replay()
    torch.cuda.synchronize()
    peaks["step_graphed"] = round(torch.cuda.max_memory_allocated(DEV) / MIB, 1)
    rows["step_graphed"] = graph.replay
    sampler = ClockSampler(DEV.index)
    sampler.start()
    times = {name: [] for name in rows}
    for _ in range(3):
        for name, fn in rows.items():
            times[name].append(time_ms(fn, args.reps, warmup=2))
    clocks = sampler.stop()
    extra = cat_bytes(m, B)
    for name in rows:
        emit({"run": "unet_sd_v1_5", "row": name, "B": B, "side": SIDE, "ms": round(statistics.median(times[name]), 2),
              "peak_mib": peaks[name], **extra}, clocks)
    del graph, rows
    m.zero_grad(set_to_none=True)
    del m
    torch.cuda.empty_cache()

    # eager bf16 autocast of the oracle in NCHW, the largest batch up to --batch that fits
    params = {k: v.to(DEV).requires_grad_(True) for k, v in sd.items()}
    eb = B
    while eb >= 1:
        xe, tse, ctxe, noisee = batch(cfg, eb)

        def eager_step():
            for p in params.values():
                p.grad = None
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = uo.forward(params, xe, tse, ctxe, cfg)
                loss = F.mse_loss(out, noisee, reduction="none").mean(dim=(1, 2, 3)).mean()
            loss.backward()

        try:
            peak = peak_mib(eager_step)
            break
        except torch.cuda.OutOfMemoryError:
            for p in params.values():
                p.grad = None
            torch.cuda.empty_cache()
            eb //= 2
    sampler = ClockSampler(DEV.index)
    sampler.start()
    t = [time_ms(eager_step, args.reps, warmup=2) for _ in range(3)]
    clocks = sampler.stop()
    emit({"run": "unet_sd_v1_5", "row": "eager_step", "B": eb, "side": SIDE, "ms": round(statistics.median(t), 2), "peak_mib": peak,
          "note": "" if eb == B else f"batch {B} does not fit eagerly; largest that fits"}, clocks)


if __name__ == "__main__":
    main()
