"""torchrun --nproc-per-node N tools/unet_train_bench.py [--batch 8] [--reps 5] [--baseline N1.jsonl]: weak scaling of the
SD-v1.5 DDPM training step (BASELINE.json configs[4]) at 64 x 64 latents, a 77 x 768 context and --batch images per GPU.  Run it
once with N = 1 (saving its output) and once with every N the machine has, passing the N = 1 output as --baseline: each row then
reports its scaling efficiency, samples/s per GPU over the same row's samples/s at N = 1 (at N = 1 without a baseline: 1.0).

Rows, each the median of three rounds of ``--reps`` steps timed with CUDA events after warm-up:
  native_graphed   B200TrainStep(DDPMB200, ArenaAdamW, clip_norm=1, graph=True): draws, q-sample, forward, loss, backward,
                   the bucketed in-graph all-reduce, clipping and AdamW as one CUDA graph replay
  eager            eager bf16 autocast of oracle/unet_oracle.py::forward with torch's q-sample and mse_loss, wrapped for N > 1 in
                   torch.nn.parallel.DistributedDataParallel (default 25 MB buckets, all-reduced while backward runs), then
                   clip_grad_norm_ and torch.optim.AdamW(fused=True)
The two rows cannot be held in memory together, so they are not alternated: the three native rounds run first, then the eager
row after the native model is freed.  peak_mib is torch.cuda.max_memory_allocated over warm-up and the timed steps (the native row
includes the graph's pool and the warm-up snapshot of parameters and moments).  Rank 0 prints one JSON line per row with the card's
name, power limit and SM clock.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench import ClockSampler  # noqa: E402
from long_seq_bench import emit, time_ms  # noqa: E402

import cflearn_b200  # noqa: F401,E402
import unet_oracle as uo  # noqa: E402
from cflearn_b200 import dp  # noqa: E402
from cflearn_b200.ddpm import DDPMB200, noise_tables  # noqa: E402
from cflearn_b200.optim import ArenaAdamW  # noqa: E402
from cflearn_b200.trainer import B200TrainStep  # noqa: E402

MIB = 1 << 20
SIDE, CONTEXT = 64, 77


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--baseline", default=None, help="the JSON lines an N = 1 run of this tool printed")
    args = ap.parse_args()
    base = {}
    if args.baseline:
        for line in open(args.baseline):
            if line.startswith("{"):
                r = json.loads(line)
                if r.get("world") == 1:
                    base[r["row"]] = r["samples_per_s"]

    def report(row: str, t: list, peak: float, clocks: dict) -> None:
        ms = statistics.median(t)
        sps = B * world * 1000 / ms
        eff = sps / world / base[row] if row in base else (1.0 if world == 1 else None)
        emit({"run": "unet_sd_v1_5_ddpm_train", "row": row, "world": world, "B_per_gpu": B, "side": SIDE, "ms": round(ms, 2),
              "spread_ms": [round(v, 2) for v in t], "samples_per_s": round(sps, 2),
              "scaling_efficiency": None if eff is None else round(eff, 3), "peak_mib": peak}, clocks)

    if not torch.cuda.is_available():
        raise SystemExit("unet_train_bench needs a GPU")
    info = dp.ddp_info()
    rank, world, local = info if info is not None else (0, 1, 0)
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    cfg = uo.unet_config("sd_v1_5")
    B = args.batch
    m = DDPMB200(SIDE * 8, cfg["in_channels"], cfg["out_channels"], use_spatial_transformer=True, num_heads=cfg["num_heads"],
                 context_dim=cfg["context_dim"], start_channels=cfg["start_channels"], num_res_blocks=cfg["num_res_blocks"],
                 attention_downsample_rates=cfg["attention_downsample_rates"], channel_multipliers=cfg["channel_multipliers"])
    sd = uo.synthetic_state_dict([(k[len("unet."):], tuple(v.shape)) for k, v in m.state_dict().items()], seed=0)
    m.unet.load_state_dict(sd, strict=True)
    m = m.to(dev)
    g = torch.Generator().manual_seed(1 + rank)
    x = torch.randn(B, cfg["in_channels"], SIDE, SIDE, generator=g).to(dev)
    ctx = torch.randn(B, CONTEXT, cfg["context_dim"], generator=g).to(dev)
    comm = dp.NativeComm(rank, world, dev) if world > 1 else None
    if comm is not None:
        dp.broadcast_parameters(m)
    torch.cuda.reset_peak_memory_stats(dev)
    opt = ArenaAdamW(m, lr=1e-4, capturable=True)
    step = B200TrainStep(m, opt, clip_norm=1.0, comm=comm, graph=True, static_inputs=[torch.zeros_like(x), torch.zeros_like(ctx)])

    def native():
        step.step(x, ctx)

    sampler = ClockSampler(dev.index)
    sampler.start()
    t = [time_ms(native, args.reps, warmup=2) for _ in range(3)]
    clocks = sampler.stop()
    peak = round(torch.cuda.max_memory_allocated(dev) / MIB, 1)
    if rank == 0:
        report("native_graphed", t, peak, clocks)
    step.close()
    del step, opt
    if comm is not None:
        comm.close()
    m.grad_arena.close()
    del m
    torch.cuda.empty_cache()

    # eager bf16 autocast + torch DDP + fused AdamW
    eager_model = _EagerUNet(sd, cfg).to(dev)
    net = eager_model if world == 1 else torch.nn.parallel.DistributedDataParallel(eager_model, device_ids=[local])
    plist = list(eager_model.parameters())
    a, s = (v.to(dev) for v in noise_tables())
    topt = torch.optim.AdamW(plist, lr=1e-4, fused=True)
    torch.cuda.reset_peak_memory_stats(dev)

    def eager():
        ts = torch.randint(0, 1000, (B,), device=dev)
        noise = torch.randn_like(x)
        xt = a[ts].view(-1, 1, 1, 1) * x + s[ts].view(-1, 1, 1, 1) * noise
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = net(xt, ts, ctx)
            loss = F.mse_loss(out, noise, reduction="none").mean(dim=(1, 2, 3)).mean()
        loss.backward()  # (N > 1: DDP's bucketed all-reduce runs inside)
        torch.nn.utils.clip_grad_norm_(plist, 1.0)
        topt.step()
        topt.zero_grad(set_to_none=True)

    sampler = ClockSampler(dev.index)
    sampler.start()
    t = [time_ms(eager, args.reps, warmup=2) for _ in range(3)]
    clocks = sampler.stop()
    peak = round(torch.cuda.max_memory_allocated(dev) / MIB, 1)
    if rank == 0:
        report("eager", t, peak, clocks)
    if world > 1:
        dist.destroy_process_group()


class _EagerUNet(torch.nn.Module):
    """oracle/unet_oracle.py::forward over its own parameters, so that DistributedDataParallel can wrap it (the state dict's dotted
    keys are kept in a side list; the parameters live in a ParameterList)."""

    def __init__(self, sd: dict, cfg: dict) -> None:
        super().__init__()
        self.keys = list(sd)
        self.ps = torch.nn.ParameterList([torch.nn.Parameter(v.clone()) for v in sd.values()])
        self.cfg = cfg

    def forward(self, xt, ts, ctx):
        return uo.forward(dict(zip(self.keys, self.ps)), xt, ts, ctx, self.cfg)


if __name__ == "__main__":
    main()
