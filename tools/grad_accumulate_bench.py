"""Gradient accumulation on the graphed trainer seam: ViT-B/16 224 px, micro-batch 256, ``B200TrainStep(graph=True,
grad_accumulate=K)`` for K in {1, 2, 4} on one GPU.

    python tools/grad_accumulate_bench.py [--batch 256] [--windows 8] [--rounds 3] [--ks 1 2 4]

Per K, one JSON line with:
  - micro_ms: one micro-step (forward, loss, backward adding to the gradient arena; no exchange, no Adam), CUDA events
    around each replay, median over the timed windows (null for K = 1, where every step closes a window);
  - closing_ms: the window's closing step (the same plus clipping and Adam), likewise;
  - samples_per_s: K * batch over the time of whole windows (events around each window, including the zeroing of the arena
    before its first micro-step and the copies of the batch into the static inputs), the median of ``--rounds`` rounds of
    ``--windows`` windows;
  - peak_mib: torch.cuda.max_memory_allocated over building the seam (warm-up, capture) and the timed windows, less what
    the model and the data held before;
and the card's name, power limit and median SM clock, read in the same run.  The K values run one after another (each
holds its own graphs), so their rounds cannot alternate.
"""
from __future__ import annotations

import argparse
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from long_seq_bench import emit  # noqa: E402

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import registry  # noqa: E402
from cflearn_b200.optim import ArenaAdam  # noqa: E402
from cflearn_b200.trainer import B200TrainStep  # noqa: E402

DEV = torch.device("cuda", 0)
MIB = 1 << 20


def vit_b16() -> torch.nn.Module:
    return registry.build_module("cv_clf", config=dict(in_channels=3, num_classes=1000, img_size=224, latent_dim=768, encoder="vit",
                                                       encoder_config=dict(patch_size=16, num_layers=12))).to(DEV)


def measure(K: int, batch: int, windows: int, rounds: int) -> dict:
    torch.manual_seed(0)
    model = vit_b16()
    opt = ArenaAdam(model, lr=1e-4, capturable=True)
    x = torch.randn(batch, 3, 224, 224, device=DEV)
    y = torch.randint(0, 1000, (batch, 1), device=DEV)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    seam = B200TrainStep(model, opt, clip_norm=1.0, graph=True, batch=batch, grad_accumulate=K)
    for _ in range(K):  # one untimed window after the capture
        seam.step(x, y)
    micro, closing, per_s = [], [], []
    for _ in range(rounds):
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(K + 1)] for _ in range(windows)]
        for w in range(windows):
            ev[w][0].record()
            for k in range(K):
                seam.step(x, y)
                ev[w][k + 1].record()
        torch.cuda.synchronize()
        for w in range(windows):
            steps = [ev[w][k].elapsed_time(ev[w][k + 1]) for k in range(K)]
            micro += steps[:-1]
            closing.append(steps[-1])
        per_s.append(windows * K * batch / (sum(ev[w][0].elapsed_time(ev[w][K]) for w in range(windows)) / 1e3))
    assert seam.updated
    peak = torch.cuda.max_memory_allocated(DEV) - base
    loss = float(seam.step(x, y).item())
    seam.close()
    return {"micro_ms": round(statistics.median(micro), 3) if micro else None, "closing_ms": round(statistics.median(closing), 3),
            "samples_per_s": round(statistics.median(per_s), 1), "samples_per_s_range": [round(min(per_s), 1), round(max(per_s), 1)],
            "peak_mib": round(peak / MIB, 1), "loss": round(loss, 4)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--windows", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 2, 4])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("grad_accumulate_bench needs a GPU")
    for K in args.ks:
        sampler = ClockSampler(DEV.index)
        sampler.start()
        res = measure(K, args.batch, args.windows, args.rounds)
        clocks = sampler.stop()
        record = {"run": "grad_accumulate", "model": "vit_b16", "batch": args.batch, "K": K, **res,
                  "note": "ms per replay (CUDA events); samples/s over whole windows; peak_mib max_memory_allocated over build + timed windows"}
        emit(record, clocks)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
