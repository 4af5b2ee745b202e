"""use_checkpoint in the SD-v1.5 UNet's blocks on one GPU: memory and time of forward + backward with the activations stored and
with them recomputed in backward, for ResidualBlockWithTimeEmbeddingB200 and SpatialTransformerB200 (one block) at the shapes of
tools/res_block_bench.py and tools/spatial_transformer_bench.py (512 px, batch 8, time width 1280, 77 x 768 context).

    python tools/checkpoint_bench.py [--reps 20] [--batch 8] [--depth 4]

Per shape and mode:
  - held_mib: memory still allocated after one forward, less what was allocated before it (the output and what autograd keeps);
  - peak_mib / peak_depth_mib: torch.cuda.max_memory_allocated after reset_peak_memory_stats, over one forward + backward, and
    over ``--depth`` forwards of the block held together before one backward (a UNet holds every block's activations until its
    backward; one isolated call cannot show a saving, as the recompute rebuilds what the stored path kept); base_mib: what was
    allocated when the peak was reset (parameters, inputs, workspaces);
  - ms: one forward + backward, CUDA events over ``--reps`` calls after warm-up, the median of three rounds alternating the modes.
Prints one JSON line per shape with the card's name, power limit and median SM clock.
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
from long_seq_bench import emit, time_ms  # noqa: E402
from res_block_bench import SHAPES as RES_SHAPES, TDIM  # noqa: E402
from spatial_transformer_bench import CONTEXT, CONTEXT_DIM, HEADS, SHAPES as ST_SHAPES  # noqa: E402

import cflearn_b200  # noqa: F401,E402
import unet_oracle as uo  # noqa: E402
from cflearn_b200.spatial_transformer import SpatialTransformerB200  # noqa: E402
from cflearn_b200.unet_blocks import ResidualBlockWithTimeEmbeddingB200  # noqa: E402

DEV = torch.device("cuda", 0)
CL = torch.channels_last
MIB = 1 << 20
MODES = ("stored", "checkpoint")


def set_checkpoint(m: torch.nn.Module, flag: bool) -> None:
    for mod in m.modules():
        if hasattr(mod, "use_checkpoint"):
            mod.use_checkpoint = flag


def measure(m: torch.nn.Module, inputs: list, up: torch.Tensor, reps: int, depth: int) -> dict:
    leaves = [x.clone().requires_grad_(True) for x in inputs]

    def step():
        m(*leaves).backward(up)

    def stack():
        torch.autograd.backward([m(*leaves) for _ in range(depth)], [up] * depth)

    out = {}
    for mode in MODES:
        set_checkpoint(m, mode == "checkpoint")
        step()  # warm-up: workspaces reach their size
        torch.cuda.synchronize()
        m0 = torch.cuda.memory_allocated(DEV)
        y = m(*leaves)
        torch.cuda.synchronize()
        held = torch.cuda.memory_allocated(DEV) - m0
        del y
        res = {"held_mib": round(held / MIB, 1)}
        for key, fn in (("peak_mib", step), ("peak_depth_mib", stack)):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(DEV)
            base = torch.cuda.memory_allocated(DEV)
            fn()
            torch.cuda.synchronize()
            res[key] = round(torch.cuda.max_memory_allocated(DEV) / MIB, 1)
            res.setdefault("base_mib", round(base / MIB, 1))
        out[mode] = res
    times = {mode: [] for mode in MODES}
    for _ in range(3):
        for mode in MODES:
            set_checkpoint(m, mode == "checkpoint")
            times[mode].append(time_ms(step, reps))
    for mode in MODES:
        out[mode]["ms"] = round(statistics.median(times[mode]), 3)
    s, c = out["stored"], out["checkpoint"]
    out["time_overhead"] = round(c["ms"] / s["ms"] - 1.0, 3)
    out["peak_depth_saved_mib"] = round(s["peak_depth_mib"] - c["peak_depth_mib"], 1)
    return out


def res_block_case(B: int, Cin: int, Cout: int, side: int):
    m = ResidualBlockWithTimeEmbeddingB200(Cin, Cout, norm_eps=1e-5, time_embedding_channels=TDIM)
    m.load_state_dict(uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=Cin + Cout + side))
    g = torch.Generator().manual_seed(1)
    net = torch.randn(B, Cin, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=CL)
    tn = torch.randn(B, TDIM, generator=g).to(DEV).to(torch.bfloat16)
    up = torch.randn(B, Cout, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=CL)
    return m.to(DEV), [net, tn], up


def transformer_case(B: int, C: int, side: int):
    m = SpatialTransformerB200(C, HEADS, C // HEADS, context_dim=CONTEXT_DIM)
    m.load_state_dict(uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=C + side))
    g = torch.Generator().manual_seed(1)
    net = torch.randn(B, C, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=CL)
    ctx = torch.randn(B, CONTEXT, CONTEXT_DIM, generator=g).to(DEV)
    up = torch.randn(B, C, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=CL)
    return m.to(DEV), [net, ctx], up


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--depth", type=int, default=4, help="forward calls held together before one backward for peak_depth_mib")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("checkpoint_bench needs a GPU")
    cases = [({"run": "res_block", "Cin": Cin, "Cout": Cout, "side": side}, lambda a=(Cin, Cout, side): res_block_case(args.batch, *a))
             for Cin, Cout, side in RES_SHAPES]
    cases += [({"run": "spatial_transformer", "C": C, "side": side, "layers": 1}, lambda a=(C, side): transformer_case(args.batch, *a))
              for C, side in ST_SHAPES]
    for record, make in cases:
        m, inputs, up = make()
        sampler = ClockSampler(DEV.index)
        sampler.start()
        res = measure(m, inputs, up, args.reps, args.depth)
        clocks = sampler.stop()
        record.update(B=args.batch, depth=args.depth, **res)
        record["note"] = ("MiB; peak_mib one forward + backward, peak_depth_mib depth forwards then one backward; ms one forward + "
                          "backward, CUDA events")
        emit(record, clocks)
        del m, inputs, up
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
