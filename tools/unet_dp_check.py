"""torchrun --nproc-per-node N tools/unet_dp_check.py [--grad-accumulate K]: data-parallel gradient parity of the SD-UNet's DDPM
step (DDPMB200) on real GPUs, the tools/dp_check.py pattern on the small UNet config.

Each rank trains its shard (rank r takes samples r, r + W, ...) with explicit noise and timesteps; the bucketed all-reduce(AVG)
of the gradient arena over the library's NCCL communicator must reproduce the gradient of the global-batch mean loss, which
rank 0 computes alone on the whole batch.  Three schedules: eager (bucket all-reduces on the forked communication stream), graphed
(the same in one CUDA graph) and flat (one all-reduce of the whole arena behind the graph).  The bound is dp_check's: relative
L2 below 5e-3, and the three schedules within 1e-6 of each other.
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import unet_oracle as uo  # noqa: E402

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import dp  # noqa: E402
from cflearn_b200.ddpm import DDPMB200  # noqa: E402
from cflearn_b200.optim import ArenaAdamW, GraphedTrainStep  # noqa: E402
from cflearn_b200.trainer import B200TrainStep  # noqa: E402

SMALL = dict(num_heads=2, context_dim=64, start_channels=64, num_res_blocks=1, attention_downsample_rates=(1, 2),
             channel_multipliers=(1, 2))


def build(sd, dev):
    m = DDPMB200(64, 4, 4, use_spatial_transformer=True, **SMALL)
    m.load_state_dict(sd, strict=True)
    return m.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grad-accumulate", type=int, default=1)
    K = ap.parse_args().grad_accumulate
    rank, world, local = dp.ddp_info()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    comm = dp.NativeComm(rank, world, dev)
    probe = DDPMB200(64, 4, 4, use_spatial_transformer=True, **SMALL)
    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in probe.state_dict().items()], seed=0)
    per_rank, side = 2, 16
    g = torch.Generator().manual_seed(3)
    batches = []
    for _ in range(K):  # (latent, context, noise, timesteps) of the global batch
        n = per_rank * world
        batches.append((torch.randn(n, 4, side, side, generator=g), torch.randn(n, 7, 64, generator=g),
                        torch.randn(n, 4, side, side, generator=g), torch.randint(0, 1000, (n,), generator=g)))
    idx = list(dp.shard_indices(per_rank * world, rank, world))
    shards = [tuple(t[idx].to(dev) for t in b) for b in batches]
    g_one = None
    if rank == 0:
        single = build(sd, dev)
        for b in batches:  # the first backward overwrites the arena, the others add to it
            single.train_step(*(t.to(dev) for t in b))
        torch.cuda.synchronize()
        g_one = single.arena.grad.clone()
        del single
    results = {}
    for mode in ("eager", "graphed", "flat"):
        m = build(sd, dev)
        dp.broadcast_parameters(m)
        gs = None
        if mode == "eager":
            seam = B200TrainStep(m, ArenaAdamW(m, lr=0.0), comm=comm, grad_accumulate=K)
            for s in shards:
                seam.step(*s)
        else:
            gs = GraphedTrainStep(m, ArenaAdamW(m, lr=0.0, capturable=True), per_rank, comm=comm, flat=(mode == "flat"),
                                  inputs=[torch.zeros_like(t) for t in shards[0]], grad_accumulate=K)
            for _ in range(2):  # replays are repeatable: same gradients
                for s in shards:
                    gs.step(*s)
        torch.cuda.synchronize()
        comm.check()
        g_dp = m.arena.grad.clone()
        ref = g_dp.clone()
        dist.broadcast(ref, src=0)
        assert torch.equal(ref, g_dp), f"{mode}: ranks disagree after the all-reduce"
        if rank == 0:
            results[mode] = ((g_dp - g_one).norm() / g_one.norm()).item()
        m.engine.reducer = None
        if gs is not None:
            gs.release()  # (ncclCommDestroy below waits for every graph that captured the communicator)
        del m
    if rank == 0:
        print(f"unet_dp_check: world {world}, grad_accumulate {K}, NCCL {comm.nccl_version}, "
              f"rel L2 (all-reduced vs single-process global batch): " + ", ".join(f"{k} {v:.3e}" for k, v in results.items()))
        assert all(v < 5e-3 for v in results.values()), results
        assert abs(results["graphed"] - results["eager"]) < 1e-6 and abs(results["flat"] - results["eager"]) < 1e-6, results
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
