"""torchrun --nproc-per-node N tools/dp_check.py : data-parallel gradient parity on real GPUs (N = 2 .. 8).

Each rank runs the native training step on its shard (DistributedSampler rule: rank r takes samples r, r+W, ...); the
bucketed all-reduce(AVG) over the library's own NCCL communicator must reproduce the gradients of the global-batch mean
loss, which rank 0 also computes alone on the concatenated batch (SURVEY.md section 8e / finding 3: the reference defines
DP parity mathematically).  Three schedules are checked, all against the same single-process answer:
  eager    kernels launched from Python, bucket all-reduces on the forked communication stream (dp.NativeBucketReducer)
  graphed  the same, captured in ONE CUDA graph (optim.GraphedTrainStep) -- the schedule bench.py times
  flat     graph up to backward, one all-reduce of the whole arena behind it (round 1's schedule, kept as an A/B switch)

``--grad-accumulate K``: each schedule runs one window of K micro-batches through the trainer seam (eager:
``B200TrainStep``), exchanging once, on the summed gradients; the single process accumulates the same K global batches.
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import vit_oracle as vo  # noqa: E402

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import dp, registry  # noqa: E402
from cflearn_b200.optim import ArenaAdam, GraphedTrainStep  # noqa: E402
from cflearn_b200.trainer import B200TrainStep  # noqa: E402


def build(cfg, sd, dev):
    m = registry.build_module("cv_clf", config=dict(in_channels=3, num_classes=cfg["num_classes"], img_size=cfg["img_size"],
                                                    latent_dim=cfg["latent_dim"], encoder="vit",
                                                    encoder_config=dict(patch_size=cfg["patch_size"], num_layers=cfg["num_layers"])))
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
    cfg = vo.vit_config("vit_small")
    sd = vo.init_state_dict(cfg, seed=0)
    per_rank = 8
    batches = [vo.synthetic_batch(cfg, per_rank * world, seed=3 + k) for k in range(K)]
    idx = list(dp.shard_indices(per_rank * world, rank, world))
    shards = [(x[idx].to(dev), y[idx].to(dev)) for x, y in batches]
    xs, ys = shards[0]
    g_one = None
    if rank == 0:
        single = build(cfg, sd, dev)
        for x, y in batches:  # the first backward overwrites the arena, the others add to it
            single.train_step(x.to(dev), y.to(dev))
        torch.cuda.synchronize()
        g_one = single.arena.grad.clone()
        del single
    results = {}
    for mode in ("eager", "graphed", "flat"):
        m = build(cfg, sd, dev)
        dp.broadcast_parameters(m)
        if mode == "eager" and K == 1:
            dp.attach_native_reducer(m, comm)
            m.train_step(xs, ys)
        elif mode == "eager":
            seam = B200TrainStep(m, ArenaAdam(m, lr=0.0), comm=comm, grad_accumulate=K)
            for xk, yk in shards:
                seam.step(xk, yk)
        else:
            gs = GraphedTrainStep(m, ArenaAdam(m, lr=0.0, capturable=True), per_rank, comm=comm, flat=(mode == "flat"),
                                  grad_accumulate=K)
            for _ in range(2):  # replays are repeatable: same gradients
                for xk, yk in shards:
                    gs.step(xk, yk)
        torch.cuda.synchronize()
        comm.check()
        g_dp = m.arena.grad.clone()
        ref = g_dp.clone()
        dist.broadcast(ref, src=0)
        assert torch.equal(ref, g_dp), f"{mode}: ranks disagree after the all-reduce"
        if rank == 0:
            results[mode] = ((g_dp - g_one).norm() / g_one.norm()).item()
        m.engine.reducer = None
        if mode != "eager":
            gs.release()  # (ncclCommDestroy below waits for every graph that captured the communicator)
        del m
    if rank == 0:
        # same bf16 noise-floor argument as tests/test_model_gpu.py: shard-wise bf16 rounding of the weight grads
        print(f"dp_check: world {world}, grad_accumulate {K}, NCCL {comm.nccl_version}, "
              f"rel L2 (all-reduced vs single-process global batch): "
              + ", ".join(f"{k} {v:.3e}" for k, v in results.items()))
        assert all(v < 5e-3 for v in results.values()), results
        assert abs(results["graphed"] - results["eager"]) < 1e-6 and abs(results["flat"] - results["eager"]) < 1e-6, results
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
