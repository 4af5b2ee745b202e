"""Long-sequence attention on one GPU: the streamed kernels (T > 256) against torch's flash SDPA, the streamed against the resident
kernels at T = 197, and a graphed ViT-B/16 384 px training step against the eager oracle.

    python tools/long_seq_bench.py [--reps 30] [--steps 20] [--warmup 5] [--skip-step]

Prints one JSON line per measurement, each with the card's name, power limit and median SM clock read during that
measurement.  FLOP conventions are bench.py's: forward 4 B H T^2 64, backward 10 B H T^2 64, halved when causal.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from torch.nn.attention import SDPBackend, sdpa_kernel  # noqa: E402

from bench import ClockSampler  # noqa: E402

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import _cabi, ops, registry  # noqa: E402

DEV = torch.device("cuda", 0)
KERNEL_SHAPES = [(64, 577, 12, False), (16, 1025, 12, False), (4, 4096, 8, False), (4, 4096, 8, True)]


def card() -> dict:
    out = {"gpu": torch.cuda.get_device_name(DEV), "power_limit_w": None}
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(DEV.index)
        out["power_limit_w"] = round(pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0, 1)
    except Exception:  # pragma: no cover - pynvml missing
        pass
    return out


def emit(record: dict, clocks: dict) -> None:
    record.update(card())
    record["sm_mhz"] = clocks["sm_mhz"]
    record["clock_reasons"] = clocks["reasons"]
    print(json.dumps(record), flush=True)


def time_ms(fn, reps: int, warmup: int = 5) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def long_fwd(qkv, out, lse, B, T, H, causal):
    _cabi.call("b200_attention_long_fwd", qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, T, H, 64, 0.125, int(causal),
               torch.cuda.current_stream().cuda_stream)


def long_bwd(qkv, out, dout, lse, dqkv, ws, B, T, H, causal):
    _cabi.call("b200_attention_long_bwd", qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), B, T, H, 64,
               0.125, int(causal), None, ws.data_ptr(), torch.cuda.current_stream().cuda_stream)


def bench_kernels(reps: int) -> None:
    for B, T, H, causal in KERNEL_SHAPES:
        D = H * 64
        g = torch.Generator(device="cpu").manual_seed(T)
        qkv = torch.randn(B * T, 3 * D, generator=g).to(torch.bfloat16).to(DEV)
        dout = torch.randn(B * T, D, generator=g).to(torch.bfloat16).to(DEV)
        dqkv = torch.empty_like(qkv)
        sampler = ClockSampler(DEV.index)
        sampler.start()
        out, lse = ops.attention_fwd(qkv, B, T, H, causal=causal)
        f_ours = time_ms(lambda: ops.attention_fwd(qkv, B, T, H, causal=causal), reps)
        b_ours = time_ms(lambda: ops.attention_bwd(qkv, out, dout, lse, B, T, H, causal=causal, dqkv=dqkv), reps)
        # torch's flash kernel on contiguous [B, H, T, 64] operands (its preferred layout)
        q, k, v = (t.contiguous().requires_grad_(True) for t in qkv.view(B, T, 3, H, 64).permute(2, 0, 3, 1, 4))
        do = dout.view(B, T, H, 64).transpose(1, 2).contiguous()
        with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
            f_sdpa = time_ms(lambda: F.scaled_dot_product_attention(q, k, v, is_causal=causal), reps)
            o = F.scaled_dot_product_attention(q, k, v, is_causal=causal)
            b_sdpa = time_ms(lambda: torch.autograd.grad(o, (q, k, v), do, retain_graph=True), reps)
        clocks = sampler.stop()
        div = 2.0 if causal else 1.0
        ff, fb = 4.0 * B * H * T * T * 64 / div, 10.0 * B * H * T * T * 64 / div
        tf = lambda flop, ms: round(flop / (ms * 1e-3) / 1e12, 1)  # noqa: E731
        emit({"run": "attention_kernels", "B": B, "T": T, "H": H, "causal": causal,
              "fwd_ms": {"ours": round(f_ours, 4), "sdpa_flash": round(f_sdpa, 4)},
              "bwd_ms": {"ours": round(b_ours, 4), "sdpa_flash": round(b_sdpa, 4)},
              "fwd_tflops": {"ours": tf(ff, f_ours), "sdpa_flash": tf(ff, f_sdpa)},
              "bwd_tflops": {"ours": tf(fb, b_ours), "sdpa_flash": tf(fb, b_sdpa)},
              "note": "CUDA events over the launches; sdpa bwd is autograd.grad of its flash forward (includes the grad allocations)"},
             clocks)
        del qkv, dout, dqkv, out, lse, q, k, v, do, o


def bench_t197(reps: int) -> None:
    """The bench shape on both kernel pairs: which attention path is faster where both apply."""
    B, T, H = 256, 197, 12
    D = H * 64
    g = torch.Generator(device="cpu").manual_seed(197)
    qkv = torch.randn(B * T, 3 * D, generator=g).to(torch.bfloat16).to(DEV)
    dout = torch.randn(B * T, D, generator=g).to(torch.bfloat16).to(DEV)
    dqkv = torch.empty_like(qkv)
    out = torch.empty(B * T, D, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(B, H, T, dtype=torch.float32, device=DEV)
    ws = torch.empty(int(_cabi.lib().b200_attention_long_bwd_workspace_floats(B, T, H)), dtype=torch.float32, device=DEV)
    sampler = ClockSampler(DEV.index)
    sampler.start()
    r_out, r_lse = ops.attention_fwd(qkv, B, T, H)  # T <= 256: the resident kernels
    f_res = time_ms(lambda: ops.attention_fwd(qkv, B, T, H), reps)
    b_res = time_ms(lambda: ops.attention_bwd(qkv, r_out, dout, r_lse, B, T, H, dqkv=dqkv), reps)
    long_fwd(qkv, out, lse, B, T, H, False)
    f_long = time_ms(lambda: long_fwd(qkv, out, lse, B, T, H, False), reps)
    b_long = time_ms(lambda: long_bwd(qkv, out, dout, lse, dqkv, ws, B, T, H, False), reps)
    clocks = sampler.stop()
    emit({"run": "attention_T197", "B": B, "T": T, "H": H,
          "fwd_ms": {"resident": round(f_res, 4), "streamed": round(f_long, 4)},
          "bwd_ms": {"resident": round(b_res, 4), "streamed": round(b_long, 4)}}, clocks)


def bench_step(steps: int, warmup: int) -> None:
    """ViT-B/16 at 384 px (T = 577), batch 64: our graphed step vs the oracle under eager bf16 autocast + fused torch Adam."""
    from cflearn_b200.optim import ArenaAdam, GraphedTrainStep

    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import vit_oracle as vo

    B, img = 64, 384
    g = torch.Generator(device="cpu").manual_seed(1000)
    x = torch.randn(B, 3, img, img, generator=g).to(DEV)
    y = torch.randint(0, 1000, (B, 1), generator=g).to(DEV)
    model = registry.build_module("cv_clf", config=dict(in_channels=3, num_classes=1000, img_size=img, latent_dim=768, encoder="vit",
                                                        encoder_config=dict(patch_size=16, num_layers=12))).to(DEV)
    opt = ArenaAdam(model, lr=1e-3, capturable=True)
    gstep = GraphedTrainStep(model, opt, B)
    sampler = ClockSampler(DEV.index)
    sampler.start()
    ms = time_ms(lambda: gstep.step(x, y), steps, warmup)
    loss = gstep.loss.item()
    clocks = sampler.stop()
    ours = B / (ms * 1e-3)
    gstep.release()  # free the graph's private pool before the eager leg allocates its activations
    del gstep, opt, model
    torch.cuda.empty_cache()

    cfg = vo.vit_config("vit_b16")
    cfg["img_size"] = img
    sd = vo.init_state_dict(cfg, seed=0, perturb=False)
    keys = list(sd.keys())
    ps = [torch.nn.Parameter(sd[k].to(DEV)) for k in keys]
    eopt = torch.optim.Adam(ps, lr=1e-3, fused=True)

    def eager_step():
        eopt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            el = vo.cross_entropy(vo.classifier_forward(dict(zip(keys, ps)), x, cfg), y)
        el.backward()
        eopt.step()

    esampler = ClockSampler(DEV.index)
    esampler.start()
    ems = time_ms(eager_step, min(steps, 10), 3)
    eclocks = esampler.stop()
    eager = B / (ems * 1e-3)
    emit({"run": "vit_b16_384px_step", "batch": B, "T": 577, "samples_per_s": {"ours_graphed": round(ours, 1), "eager_oracle": round(eager, 1)},
          "ms_per_step": {"ours_graphed": round(ms, 3), "eager_oracle": round(ems, 3)}, "speedup": round(ours / eager, 3),
          "loss": loss, "eager_sm_mhz": eclocks["sm_mhz"],
          "eager": "oracle port, PyTorch eager, bf16 autocast, fused torch Adam"}, clocks)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=30, help="timed launches per kernel (>= 20)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--skip-step", action="store_true", help="kernels only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("long_seq_bench.py needs a CUDA device")
    bench_kernels(max(args.reps, 20))
    bench_t197(max(args.reps, 20))
    if not args.skip_step:
        bench_step(args.steps, args.warmup)


if __name__ == "__main__":
    main()
