"""Decoding SD latents to pixels on one GPU: the KL-f8 autoencoder's decoder (AttentionAutoEncoderKLB200.decode) against eager bf16
autocast of oracle/ae_oracle.py::decode (channels-last, cudnn.benchmark on).  Synthetic weights, 64 x 64 latents (512 px).

    python tools/ae_decode_bench.py [--batches 1 4 8] [--reps 3]

Rows per batch, each the median of --reps decodes timed with CUDA events after one warm-up decode, the rows alternating:
  native      AttentionAutoEncoderKLB200.decode
  eager       the oracle on eager autocast
Each row reports ms, peak_mib (torch.cuda.max_memory_allocated over one decode, parameters included) and tflops: the decoder's
multiply-adds computed from its shapes (convolutions, 1x1 projections, Q K^T and P V; 2 FLOP each) over the time.  A separate
run of one native decode, with CUDA events around every ``spatial_attention`` call and around the decode, reports attn_ms (the
mid block's attention), attn_share (attn_ms over that decode's time) and attn_floor_ms, the least time the data sheet's H100
could take for the attention (its FLOPs at the dense BF16 peak, or the bytes of S and P at the HBM peak, whichever is larger);
a measured time under that floor stops the run.  Prints one JSON line per row with the card's name, power limit and SM clock.
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
from torch import nn  # noqa: E402

from bench import ClockSampler  # noqa: E402
from long_seq_bench import emit  # noqa: E402

import ae_oracle as ao  # noqa: E402
import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import autoencoder  # noqa: E402
from cflearn_b200.autoencoder import AttentionAutoEncoderKLB200  # noqa: E402

DEV = torch.device("cuda", 0)
MIB = 1 << 20
SIDE = 64


def timed_ms(fn) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def peak_mib(fn) -> float:
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    fn()
    torch.cuda.synchronize()
    return round(torch.cuda.max_memory_allocated(DEV) / MIB, 1)


def decode_flops(m: AttentionAutoEncoderKLB200, B: int, h: int, w: int) -> tuple:
    """(all, attention) FLOPs of one decode of B latents h x w, from the shapes: 2 per multiply-add."""
    total = 2 * B * h * w * m.from_embedding.weight.numel()
    attn = 0
    for block in m.generator.decoder.decoder:
        hw = h * w
        if isinstance(block, autoencoder._SpatialAttention):
            C = block.to_q.weight.shape[0]
            a = 2 * B * hw * 4 * C * C + 2 * 2 * B * hw * hw * C  # four 1x1 projections, Q K^T and P V
            attn += a
            total += a
            continue
        if isinstance(block, autoencoder._Resample):
            h, w = 2 * h, 2 * w
        for mod in block.modules():
            if isinstance(mod, nn.Conv2d):
                total += 2 * B * h * w * mod.weight.numel()
    total += 2 * B * h * w * m.generator.decoder.head[2].weight.numel()
    return total, attn


PEAK_BF16_FLOPS = 989e12  # H100 SXM data sheet, dense BF16
PEAK_HBM_BYTES = 3.35e12  # H100 SXM data sheet, HBM3


def attention_time(m: AttentionAutoEncoderKLB200, z: torch.Tensor) -> tuple:
    """(ms inside ``spatial_attention``, ms of the whole decode) of one native decode, both from CUDA events on the decode's
    stream: events around every ``spatial_attention`` call and around the decode, in a run of its own."""
    inner = autoencoder.spatial_attention
    spans = []

    def timed(*args, **kwargs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = inner(*args, **kwargs)
        e1.record()
        spans.append((e0, e1))
        return out

    autoencoder.spatial_attention = timed
    try:
        total = timed_ms(lambda: m.decode(z))
    finally:
        autoencoder.spatial_attention = inner
    return sum(e0.elapsed_time(e1) for e0, e1 in spans), total


def attention_floor_ms(B: int, T: int, attn_flops: float) -> float:
    """The least time the attention could take on the data sheet's H100: the larger of its FLOPs at the dense BF16 peak and the
    bytes its S and P must move at the HBM peak (per image, fp32 S [T, T] written and read, bf16 P written and read)."""
    return 1e3 * max(attn_flops / PEAK_BF16_FLOPS, B * 12 * T * T / PEAK_HBM_BYTES)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ae_decode_bench needs a GPU")
    torch.backends.cudnn.benchmark = True
    cfg = ao.ae_config("kl_f8")
    m = AttentionAutoEncoderKLB200(cfg.pop("img_size"), cfg.pop("in_channels"), cfg.pop("out_channels"), cfg.pop("inner_channels"),
                                   cfg.pop("latent_channels"), cfg.pop("channel_multipliers"), **cfg)
    sd = ao.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=0)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV)
    params = {k: v.to(DEV) for k, v in sd.items()}
    g = torch.Generator().manual_seed(1)

    def eager(z):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            return ao.decode(params, z.contiguous(memory_format=torch.channels_last))

    for B in args.batches:
        z = torch.randn(B, m.embedding_channels, SIDE, SIDE, generator=g).to(DEV)
        rows = {"native": lambda: m.decode(z), "eager": lambda: eager(z)}
        peaks = {}
        for name, fn in rows.items():
            fn()  # warm-up (module loads, cudnn's algorithm search)
            peaks[name] = peak_mib(fn)
        flops, attn_flops = decode_flops(m, B, SIDE, SIDE)
        attn_ms, attn_total_ms = attention_time(m, z)
        floor_ms = attention_floor_ms(B, SIDE * SIDE, attn_flops)
        if attn_ms < floor_ms:
            raise SystemExit(f"attention measured at {attn_ms:.3f} ms, under the hardware's floor of {floor_ms:.3f} ms: mis-timed")
        clocks_sampler = ClockSampler(DEV.index)
        clocks_sampler.start()
        times = {name: [] for name in rows}
        for _ in range(args.reps):
            for name, fn in rows.items():
                times[name].append(timed_ms(fn))
        clocks = clocks_sampler.stop()
        for name in rows:
            ms = statistics.median(times[name])
            rec = {"run": "ae_kl_f8_decode", "row": name, "B": B, "px": 8 * SIDE, "ms": round(ms, 2), "peak_mib": peaks[name],
                   "gflop": round(flops / 1e9, 1), "attn_gflop": round(attn_flops / 1e9, 1), "tflops": round(flops / ms / 1e9, 1)}
            if name == "native":
                rec.update(attn_ms=round(attn_ms, 3), attn_floor_ms=round(floor_ms, 3), attn_share=round(attn_ms / attn_total_ms, 4))
            emit(rec, clocks)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
