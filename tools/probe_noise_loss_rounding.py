"""Which fp32 operations eager PyTorch performs on CUDA for the gradient of the DDPM noise-prediction loss under bf16 autocast,
``F.mse_loss(pred, noise, reduction="none").mean(dim=(1, 2, 3)).mean()`` with bf16 ``pred``.

Candidates for d loss / d pred, before the bf16 cast of autocast's backward (g0: the loss's upstream gradient, N = C H W):
  reciprocal:  fl(fl(2 fl(pred - noise)) fl(fl(g0 fl(1/B)) fl(1/N)))   (the means' backward multiply by the reciprocal)
  division:    fl(fl(2 fl(pred - noise)) fl(fl(g0 / B) / N))
Where N is a power of two the two scales agree; the probe also runs shapes where they differ, with values planted where the
two scales round to different bf16 gradients, so that eager's order is established, not merely consistent.  Prints how many
elements each candidate gets wrong, and the native kernel's count.  Needs a GPU."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cflearn_b200.unet import noise_prediction_loss  # noqa: E402


def scales(B: int, N: int, g0: float) -> tuple:
    """The two candidate scales as fp32 tensors, from IEEE fp32 arithmetic on the host (numpy: a true division is a division)."""
    f = np.float32
    rec, div = f(f(g0) * (f(1) / f(B))) * (f(1) / f(N)), f(f(g0) / f(B)) / f(N)
    return torch.tensor(float(rec), dtype=torch.float32), torch.tensor(float(div), dtype=torch.float32)


def split_values(B: int, N: int, g0: float, count: int = 32) -> torch.Tensor:
    """Values of pred - noise whose bf16 gradients differ between the two candidates (empty where their scales agree)."""
    g_rec, g_div = scales(B, N, g0)
    d = torch.rand(1 << 22, generator=torch.Generator().manual_seed(B * N)) * 3.5 + 0.5
    rec, div = ((2 * d) * g_rec).to(torch.bfloat16), ((2 * d) * g_div).to(torch.bfloat16)
    return d[torch.nonzero(rec.view(torch.int16) != div.view(torch.int16))[:count, 0]]


def main() -> int:
    dev = torch.device("cuda")
    worst, separated = 0, 0
    # the last three shapes (N = 4 H W not a power of two) give the candidates different scales; values that the two scales
    # round to different bf16 gradients are planted in the batch (pred 0, noise -d), so there the candidates disagree
    for B, H, W, g0 in ((1, 8, 8, 1.0), (3, 64, 64, 1.0), (8, 64, 64, 1.0), (6, 64, 64, 3.0), (3, 24, 40, 1.0), (2, 24, 40, 0.37),
                        (1, 48, 64, 1.3)):
        N = 4 * H * W
        g = torch.Generator().manual_seed(B * H)
        pred = torch.randn(B * N, generator=g).to(torch.bfloat16)
        noise = torch.randn(B * N, generator=g)
        d = split_values(B, N, g0)
        if d.numel():
            pos = torch.arange(d.numel()) * (B * N // d.numel())
            pred[pos], noise[pos] = 0, -d
        pred = pred.view(B, 4, H, W).to(dev).contiguous(memory_format=torch.channels_last)
        noise = noise.view(B, 4, H, W).to(dev).contiguous(memory_format=torch.channels_last)
        p = pred.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.mse_loss(p, noise, reduction="none").mean(dim=(1, 2, 3)).mean()
        (loss * g0).backward()
        eager = p.grad
        d2 = 2 * (pred.float() - noise)
        g_rec, g_div = (s.to(dev) for s in scales(B, N, g0))
        ours = pred.clone().requires_grad_(True)
        (noise_prediction_loss(ours, noise) * g0).backward()
        counts = {name: int(((d2 * s).to(torch.bfloat16).view(torch.int16) != eager.view(torch.int16)).sum())
                  for name, s in (("reciprocal", g_rec), ("division", g_div))}
        counts["native kernel"] = int((ours.grad.view(torch.int16) != eager.view(torch.int16)).sum())
        worst = max(worst, counts["native kernel"], counts["reciprocal"])
        separated += counts["division"] > 0
        print(f"B {B} {H}x{W} g0 {g0}, {d.numel()} planted values: elements differing from eager: "
              + ", ".join(f"{k} {v}" for k, v in counts.items()))
    print(f"the true-division order is ruled out on {separated} shapes; the reciprocal order and the kernel match eager everywhere"
          if worst == 0 else "MISMATCH")
    return 1 if worst or not separated else 0


if __name__ == "__main__":
    sys.exit(main())
