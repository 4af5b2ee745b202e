"""Where eager bf16 autocast rounds in the SD-UNet's resampling layers (oracle/unet_oracle.py::_sequential, the ResDownsample and
ResUpsample branches), on CUDA:
  - the biased stride-2 convolution and the biased convolution of the upsampled image: ONE rounding bf16(acc + bias), or TWO, the
    convolution rounded to bf16 and the bias added by a second bf16 op;
  - nearest interpolation of bf16: an exact copy;
  - its backward: the four bf16 gradients of a 2x2 block summed in fp32 and rounded once.
Prints the fraction of elements bit-identical to each model, and how often ResDownsampleB200 / ResUpsampleB200 agree with eager.

    python tools/probe_resample_rounding.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import cflearn_b200  # noqa: F401,E402
import unet_oracle as uo  # noqa: E402
from cflearn_b200 import ops  # noqa: E402
from cflearn_b200.unet_blocks import ResDownsampleB200, ResUpsampleB200  # noqa: E402

dev = "cuda"
g = torch.Generator().manual_seed(0)
eq = lambda a, c: (a == c).float().mean().item()  # noqa: E731
for name, (B, C, S, up) in {"down 64x64 / 320": (2, 320, 64, False), "down 16x16 / 1280": (2, 1280, 16, False),
                            "up 8x8 / 1280": (2, 1280, 8, True), "up 32x32 / 640": (2, 640, 32, True)}.items():
    x = torch.randn(B, C, S, S, generator=g).to(dev).to(torch.bfloat16)
    w = (torch.randn(C, C, 3, 3, generator=g) * (9 * C) ** -0.5).to(dev)
    b = (0.5 * torch.randn(C, generator=g)).to(dev)
    stride = 1 if up else 2
    xin = F.interpolate(x, scale_factor=2, mode="nearest") if up else x
    with torch.autocast("cuda", dtype=torch.bfloat16):
        eager = uo._sequential({"0.conv.weight" if up else "0.net.weight": w, "0.conv.bias" if up else "0.net.bias": b}, "", x, None,
                               None, 1)
    acc = F.conv2d(xin.float(), w.to(torch.bfloat16).float(), None, stride=stride, padding=1)
    bb = b.to(torch.bfloat16).float().view(1, -1, 1, 1)
    two = (acc.to(torch.bfloat16).float() + bb).to(torch.bfloat16)
    one = (acc + bb).to(torch.bfloat16)
    m = (ResUpsampleB200 if up else ResDownsampleB200)(C, True).to(dev)
    with torch.no_grad():
        (m.conv if up else m.net).weight.copy_(w)
        (m.conv if up else m.net).bias.copy_(b)
        ours = m(x.contiguous(memory_format=torch.channels_last))
    print(f"{name}: eager == bf16(bf16(fp32 conv) + bias) {eq(eager, two):.6f} | eager == bf16(fp32 conv + bias) {eq(eager, one):.6f} | "
          f"ours == eager {eq(ours, eager):.6f}")
    if up:
        xg = x.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = F.interpolate(xg, scale_factor=2, mode="nearest")
        dy = torch.randn(y.shape, generator=g).to(dev).to(torch.bfloat16)
        y.backward(dy)
        f = dy.float()
        once = (f[:, :, 0::2, 0::2] + f[:, :, 0::2, 1::2] + f[:, :, 1::2, 0::2] + f[:, :, 1::2, 1::2]).to(torch.bfloat16)
        pairwise = dy[:, :, 0::2, 0::2] + dy[:, :, 0::2, 1::2] + dy[:, :, 1::2, 0::2] + dy[:, :, 1::2, 1::2]
        ours_bwd = ops.sum2x2(dy.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2)
        print(f"{name} interpolate: copy exact {torch.equal(y, x.repeat_interleave(2, 2).repeat_interleave(2, 3))} | backward == fp32 sum "
              f"rounded once {eq(xg.grad, once):.6f} | == bf16 adds {eq(xg.grad, pairwise):.6f} | ours == eager {eq(ours_bwd, xg.grad):.6f}")
