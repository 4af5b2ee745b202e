"""TEST INFRASTRUCTURE ONLY -- plain-PyTorch functional restatement of the reference's KL autoencoder decode
(``AttentionAutoEncoderKL.decode``, cflearn/modules/cv/ae/kl.py:76-79 -> ``AttentionDecoder``, cv/decoder/attn.py), the first
stage that turns SD latents into pixels (``LDM.decode``, multimodal/diffusion/ldm.py:192-202).  Never imported by the product
package.

The structure is read off the reference ``state_dict``: every child of ``generator.decoder.decoder`` is recognised by the
parameter names it owns (bare ``weight`` -> the input convolution, ``norm1`` -> ResBlock, ``group_norm`` -> SpatialAttention,
``conv`` -> Upsample), so a reference checkpoint drives the oracle directly.  Pinned bit for bit on CPU fp32 against the
reference's own module by ``oracle/make_golden_ae.py`` (tests/golden/ae_kl_tiny_reference.pt).
Paths below are relative to carefree-learn's cflearn/.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

StateDict = Dict[str, Tensor]
EPS = 1e-6  # every GroupNorm of the autoencoder


def ae_config(name: str = "kl_f8") -> Dict:
    table = {
        # zoo/configs/ae/kl/f4.json with f8.json's overrides: 3 -> 3 channels, 128 inner channels, multipliers (1, 2, 4, 4),
        # latent and embedding channels 4, 2 res blocks per level
        "kl_f8": dict(img_size=256, in_channels=3, out_channels=3, inner_channels=128, latent_channels=4, channel_multipliers=(1, 2, 4, 4),
                      embedding_channels=4, num_res_blocks=2),
        # the smallest config the native kernels take (64-channel multiples): inner 64, multipliers (1, 2), one res block
        "kl_tiny": dict(img_size=16, in_channels=3, out_channels=3, inner_channels=64, latent_channels=4, channel_multipliers=(1, 2),
                        embedding_channels=4, num_res_blocks=1),
    }
    return dict(table[name])


def synthetic_state_dict(shapes: List[Tuple[str, Tuple[int, ...]]], seed: int = 0) -> StateDict:
    """Random weights for every key (the reference zero-initialises every ResBlock's conv2, residual.py:196, which would hide
    most of the network from a parity check): GroupNorm scales 1 + 0.1 N(0, 1), biases 0.02 N(0, 1), the rest N(0, 1) scaled by
    0.7 / sqrt(fan_in)."""
    g = torch.Generator().manual_seed(seed)
    sd: StateDict = {}
    for key, shape in shapes:
        if key.endswith("weight") and len(shape) == 1:
            sd[key] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif key.endswith("bias"):
            sd[key] = 0.02 * torch.randn(shape, generator=g)
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            sd[key] = torch.randn(shape, generator=g) * (0.7 / math.sqrt(max(fan_in, 1)))
    return sd


def _gn(sd: StateDict, p: str, net: Tensor) -> Tensor:
    return F.group_norm(net, 32, sd[p + "weight"], sd[p + "bias"], EPS)


def res_block(sd: StateDict, p: str, net: Tensor) -> Tensor:
    """ResidualBlockWithTimeEmbedding._forward (core/convs/residual.py:216-251) with no time embedding: GroupNorm -> SiLU ->
    conv3x3, GroupNorm -> SiLU -> Dropout(0) -> conv3x3, + shortcut (1x1 conv when the width changes), clamped to the dtype's
    finite range (toolkit.py:1236-1255)."""
    inp = net
    net = F.conv2d(F.silu(_gn(sd, p + "norm1.", net)), sd[p + "conv1.weight"], sd[p + "conv1.bias"], padding=1)
    if p + "shortcut.weight" in sd:
        inp = F.conv2d(inp, sd[p + "shortcut.weight"], sd[p + "shortcut.bias"])
    net = F.conv2d(F.silu(_gn(sd, p + "norm2.", net)), sd[p + "conv2.weight"], sd[p + "conv2.bias"], padding=1)
    net = inp + net
    fi = torch.finfo(net.dtype)
    return net.clamp(fi.min, fi.max)


def spatial_attention(sd: StateDict, p: str, net: Tensor) -> Tensor:
    """SpatialAttention.forward (core/attentions.py:350-370): GroupNorm, 1x1 q / k / v, one head of width C over the H * W
    pixels through sdp_attn -> F.scaled_dot_product_attention (toolkit.py:952-963), 1x1 to_out, + input."""
    inp = net
    net = _gn(sd, p + "group_norm.", net)
    b, c, h, w = net.shape
    q, k, v = (F.conv2d(net, sd[p + n + ".weight"], sd[p + n + ".bias"]).view(b, c, h * w).transpose(1, 2).contiguous()
               for n in ("to_q", "to_k", "to_v"))
    net = F.scaled_dot_product_attention(q, k, v, None, 0.0)
    net = net.transpose(1, 2).contiguous().view(b, c, h, w)
    return inp + F.conv2d(net, sd[p + "to_out.weight"], sd[p + "to_out.bias"])


def decode(sd: StateDict, z: Tensor, *, no_head: bool = False) -> Tensor:
    """``AttentionAutoEncoderKL.decode(DecoderInputs(z=z, no_head=no_head))``: from_embedding, the decoder's blocks, the head."""
    net = F.conv2d(z, sd["from_embedding.weight"], sd["from_embedding.bias"])
    i = 0
    while True:
        p = f"generator.decoder.decoder.{i}."
        if p + "weight" in sd:  # the input convolution
            net = F.conv2d(net, sd[p + "weight"], sd[p + "bias"], padding=1)
        elif p + "norm1.weight" in sd:
            net = res_block(sd, p, net)
        elif p + "group_norm.weight" in sd:
            net = spatial_attention(sd, p, net)
        elif p + "conv.weight" in sd:  # Upsample (decoder/attn.py:18-31)
            net = F.conv2d(F.interpolate(net, scale_factor=2.0, mode="nearest"), sd[p + "conv.weight"], sd[p + "conv.bias"], padding=1)
        else:
            break
        i += 1
    if no_head:
        return net
    h = "generator.decoder.head."
    net = F.silu(F.group_norm(net, 32, sd[h + "0.weight"], sd[h + "0.bias"], EPS))
    return F.conv2d(net, sd[h + "2.weight"], sd[h + "2.bias"], padding=1)
