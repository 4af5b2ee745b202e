"""TEST INFRASTRUCTURE ONLY -- plain-PyTorch functional restatement of the reference's ``UNetDiffuser`` forward
(BASELINE.json configs[4], SURVEY.md 8f row N3: the SD-v1.5 UNet of cflearn/modules/multimodal/diffusion/unet.py:97-322).
Prepared ahead of the kernels: nothing in the product uses it yet.  Never imported by the product package.

The structure is read off the reference ``state_dict`` itself: every ``TimestepAttnSequential`` child is recognised by the
parameter names it owns (``norm1`` -> ResBlock, ``to_latent`` -> SpatialTransformer, ``net`` -> ResDownsample, ``conv`` ->
ResUpsample, bare ``weight`` -> the stem convolution), so a reference checkpoint drives the oracle directly.
Pinned bit-for-bit (fp32 and bf16 autocast; output and every gradient for a seeded upstream gradient) against the
reference's own module by ``oracle/make_golden_unet.py`` (tiny config stored in tests/golden/unet_tiny_reference.pt; the real
SD-v1.5 channel layout is pinned once at reduced resolution when the script runs).
Paths below are relative to carefree-learn's cflearn/.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

StateDict = Dict[str, Tensor]


def unet_config(name: str = "sd_v1_5") -> Dict:
    table = {
        # zoo/configs/diffusion/ldm/sd.json (SURVEY.md 8d config 5): 4 -> 4 channels, 320 start channels, multipliers (1,2,4,4),
        # 2 res blocks per level, spatial transformers at downsample rates 1/2/4 with 8 heads, context width 768
        "sd_v1_5": dict(in_channels=4, out_channels=4, num_heads=8, context_dim=768, start_channels=320, num_res_blocks=2,
                        attention_downsample_rates=(1, 2, 4), channel_multipliers=(1, 2, 4, 4)),
        "unet_tiny": dict(in_channels=4, out_channels=4, num_heads=2, context_dim=32, start_channels=32, num_res_blocks=1,
                          attention_downsample_rates=(1, 2), channel_multipliers=(1, 2)),
    }
    return dict(table[name])


def timestep_embedding(timesteps: Tensor, output_dim: int, dtype: torch.dtype, max_period: int = 10000) -> Tensor:
    """multimodal/diffusion/unet.py:53-77 (sinusoidal; cos first, then sin)."""
    half = output_dim // 2
    frequency = torch.exp(-math.log(max_period) * torch.arange(start=0, end=half, dtype=torch.float32) / half).to(timesteps.device)
    args = timesteps[:, None].float() * frequency[None]
    embedding = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if output_dim % 2:
        embedding = torch.cat([embedding, torch.zeros_like(embedding[:, :1])], dim=-1)
    return embedding.to(dtype)


def _gn(sd: StateDict, p: str, net: Tensor, eps: float) -> Tensor:
    return F.group_norm(net, 32, sd[p + "weight"], sd[p + "bias"], eps)


def res_block(sd: StateDict, p: str, net: Tensor, time_net: Tensor) -> Tensor:
    """ResidualBlockWithTimeEmbedding._forward (core/convs/residual.py:216-251) as the UNet builds it (unet.py:151-161):
    GroupNorm(32, eps 1e-5) -> SiLU -> conv3x3, + Linear(SiLU(time)), GroupNorm -> SiLU -> Dropout(0) -> conv3x3, + shortcut
    (1x1 conv when the width changes), then clamp to the dtype's finite range (toolkit.py:1236-1255)."""
    inp = net
    net = F.conv2d(F.silu(_gn(sd, p + "norm1.", net, 1e-5)), sd[p + "conv1.weight"], sd[p + "conv1.bias"], padding=1)
    if p + "shortcut.weight" in sd:
        inp = F.conv2d(inp, sd[p + "shortcut.weight"], sd[p + "shortcut.bias"])
    t = F.linear(F.silu(time_net), sd[p + "time_embedding.weight"], sd[p + "time_embedding.bias"])
    net = net + t[..., None, None]
    net = F.conv2d(F.silu(_gn(sd, p + "norm2.", net, 1e-5)), sd[p + "conv2.weight"], sd[p + "conv2.bias"], padding=1)
    net = inp + net
    fi = torch.finfo(net.dtype)
    return net.clamp(fi.min, fi.max)


def cross_attention(sd: StateDict, p: str, net: Tensor, context: Optional[Tensor], heads: int) -> Tensor:
    """CrossAttention.forward (core/attentions.py:535-569): bias-free q/k/v projections, heads folded into the batch,
    sdp_attn -> F.scaled_dot_product_attention (toolkit.py:959-963), out_linear with bias."""
    b, tq, dq = net.shape
    ctx = net if context is None else context
    q = F.linear(net, sd[p + "to_q.weight"])
    k = F.linear(ctx, sd[p + "to_k.weight"])
    v = F.linear(ctx, sd[p + "to_v.weight"])

    def fold(z: Tensor) -> Tensor:
        bb, t, d = z.shape
        return z.view(bb, t, heads, d // heads).permute(0, 2, 1, 3).reshape(bb * heads, t, d // heads)

    out = F.scaled_dot_product_attention(fold(q).contiguous(), fold(k).contiguous(), fold(v).contiguous(), None, 0.0)
    out = out.reshape(b, heads, tq, dq // heads).permute(0, 2, 1, 3).contiguous().view(b, tq, dq)
    return F.linear(out, sd[p + "out_linear.0.weight"], sd[p + "out_linear.0.bias"])


def transformer_block(sd: StateDict, p: str, net: Tensor, context: Optional[Tensor], heads: int) -> Tensor:
    """SpatialTransformerBlock._forward (core/mixed_stacks/api.py:806-812): self-attention, cross-attention, GEGLU feed-forward
    (core/activations.py:155-163; channel_mixers.py:25-33 with add_last_dropout=False), each pre-LayerNorm (eps 1e-5) + residual."""
    d = net.shape[-1]
    ln = lambda i, z: F.layer_norm(z, (d,), sd[p + f"norm{i}.weight"], sd[p + f"norm{i}.bias"], 1e-5)  # noqa: E731
    net = cross_attention(sd, p + "attn1.", ln(1, net), None, heads) + net
    net = cross_attention(sd, p + "attn2.", ln(2, net), context, heads) + net
    h, gate = F.linear(ln(3, net), sd[p + "ff.net.0.net.weight"], sd[p + "ff.net.0.net.bias"]).chunk(2, dim=-1)
    return F.linear(h * F.gelu(gate), sd[p + "ff.net.2.linear.weight"], sd[p + "ff.net.2.linear.bias"]) + net


def spatial_transformer(sd: StateDict, p: str, net: Tensor, context: Optional[Tensor], heads: int) -> Tensor:
    """SpatialTransformer.forward (core/mixed_stacks/api.py:866-883, use_linear=False): GroupNorm(32, eps 1e-6), 1x1 conv in,
    [B, HW, C] tokens through the blocks, 1x1 conv out, residual."""
    inp = net
    b, c, h, w = net.shape
    net = F.conv2d(_gn(sd, p + "norm.", net, 1e-6), sd[p + "to_latent.weight"], sd[p + "to_latent.bias"])
    net = net.permute(0, 2, 3, 1).reshape(b, h * w, c)
    i = 0
    while p + f"blocks.{i}.norm1.weight" in sd:
        net = transformer_block(sd, p + f"blocks.{i}.", net, context, heads)
        i += 1
    net = net.permute(0, 2, 1).contiguous().view(b, c, h, w)
    return inp + F.conv2d(net, sd[p + "from_latent.weight"], sd[p + "from_latent.bias"])


# ------------------------------------------------------------------------------------------------------------------------------
# the same computations with every op boundary returned, for the per-op teacher-forced tests (tests/test_unet_ops_gpu.py).
# ``out`` of each is bit-identical to the function above it (tests/test_oracle.py).  Where one tensor feeds two paths (x into
# GroupNorm and the shortcut, a context into several blocks), each path reads its own ``view_as`` of it, so that one backward
# yields each path's gradient apart (the views change no value and no op).  Every non-leaf entry can ``retain_grad()``.
# ------------------------------------------------------------------------------------------------------------------------------
def res_block_ops(sd: StateDict, p: str, net: Tensor, time_net: Tensor) -> Dict[str, Tensor]:
    """``res_block``'s op boundaries: x, x_gn / x_sc (the GroupNorm and shortcut paths' views of x), gn1, silu1, conv1 (with its
    bias), time_silu, t, h (conv1 + t), gn2, silu2, conv2, shortcut (1x1 conv, when the width changes), sum (pre-clamp), out."""
    o: Dict[str, Tensor] = {"x": net, "x_gn": net.view_as(net), "x_sc": net.view_as(net)}
    o["gn1"] = _gn(sd, p + "norm1.", o["x_gn"], 1e-5)
    o["silu1"] = F.silu(o["gn1"])
    o["conv1"] = F.conv2d(o["silu1"], sd[p + "conv1.weight"], sd[p + "conv1.bias"], padding=1)
    inp = o["x_sc"]
    if p + "shortcut.weight" in sd:
        inp = o["shortcut"] = F.conv2d(o["x_sc"], sd[p + "shortcut.weight"], sd[p + "shortcut.bias"])
    o["time_silu"] = F.silu(time_net)
    o["t"] = F.linear(o["time_silu"], sd[p + "time_embedding.weight"], sd[p + "time_embedding.bias"])
    o["h"] = o["conv1"] + o["t"][..., None, None]
    o["gn2"] = _gn(sd, p + "norm2.", o["h"], 1e-5)
    o["silu2"] = F.silu(o["gn2"])
    o["conv2"] = F.conv2d(o["silu2"], sd[p + "conv2.weight"], sd[p + "conv2.bias"], padding=1)
    o["sum"] = inp + o["conv2"]
    fi = torch.finfo(o["sum"].dtype)
    o["out"] = o["sum"].clamp(fi.min, fi.max)
    return o


def cross_attention_ops(sd: StateDict, p: str, net: Tensor, context: Optional[Tensor], heads: int) -> Dict[str, Tensor]:
    """``cross_attention``'s op boundaries: x, q, k, v (the projections, [B, T, L]), attn (the attention output with the heads
    unfolded, [B, Tq, L]) and out (out_linear)."""
    b, tq, dq = net.shape
    ctx = net if context is None else context
    o: Dict[str, Tensor] = {"x": net}
    o["q"] = F.linear(net, sd[p + "to_q.weight"])
    o["k"] = F.linear(ctx, sd[p + "to_k.weight"])
    o["v"] = F.linear(ctx, sd[p + "to_v.weight"])

    def fold(z: Tensor) -> Tensor:
        bb, t, d = z.shape
        return z.view(bb, t, heads, d // heads).permute(0, 2, 1, 3).reshape(bb * heads, t, d // heads)

    out = F.scaled_dot_product_attention(fold(o["q"]).contiguous(), fold(o["k"]).contiguous(), fold(o["v"]).contiguous(), None, 0.0)
    o["attn"] = out.reshape(b, heads, tq, dq // heads).permute(0, 2, 1, 3).contiguous().view(b, tq, dq)
    o["out"] = F.linear(o["attn"], sd[p + "out_linear.0.weight"], sd[p + "out_linear.0.bias"])
    return o


def transformer_block_ops(sd: StateDict, p: str, net: Tensor, context: Optional[Tensor], heads: int) -> Dict[str, Tensor]:
    """``transformer_block``'s op boundaries: x, ln1, attn1.* (``cross_attention_ops`` of the self-attention), x1 (its residual
    sum), ln2, attn2.*, x2, ln3, hg (the GEGLU projection), h / gate (its halves), gelu, prod (h * gelu), ff2, out."""
    d = net.shape[-1]
    ln = lambda i, z: F.layer_norm(z, (d,), sd[p + f"norm{i}.weight"], sd[p + f"norm{i}.bias"], 1e-5)  # noqa: E731
    o: Dict[str, Tensor] = {"x": net}
    o["ln1"] = ln(1, net)
    o.update({"attn1." + k: v for k, v in cross_attention_ops(sd, p + "attn1.", o["ln1"], None, heads).items() if k != "x"})
    o["x1"] = o["attn1.out"] + net
    o["ln2"] = ln(2, o["x1"])
    o.update({"attn2." + k: v for k, v in cross_attention_ops(sd, p + "attn2.", o["ln2"], context, heads).items() if k != "x"})
    o["x2"] = o["attn2.out"] + o["x1"]
    o["ln3"] = ln(3, o["x2"])
    o["hg"] = F.linear(o["ln3"], sd[p + "ff.net.0.net.weight"], sd[p + "ff.net.0.net.bias"])
    o["h"], o["gate"] = o["hg"].chunk(2, dim=-1)
    o["gelu"] = F.gelu(o["gate"])
    o["prod"] = o["h"] * o["gelu"]
    o["ff2"] = F.linear(o["prod"], sd[p + "ff.net.2.linear.weight"], sd[p + "ff.net.2.linear.bias"])
    o["out"] = o["ff2"] + o["x2"]
    return o


def spatial_transformer_ops(sd: StateDict, p: str, net: Tensor, context: Optional[Tensor], heads: int) -> Dict[str, Tensor]:
    """``spatial_transformer``'s op boundaries: x, x_gn / x_res (the GroupNorm and residual paths' views of x), gn, latent_in (to_latent),
    tokens ([B, HW, C]), blocks.{i}.* (``transformer_block_ops``, with blocks.{i}.context the block's view of the context), latent
    ([B, C, H, W]), latent_out (from_latent) and out."""
    b, c, h, w = net.shape
    o: Dict[str, Tensor] = {"x": net, "x_gn": net.view_as(net), "x_res": net.view_as(net)}
    o["gn"] = _gn(sd, p + "norm.", o["x_gn"], 1e-6)
    o["latent_in"] = F.conv2d(o["gn"], sd[p + "to_latent.weight"], sd[p + "to_latent.bias"])
    t = o["tokens"] = o["latent_in"].permute(0, 2, 3, 1).reshape(b, h * w, c)
    i = 0
    while p + f"blocks.{i}.norm1.weight" in sd:
        q = f"blocks.{i}."
        ctx = None if context is None else context.view_as(context)
        if ctx is not None:
            o[q + "context"] = ctx
        o.update({q + k: v for k, v in transformer_block_ops(sd, p + q, t, ctx, heads).items() if k != "x"})
        t = o[q + "out"]
        i += 1
    o["latent"] = t.permute(0, 2, 1).contiguous().view(b, c, h, w)
    o["latent_out"] = F.conv2d(o["latent"], sd[p + "from_latent.weight"], sd[p + "from_latent.bias"])
    o["out"] = o["x_res"] + o["latent_out"]
    return o


def resample_ops(sd: StateDict, p: str, net: Tensor) -> Dict[str, Tensor]:
    """The op boundaries of the resampling child at ``p`` as ``_sequential`` runs it: ResDownsample (``net.weight``: x, out) or
    ResUpsample (``conv.weight``: x, up = the nearest 2x copy, out)."""
    o: Dict[str, Tensor] = {"x": net}
    if p + "net.weight" in sd:
        o["out"] = F.conv2d(net, sd[p + "net.weight"], sd[p + "net.bias"], stride=2, padding=1)
    else:
        o["up"] = F.interpolate(net, scale_factor=2, mode="nearest")
        o["out"] = F.conv2d(o["up"], sd[p + "conv.weight"], sd[p + "conv.bias"], padding=1)
    return o


def _sequential(sd: StateDict, p: str, net: Tensor, time_net: Tensor, context: Optional[Tensor], heads: int) -> Tensor:
    """TimestepAttnSequential.forward (unet.py:31-45): children dispatched by type; here by the parameter names they own."""
    j = 0
    while any(k.startswith(p + f"{j}.") for k in sd):
        q = p + f"{j}."
        if q + "norm1.weight" in sd:
            net = res_block(sd, q, net, time_net)
        elif q + "to_latent.weight" in sd:
            net = spatial_transformer(sd, q, net, context, heads)
        elif q + "net.weight" in sd:      # ResDownsample with conv (residual.py:108-115): 3x3, stride 2, padding 1
            net = F.conv2d(net, sd[q + "net.weight"], sd[q + "net.bias"], stride=2, padding=1)
        elif q + "conv.weight" in sd:     # ResUpsample (residual.py:139-148): nearest x2 then 3x3 conv
            net = F.conv2d(F.interpolate(net, scale_factor=2, mode="nearest"), sd[q + "conv.weight"], sd[q + "conv.bias"], padding=1)
        elif q + "weight" in sd:          # the stem convolution (unet.py:213-217)
            net = F.conv2d(net, sd[q + "weight"], sd[q + "bias"], padding=1)
        else:
            raise KeyError(f"unrecognised block at {q}")
        j += 1
    return net


def forward(sd: StateDict, net: Tensor, timesteps: Tensor, context: Optional[Tensor], cfg: Dict) -> Tensor:
    """UNetDiffuser.forward (unet.py:275-322) without labels / control: time MLP, down path with skip stack, middle, up path
    with concatenated skips, GroupNorm(32, eps 1e-5) -> SiLU -> conv3x3 head."""
    heads = cfg["num_heads"]
    t = timestep_embedding(timesteps, cfg["start_channels"], net.dtype)
    t = F.linear(t, sd["time_embedding.0.weight"], sd["time_embedding.0.bias"])
    t = F.linear(F.silu(t), sd["time_embedding.2.weight"], sd["time_embedding.2.bias"])
    nets: List[Tensor] = []
    i = 0
    while any(k.startswith(f"input_blocks.{i}.") for k in sd):
        net = _sequential(sd, f"input_blocks.{i}.", net, t, context, heads)
        nets.append(net)
        i += 1
    net = _sequential(sd, "residual.", net, t, context, heads)
    i = 0
    while any(k.startswith(f"output_blocks.{i}.") for k in sd):
        net = torch.cat([net, nets.pop()], dim=1)
        net = _sequential(sd, f"output_blocks.{i}.", net, t, context, heads)
        i += 1
    net = F.silu(F.group_norm(net, 32, sd["head.0.weight"], sd["head.0.bias"], 1e-5))
    return F.conv2d(net, sd["head.2.weight"], sd["head.2.bias"], padding=1)


def synthetic_state_dict(shapes: List[Tuple[str, Tuple[int, ...]]], seed: int = 0) -> StateDict:
    """Random weights for every key (the reference zero-initialises conv2 / from_latent / the head conv, unet.py:271 and
    residual.py:196, which would hide most of the network from a parity check)."""
    g = torch.Generator().manual_seed(seed)
    sd: StateDict = {}
    for key, shape in shapes:
        if "norm" in key and key.endswith("weight") or key == "head.0.weight":
            sd[key] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif key.endswith("bias"):
            sd[key] = 0.02 * torch.randn(shape, generator=g)
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            sd[key] = torch.randn(shape, generator=g) * (0.7 / math.sqrt(max(fan_in, 1)))
    return sd


def train_step(sd: StateDict, x: Tensor, timesteps: Tensor, context: Tensor, upstream: Tensor, cfg: Dict, *, autocast_bf16: bool):
    """Forward + backward with ``upstream`` as the gradient of the predicted noise (the reference's DDPM loss is an MSE to the
    noise, models/cv/diffusion.py:56-86: its gradient is exactly such a tensor)."""
    params = {k: v.detach().clone().requires_grad_(True) for k, v in sd.items()}
    with torch.autocast(x.device.type, dtype=torch.bfloat16, enabled=autocast_bf16):
        out = forward(params, x, timesteps, context, cfg)
    (out.float() * upstream).sum().backward()
    return out.detach(), {k: v.grad for k, v in params.items()}
