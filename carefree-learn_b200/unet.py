"""The SD-v1.5 UNet, ``UNetDiffuser`` (cflearn/modules/multimodal/diffusion/unet.py:97-322), assembled from the native blocks
(BASELINE.json configs[4]; SURVEY.md 8f row N3), and the DDPM noise-prediction loss it trains with.

``UNetDiffuserB200`` takes the reference's constructor keywords, builds its children in the reference's order under the
reference's names, so ``state_dict`` keys, shapes and order are the reference's, and runs them on CHANNELS-LAST bf16
activations:

    timestep MLP        sinusoidal embedding (torch glue, fp32) -> Linear -> SiLU -> Linear   ops.gemm with the bias epilogue
    input_blocks.0      Conv2d(in, start) on the input zero-padded to 64 channels               ops.pad_channels, conv3x3
    input_blocks.1..    ResidualBlockWithTimeEmbeddingB200, SpatialTransformerB200, ResDownsampleB200
    residual            ResBlock, SpatialTransformer, ResBlock
    output_blocks       torch.cat([net, skip], dim=1), then ResBlock, SpatialTransformer, ResUpsampleB200
    head                GroupNorm(32) + SiLU, Conv2d(start, out) with its output channels zero-padded to 64

Rounding points are eager's under bf16 autocast (oracle/unet_oracle.py::forward).  The time embedding is fp32 and rounded to
bf16 once, at the first Linear, so an fp32 and a bf16 latent give the same bits.  The stem and head add their biases as
eager's convolution does on CUDA, bf16(bf16(conv) + bias), through the per-image epilogue (DESIGN.md section 2).  Padding
with exact zeros leaves every fp32 partial sum of the real channels unchanged, so the padded convolutions compute what the
4-channel ones do.  The skip concatenation is ``torch.cat`` on channels-last tensors, so its result is channels-last and the
next ResBlock reads it without a copy; autograd slices its gradient and adds each skip's two bf16 gradients, which round the
same in either order.

``noise_prediction_loss(pred, noise)`` is ``DDPMStep.loss_fn`` (cflearn/models/cv/diffusion.py:44-94) at its defaults.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor, nn

from . import checkpoint, ops
from ._cabi import B200Error
from .arena import ParamArena
from .attention import _bf, _check_cuda
from .spatial_transformer import SpatialTransformerB200
from .unet_blocks import (ResDownsampleB200, ResidualBlockWithTimeEmbeddingB200, ResUpsampleB200, _bias_rows, _nhwc,
                          check_geometry, check_resample_geometry)

PAD_CHANNELS = 64  # the convolutions reduce over 64-channel blocks


def _f32(*shape: int, device: torch.device) -> Tensor:
    return torch.empty(shape, dtype=torch.float32, device=device)


# ------------------------------------------------------------------------------------------------------------------------------
# the pieces between the blocks, each one checkpoint.OpFn node
# ------------------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class _TimeMLPOp:
    """time_embedding = Linear -> SiLU -> Linear on (emb fp32 [B, start], w0, b0, w2, b2): bf16 [B, 4 start].  Backward gets the
    sum of every ResBlock's time-embedding gradient."""

    def forward(self, emb: Tensor, w0: Tensor, b0: Tensor, w2: Tensor, b2: Tensor) -> Tuple[Tensor, tuple]:
        e = emb.to(torch.bfloat16).contiguous()  # autocast's cast at the first Linear
        w0b, w2b = _bf(w0), _bf(w2)
        h = ops.gemm(e, w0b, bias=_bf(b0))
        a = F.silu(h).contiguous()  # eager's F.silu on the bf16 tensor (fp32 maths, bf16 result)
        return ops.gemm(a, w2b, bias=_bf(b2)), (e, h, a, w0b, w2b)

    def backward(self, saved: tuple, dt: Tensor, pg: Optional[checkpoint.ParamGrads] = None) -> tuple:
        pg = pg or checkpoint.NO_GRADS
        e, h, a, w0b, w2b = saved
        dev = dt.device
        dt = dt.to(torch.bfloat16).contiguous()
        dw2 = ops.wgrad(dt, a, pg.out(3, tuple(w2b.shape), dev), **pg.mode)
        db2 = ops.colsum(dt, pg.out(4, (w2b.shape[0],), dev), **pg.mode)
        dh = torch.ops.aten.silu_backward(ops.gemm(dt, w2b, b_mn_major=True), h).contiguous()
        dw0 = ops.wgrad(dh, e, pg.out(1, tuple(w0b.shape), dev), **pg.mode)
        db0 = ops.colsum(dh, pg.out(2, (w0b.shape[0],), dev), **pg.mode)
        return None, dw0, db0, dw2, db2


def stem_conv(net: Tensor, weight: Tensor, bias: Tensor, padded: bool = False) -> Tuple[Tensor, Tensor, Tensor]:
    """Conv2d(C, Cout, 3, padding 1) of net fp32 / bf16 [B, C, H, W] (C <= 64): the input zero-padded to 64 channels (x, bf16
    [B, H, W, 64]) and the weight to [Cout, 64, 3, 3] (wp).  Returns (out bf16 [B, H, W, Cout] = bf16(bf16(conv) + bias), x, wp).
    ``padded``: net is already x (``ops.q_sample_pad``'s output)."""
    C = weight.shape[1]
    x = net if padded else ops.pad_channels(net, PAD_CHANNELS)
    wp = F.pad(weight, (0, 0, 0, 0, 0, PAD_CHANNELS - C))
    out = ops.conv3x3(x, ops.pack_conv3x3_weight(wp), epilogue=ops.EPI_BIAS_ADD_PER_IMAGE_BF16, aux=_bias_rows(bias, net.shape[0]))
    return out, x, wp


def stem_conv_bwd(d: Tensor, x: Tensor, wp: Tensor, C: int, need_dx: bool) -> Tuple[Optional[Tensor], Tensor, Tensor]:
    """Backward of ``stem_conv`` for d bf16 [B, H, W, Cout]: (dx bf16 [B, H, W, C] view or None, dw fp32 [Cout, C, 3, 3], db fp32
    [Cout]), the weight and bias gradients rounded to bf16 like eager's."""
    Cout = wp.shape[0]
    dw = ops.unpack_conv3x3_weight(ops.conv3x3_wgrad(d, x), PAD_CHANNELS)[:, :C].contiguous()
    db = ops.colsum(d.view(-1, Cout), _f32(Cout, device=d.device))
    dx = ops.conv3x3(d, ops.pack_conv3x3_weight_dgrad(wp))[..., :C] if need_dx else None
    return dx, dw, db


def head_conv(y: Tensor, weight: Tensor, bias: Tensor) -> Tuple[Tensor, Tensor]:
    """Conv2d(C, Co, 3, padding 1) of y bf16 [B, H, W, C] (Co <= 64) with its output channels zero-padded to 64 (weight rows wp
    and bias), so that one width serves the forward, the weight gradient and the input gradient, which reduces over them.
    Returns (out bf16 [B, H, W, Co] dense = bf16(bf16(conv) + bias), wp)."""
    B = y.shape[0]
    Co = weight.shape[0]
    wp = F.pad(weight, (0, 0, 0, 0, 0, 0, 0, PAD_CHANNELS - Co))
    out = ops.conv3x3(y, ops.pack_conv3x3_weight(wp), epilogue=ops.EPI_BIAS_ADD_PER_IMAGE_BF16,
                      aux=_bias_rows(F.pad(bias, (0, PAD_CHANNELS - Co)), B))
    return out[..., :Co].contiguous(), wp


def head_conv_bwd(dout: Tensor, y: Tensor, wp: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    """Backward of ``head_conv`` for dout fp32 / bf16 [B, Co, H, W] (contiguous NCHW or channels-last), padded back to 64 channels:
    (dy bf16 [B, H, W, C], dw fp32 [Co, C, 3, 3], db fp32 [Co]), the weight and bias gradients rounded to bf16 like eager's."""
    C, Co = y.shape[3], dout.shape[1]
    d = ops.pad_channels(dout, PAD_CHANNELS)
    dw = ops.unpack_conv3x3_weight(ops.conv3x3_wgrad(d, y), C)[:Co]
    db = ops.colsum(d.view(-1, PAD_CHANNELS), _f32(PAD_CHANNELS, device=d.device))[:Co]
    return ops.conv3x3(d, ops.pack_conv3x3_weight_dgrad(wp)), dw, db


@dataclass(frozen=True)
class _StemOp:
    """input_blocks.0.0 as an op on (net [B, C, H, W] fp32 / bf16, weight, bias).  ``need_dx``: the latent requires grad (a
    DDPM's noised latent does not).  ``padded``: net is the stem's padded bf16 input [B, H, W, 64] (the DDPM's noised latent)."""
    channels: int
    need_dx: bool
    padded: bool = False

    def forward(self, net: Tensor, weight: Tensor, bias: Tensor) -> Tuple[Tensor, tuple]:
        out, x, wp = stem_conv(net, weight, bias, self.padded)
        return out.permute(0, 3, 1, 2), (x, wp)

    def backward(self, saved: tuple, dout: Tensor, pg: Optional[checkpoint.ParamGrads] = None) -> tuple:
        pg = pg or checkpoint.NO_GRADS
        x, wp = saved
        dx, dw, db = stem_conv_bwd(_nhwc(dout), x, wp, self.channels, self.need_dx)
        return None if dx is None else dx.permute(0, 3, 1, 2), pg.put(1, dw), pg.put(2, db)


@dataclass(frozen=True)
class _HeadOp:
    """head = GroupNorm(32) + SiLU, then ``head_conv``, as an op on (net [B, C, H, W] bf16, norm w / b, conv w / b): bf16
    [B, Co, H, W] with dense channels-last strides."""
    eps: float

    def forward(self, net: Tensor, gn_w: Tensor, gn_b: Tensor, weight: Tensor, bias: Tensor) -> Tuple[Tensor, tuple]:
        xt = _nhwc(net)
        B, H, W, C = xt.shape
        g, b = gn_w.float().contiguous(), gn_b.float().contiguous()
        y, m, r = ops.groupnorm_silu_fwd(xt.view(B, H * W, C), g, b, self.eps)
        out, wp = head_conv(y.view(B, H, W, C), weight, bias)
        return out.permute(0, 3, 1, 2), (xt, y, m, r, g, b, wp)

    def backward(self, saved: tuple, dout: Tensor, pg: Optional[checkpoint.ParamGrads] = None) -> tuple:
        pg = pg or checkpoint.NO_GRADS
        xt, y, m, r, g, b, wp = saved
        B, H, W, C = xt.shape
        if not (dout.is_contiguous() or dout.is_contiguous(memory_format=torch.channels_last)):
            dout = dout.contiguous()
        dy, dw, db = head_conv_bwd(dout, y.view(B, H, W, C), wp)
        dx, dg, dbe = ops.groupnorm_silu_bwd(xt.view(B, H * W, C), dy.view(B, H * W, C), g, b, m, r, **pg.norm_kw(1, 2))
        return dx.view(B, H, W, C).permute(0, 3, 1, 2), dg, dbe, pg.put(3, dw), pg.put(4, db)


def timestep_embedding(timesteps: Tensor, frequency: Tensor) -> Tensor:
    """unet.py:52-74 (cos first, then sin) in fp32, with the reference's frequencies
    ``frequency`` [half] (computed on the host, as the reference does, and kept on the device)."""
    args = timesteps[:, None].float() * frequency[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


# ------------------------------------------------------------------------------------------------------------------------------
# the loss
# ------------------------------------------------------------------------------------------------------------------------------
def _dense(t: Tensor) -> Tensor:
    return t if t.is_contiguous() or t.is_contiguous(memory_format=torch.channels_last) else t.contiguous()


class _NoiseLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx: Any, pred: Tensor, noise: Tensor) -> Tensor:  # type: ignore[override]
        pred = _dense(pred)
        cl = pred.is_contiguous(memory_format=torch.channels_last) and not pred.is_contiguous()
        noise = noise.contiguous(memory_format=torch.channels_last if cl else torch.contiguous_format)
        ctx.save_for_backward(pred, noise)
        return ops.noise_prediction_loss(pred, noise).reshape(())

    @staticmethod
    def backward(ctx: Any, grad_out: Tensor):  # type: ignore[override]
        pred, noise = ctx.saved_tensors
        return ops.noise_prediction_loss(pred, noise, grad_out=grad_out.reshape(1).float().contiguous()), None


def noise_prediction_loss(pred: Tensor, noise: Tensor) -> Tensor:
    """``DDPMStep.loss_fn`` (cflearn/models/cv/diffusion.py:44-94) at its defaults, ``loss_type="l2"``,
    ``parameterization="eps"``, ``l_simple_weight=1``, ``original_elbo_weight=0`` and a zero ``log_var``:
    ``F.mse_loss(pred, noise, reduction="none").mean(dim=(1, 2, 3)).mean()`` under bf16 autocast, i.e. in fp32.

    ``pred``: bf16 [B, C, H, W] (the UNet's output); ``noise``: fp32 or bf16, the same shape.  Returns the fp32 scalar loss,
    summed in a fixed order (bit-identical run to run); its gradient is eager's bit for bit, bf16 in pred's layout.  Other loss
    settings (``l1``, the ``x0`` / ``v`` parameterizations, a learned or non-zero ``log_var``, an ELBO weight) are not
    implemented: compute those losses in PyTorch on the UNet's output."""
    return _NoiseLossFn.apply(pred, noise)


# ------------------------------------------------------------------------------------------------------------------------------
# the module
# ------------------------------------------------------------------------------------------------------------------------------
class UNetDiffuserB200(nn.Module):
    """Drop-in for cflearn's ``UNetDiffuser`` on the native kernels (bf16 activations, fp32 parameters; CUDA only).

    ``forward(net, *, timesteps, context=None)``: ``net`` fp32 or bf16 [B, in_channels, H, W] in either memory format,
    ``timesteps`` an integer or float [B] tensor, ``context`` fp32 or bf16 [B, Tk, context_dim] (cast to bf16 once).  Returns
    bf16 [B, out_channels, H, W] with channels-last strides.  A geometry the blocks cannot tile raises ``B200Error`` before any
    launch, naming the first level that fails; at SD-v1.5's four levels, 64 x 64 latents (512 px) are admitted."""

    def __init__(self, in_channels: int, out_channels: int, *, num_heads: Optional[int] = None, num_head_channels: Optional[int] = None,
                 use_spatial_transformer: bool = False, num_transformer_layers: int = 1, context_dim: Optional[int] = None,
                 signal_dim: int = 2, start_channels: int = 320, num_res_blocks: int = 2,
                 attention_downsample_rates: Tuple[int, ...] = (1, 2, 4), dropout: float = 0.0,
                 channel_multipliers: Tuple[int, ...] = (1, 2, 4, 8), resample_with_conv: bool = True,
                 resample_with_resblock: bool = False, use_scale_shift_norm: bool = False, num_classes: Optional[int] = None,
                 use_linear_in_transformer: bool = False, use_checkpoint: bool = False,
                 hooks_kwargs: Optional[Dict[str, Any]] = None) -> None:
        super().__init__()
        what = "UNetDiffuserB200"
        refused = [(not use_spatial_transformer, "use_spatial_transformer=False (MultiHeadSpatialAttention)"),
                   (not resample_with_conv, "resample_with_conv=False"), (resample_with_resblock, "resample_with_resblock=True"),
                   (use_scale_shift_norm, "use_scale_shift_norm"), (num_classes is not None, "num_classes (label embedding)"),
                   (dropout > 0.0, "dropout > 0"), (signal_dim != 2, f"signal_dim={signal_dim} (2-D signals only)"),
                   (use_linear_in_transformer, "use_linear_in_transformer"), (hooks_kwargs is not None, "hooks_kwargs")]
        for bad, option in refused:
            if bad:
                raise NotImplementedError(f"{what}: {option} is not supported")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.context_dim, self.start_channels = context_dim, start_channels
        self.num_res_blocks, self.channel_multipliers = num_res_blocks, tuple(channel_multipliers)
        self.attention_downsample_rates = tuple(attention_downsample_rates)
        self.use_checkpoint = use_checkpoint
        if in_channels > PAD_CHANNELS or out_channels > PAD_CHANNELS:
            raise NotImplementedError(f"{what}: in_channels and out_channels must be at most {PAD_CHANNELS} (the padded stem and head)")
        half = start_channels // 2
        frequency = torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
        self.register_buffer("_frequency", frequency, persistent=False)

        tdim = start_channels * 4
        self.time_embedding = nn.Sequential(nn.Linear(start_channels, tdim), nn.SiLU(), nn.Linear(tdim, tdim))
        # (level, kind, Cin, Cout) of every block, for the geometry check at the start of forward
        self._plan: List[Tuple[int, str, int, int]] = []

        def res_block(level: int, cin: int, cout: int) -> nn.Module:
            self._plan.append((level, "res", cin, cout))
            return ResidualBlockWithTimeEmbeddingB200(cin, cout, signal_dim=signal_dim, norm_eps=1.0e-5, time_embedding_channels=tdim,
                                                      dropout=dropout, use_checkpoint=use_checkpoint)

        def attn_block(c: int) -> nn.Module:
            if num_head_channels is not None:
                heads, head_c = c // num_head_channels, num_head_channels
            elif num_heads is None:
                raise ValueError("either `num_heads` or `num_head_channels` should be provided")
            else:
                heads, head_c = num_heads, c // num_heads
            return SpatialTransformerB200(c, heads, head_c, num_layers=num_transformer_layers, context_dim=context_dim,
                                          use_checkpoint=use_checkpoint)

        stem = nn.Conv2d(in_channels, start_channels, 3, padding=1)
        input_blocks: List[nn.Module] = [nn.ModuleList([stem])]
        chans = [start_channels]
        c, rate, level = start_channels, 1, 0
        for i, mult in enumerate(channel_multipliers):
            for _ in range(num_res_blocks):
                blocks = [res_block(level, c, mult * start_channels)]
                c = mult * start_channels
                if rate in attention_downsample_rates:
                    blocks.append(attn_block(c))
                input_blocks.append(nn.ModuleList(blocks))
                chans.append(c)
            if i != len(channel_multipliers) - 1:
                self._plan.append((level, "down", c, c))
                input_blocks.append(nn.ModuleList([ResDownsampleB200(c, True, signal_dim=signal_dim, out_channels=c)]))
                rate, level = rate * 2, level + 1
                chans.append(c)
        self.input_blocks = nn.ModuleList(input_blocks)
        self.residual = nn.ModuleList([res_block(level, c, c), attn_block(c), res_block(level, c, c)])
        output_blocks: List[nn.Module] = []
        for i, mult in list(enumerate(channel_multipliers))[::-1]:
            for j in range(num_res_blocks + 1):
                cout = start_channels * mult
                blocks = [res_block(level, c + chans.pop(), cout)]
                c = cout
                if rate in attention_downsample_rates:
                    blocks.append(attn_block(c))
                if i != 0 and j == num_res_blocks:
                    self._plan.append((level, "up", c, c))
                    blocks.append(ResUpsampleB200(c, True, signal_dim=signal_dim, out_channels=c))
                    rate, level = rate // 2, level - 1
                output_blocks.append(nn.ModuleList(blocks))
        self.output_blocks = nn.ModuleList(output_blocks)
        self.levels = len(channel_multipliers)
        head_conv = nn.Conv2d(start_channels, out_channels, 3, padding=1)
        with torch.no_grad():  # zero_module(head_conv), as the reference
            head_conv.weight.zero_()
            head_conv.bias.zero_()
        self.head = nn.Sequential(nn.GroupNorm(32, c), nn.SiLU(), head_conv)

    _grad_arena: Optional["UNetGradArena"] = None  # set by enable_grad_arena

    def check_geometry(self, B: int, H: int, W: int) -> None:
        """Raise one ``B200Error`` naming the first level (and the rule) whose H x W grid the blocks cannot tile."""
        for level in range(self.levels):
            h, w = H >> level, W >> level
            try:
                if (h << level) != H or (w << level) != W:
                    raise B200Error(f"H = {H} and W = {W} must be divisible by {1 << level}")
                for lv, kind, cin, cout in self._plan:
                    if lv != level:
                        continue
                    if kind == "res":
                        check_geometry(B, h, w, cin, cout)
                    elif kind == "down":
                        check_resample_geometry("ResDownsampleB200", False, h, w, cin, cout)
                    else:
                        check_resample_geometry("ResUpsampleB200", True, h, w, cin, cout)
            except B200Error as err:
                raise B200Error(f"UNetDiffuserB200: level {level} ({h} x {w} of a {H} x {W} latent): {err}") from None

    @staticmethod
    def _run(blocks: nn.ModuleList, net: Tensor, time_net: Tensor, context: Optional[Tensor]) -> Tensor:
        for layer in blocks:  # TimestepAttnSequential.forward (unet.py:31-45)
            if isinstance(layer, ResidualBlockWithTimeEmbeddingB200):
                net = layer(net, time_net)
            elif isinstance(layer, SpatialTransformerB200):
                net = layer(net, context)
            else:
                net = layer(net)
        return net

    def forward(self, net: Tensor, *, timesteps: Tensor, context: Optional[Tensor] = None, labels: Optional[Tensor] = None,
                control: Optional[List[Tensor]] = None, only_mid_control: bool = False) -> Tensor:
        what = "UNetDiffuserB200"
        if labels is not None:
            raise NotImplementedError(f"{what}: labels (num_classes, the label embedding) are not supported")
        if control is not None:
            raise NotImplementedError(f"{what}: control (ControlNet residuals) is not supported")
        if net.dim() != 4 or net.shape[1] != self.in_channels or net.dtype not in (torch.float32, torch.bfloat16):
            raise B200Error(f"{what}: net must be fp32 or bf16 [B, {self.in_channels}, H, W]")
        B, _, H, W = net.shape
        if timesteps.shape != (B,):
            raise B200Error(f"{what}: timesteps must be [B] = [{B}]")
        if context is not None and (context.dim() != 3 or context.shape[0] != B or context.shape[2] != self.context_dim):
            raise B200Error(f"{what}: context must be [B, Tk, {self.context_dim}]")
        self.check_geometry(B, H, W)
        _check_cuda(what, net, timesteps, context)
        if not (net.is_contiguous() or net.is_contiguous(memory_format=torch.channels_last)):
            net = net.contiguous()
        return self._body(net, False, timesteps, context)

    def forward_padded(self, x: Tensor, timesteps: Tensor, context: Optional[Tensor] = None) -> Tensor:
        """``forward`` on the stem's padded input x, bf16 [B, H, W, 64] with channels >= in_channels zero (``ops.q_sample_pad``'s
        output, which needs no gradient)."""
        what = "UNetDiffuserB200"
        if x.dim() != 4 or x.shape[3] != PAD_CHANNELS or x.dtype != torch.bfloat16 or not x.is_contiguous():
            raise B200Error(f"{what}: the padded input must be contiguous bf16 [B, H, W, {PAD_CHANNELS}]")
        B, H, W, _ = x.shape
        if timesteps.shape != (B,):
            raise B200Error(f"{what}: timesteps must be [B] = [{B}]")
        if context is not None and (context.dim() != 3 or context.shape[0] != B or context.shape[2] != self.context_dim):
            raise B200Error(f"{what}: context must be [B, Tk, {self.context_dim}]")
        self.check_geometry(B, H, W)
        _check_cuda(what, x, timesteps, context)
        return self._body(x, True, timesteps, context)

    def _body(self, net: Tensor, padded: bool, timesteps: Tensor, context: Optional[Tensor]) -> Tensor:
        if self._grad_arena is not None:
            self._grad_arena.begin()
        time_net = self._time_mlp(timestep_embedding(timesteps, self._frequency))
        ctx = None if context is None else context.to(torch.bfloat16)  # autocast's cast at to_k / to_v, made once
        h = self._stem(net, padded)
        skips = [h]
        for blocks in self.input_blocks[1:]:
            h = self._run(blocks, h, time_net, ctx)
            skips.append(h)
        h = self._run(self.residual, h, time_net, ctx)
        for blocks in self.output_blocks:
            h = self._run(blocks, torch.cat([h, skips.pop()], dim=1), time_net, ctx)
        return self._head(h)

    def _time_mlp(self, emb: Tensor) -> Tensor:
        te = self.time_embedding
        return checkpoint.OpFn.apply(_TimeMLPOp(), False, emb, te[0].weight, te[0].bias, te[2].weight, te[2].bias)

    def _stem(self, net: Tensor, padded: bool = False) -> Tensor:
        stem = self.input_blocks[0][0]
        return checkpoint.OpFn.apply(_StemOp(self.in_channels, net.requires_grad, padded), False, net, stem.weight, stem.bias)

    def _head(self, net: Tensor) -> Tensor:
        gn, conv = self.head[0], self.head[2]
        return checkpoint.OpFn.apply(_HeadOp(gn.eps), False, net, gn.weight, gn.bias, conv.weight, conv.bias)


# ------------------------------------------------------------------------------------------------------------------------------
# the flat gradient arena
# ------------------------------------------------------------------------------------------------------------------------------
SHRINK_LAUNCHES = 4  # persistent launches (convolutions, GEMMs) that leave the communicator's SMs free after a bucket starts


def bucket_plan(unet: UNetDiffuserB200) -> List[Tuple[str, List[str]]]:
    """The all-reduce buckets in the order backward completes them, each a top-level child: ``head``, the output blocks last
    first, ``residual``, the input blocks last first, then ``stem``: the stem and the timestep MLP, whose gradient is complete
    only once every ResBlock has added its share.  Keys are ``unet.named_parameters()`` names, in state_dict order inside a
    bucket."""
    names = [n for n, _ in unet.named_parameters()]

    def under(prefix: str) -> List[str]:
        return [n for n in names if n.startswith(prefix + ".")]

    plan = [("head", under("head"))]
    plan += [(f"output_blocks.{i}", under(f"output_blocks.{i}")) for i in reversed(range(len(unet.output_blocks)))]
    plan += [("residual", under("residual"))]
    plan += [(f"input_blocks.{i}", under(f"input_blocks.{i}")) for i in reversed(range(1, len(unet.input_blocks)))]
    plan += [("stem", under("input_blocks.0") + under("time_embedding"))]
    return plan


class UNetGradArena:
    """The UNet's parameters in one ``arena.ParamArena`` laid out by ``bucket_plan``, each parameter carrying a
    ``checkpoint.GradSlot``: every op's backward writes its parameter gradients straight into their views (overwriting, or adding
    while the parameters hold gradients, ``ParamArena.claim_grads``), and ``p.grad`` is the view.  When a bucket's last gradient
    is written it is handed to ``reducer.ready`` (``dp.NativeBucketReducer``), which all-reduces it on a side stream while
    backward goes on; the persistent kernels launched next then leave the communicator's SMs free (``shrink_next``).

    It is the DDPM module's one exchange site (``arena.ArenaModule.exchanges``): ``arena``, ``buckets()``, ``reducer`` and
    ``shrink_next``.

    The arena is built on the parameters' device by its first ``arena.ensure()`` (the UNet's forward calls ``begin``, which
    does it, and rebuilds it after ``.to(device)``), so a module constructed on the host holds no second copy there.  Each forward
    also restarts the buckets' counts: a bucket is complete when each of its trainable parameters' gradients was written once
    since (``check``)."""

    def __init__(self, unet: UNetDiffuserB200) -> None:
        params = dict(unet.named_parameters())
        self.plan = bucket_plan(unet)
        self.arena = ParamArena([(k, tuple(params[k].shape)) for _, keys in self.plan for k in keys], bf16_shadow=False)
        self.arena.params = {k: params[k] for _, keys in self.plan for k in keys}  # attached by the first ensure()
        self.reducer: Any = None
        self._shrunk = False
        self._buckets = {name: checkpoint.Bucket(name, len(keys), self._ready) for name, keys in self.plan}
        for name, keys in self.plan:
            for k in keys:
                setattr(params[k], checkpoint.SLOT_ATTR, checkpoint.GradSlot(self.arena, k, self._buckets[name]))
        self._params = params
        self._unet = unet
        unet._grad_arena = self

    def buckets(self) -> Dict[str, List[List[str]]]:
        return {name: [keys] for name, keys in self.plan}

    def begin(self) -> None:
        """At the start of a forward: the arena on the parameters' device, and every bucket waiting for the gradients of its
        trainable parameters (a frozen parameter's op skips its slot)."""
        self.arena.ensure()
        for name, keys in self.plan:
            self._buckets[name].reset(sum(self._params[k].requires_grad for k in keys))

    def check(self) -> None:
        """Raise ``B200Error`` unless every bucket was completed exactly once since the last forward, i.e. each was handed to the
        reducer after all of its gradients were written: anything else would skip or truncate a bucket's exchange."""
        bad = [f"{b.name} ({b.size - b.left} of {b.size} written)" for b in self._buckets.values() if b.left != 0]
        if bad:
            raise B200Error("UNetGradArena: gradient buckets not completed exactly once by this backward (one forward, then one "
                            f"backward per exchange): {', '.join(bad)}")

    def end_backward(self) -> None:
        """Lift what is left of a lowered persistent grid, so that it cannot reach the next step's launches."""
        if self._shrunk:
            from . import _cabi
            _cabi.lib().b200_set_persistent_ctas(0, 0)
            self._shrunk = False

    def _ready(self, name: str) -> None:
        if self.reducer is not None:
            self.reducer.ready(name)

    @property
    def shrink_next(self) -> int:
        return 0

    @shrink_next.setter
    def shrink_next(self, ctas: int) -> None:
        if ctas > 0:
            from . import _cabi
            _cabi.lib().b200_set_persistent_ctas(ops.num_sms() - ctas, SHRINK_LAUNCHES)
            self._shrunk = True

    def close(self) -> None:
        """Take the slots off the parameters: their gradients go back to autograd."""
        for p in self._params.values():
            if hasattr(p, checkpoint.SLOT_ATTR):
                delattr(p, checkpoint.SLOT_ATTR)
        self._unet._grad_arena = None


def enable_grad_arena(unet: UNetDiffuserB200) -> UNetGradArena:
    """Put the UNet's parameters in a flat arena whose gradient views their ops' backwards write directly (``UNetGradArena``).
    Keys, shapes and ``state_dict`` order do not change; the arena is built on the parameters' device by the next forward (or
    ``arena.ensure()``).  ``close()`` on the result turns it off."""
    return UNetGradArena(unet)
