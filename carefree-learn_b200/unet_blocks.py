"""The SD-v1.5 UNet's ``ResidualBlockWithTimeEmbedding`` (cflearn/modules/core/convs/residual.py:154-253) on the native kernels,
forward and backward (BASELINE.json configs[4]; SURVEY.md 8f row N3), as ``UNetDiffuser`` builds it
(cflearn/modules/multimodal/diffusion/unet.py:151-161), on CHANNELS-LAST bf16 activations:

    GroupNorm(32) -> SiLU -> conv3x3 + Linear(SiLU(time))[b, c]     b200_groupnorm_silu_fwd, b200_conv3x3_nhwc_bf16 with the
                                                                    per-image epilogue (t from b200_gemm_bf16)
    GroupNorm -> SiLU -> Dropout(0) -> conv3x3 + shortcut, clamped  conv3x3 with the clamped bf16 residual epilogue; the shortcut is
                                                                    x, or the 1x1 conv = a plain GEMM on [B*H*W, Cin] when the width changes

Rounding points are eager's under bf16 autocast (oracle/unet_oracle.py::res_block): GroupNorm / SiLU in fp32 with one bf16
rounding at the conv input, every conv / Linear output rounded to bf16, the two adds (time embedding, shortcut) in bf16, then
the clamp to bf16's finite range (safe_clip_).  One difference: our conv adds its bias in fp32 and rounds once, eager rounds
the product and adds the bias in a second bf16 op.

Backward, with eager's bf16 rounding points and every conv / Linear parameter gradient rounded to bf16 (DESIGN.md section 2):
conv2's weight gradient (b200_conv3x3_wgrad_nhwc_bf16), its input gradient (conv3x3 with flipped weights) and bias gradient
(column sums of dout, also the shortcut's bias gradient); GroupNorm2 + SiLU backward gives dh; one pass over dh
(b200_colsum_per_image_bf16) gives the time embedding's upstream gradient dt [B, C] and conv1's bias gradient; conv1's weight and
input gradients; GroupNorm1 + SiLU backward, plus the shortcut path's gradient (dout, or dout . Ws) in one bf16 add; the time
embedding's weight / bias gradients from dt and dtime = silu_backward(bf16(dt . Wt), time) on the [B, tdim] rows.  The one
intended difference from eager: the backward treats the clamp as the identity, where eager zeroes the gradient of an element
whose sum overflowed bf16 (a block whose output overflows is already broken; the clamp only keeps the forward finite).

``ResidualBlockWithTimeEmbeddingB200`` is the drop-in module: one ``checkpoint.OpFn`` node over ``res_block_fwd`` /
``res_block_bwd`` that keeps their saved tensors, or with ``use_checkpoint=True`` keeps only its inputs and reruns the forward
at the start of backward (the same gradients bit for bit, less memory held between forward and backward).  ``res_block_forward``
runs the same forward on a state dict.  Up / down-sampling, the timestep MLP and the assembled UNet with its training step are
the open part of row N3.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor, nn

from . import checkpoint, ops
from ._cabi import B200Error
from .attention import _bf, _check_cuda

MAX_CHANNELS = 2560  # GroupNorm kernels


def check_geometry(B: int, H: int, W: int, Cin: int, Cout: int) -> None:
    """Raise ``B200Error`` (with the reason) for shapes the convolution kernels do not take."""
    for name, c in (("Cin", Cin), ("Cout", Cout)):
        if c % 64 != 0 or c <= 0 or c > MAX_CHANNELS:
            raise B200Error(f"ResBlock: {name} = {c} must be a positive multiple of 64, at most {MAX_CHANNELS} (conv3x3 / GroupNorm kernels)")
    if W > 64 or 64 % W != 0:
        raise B200Error(f"ResBlock: the width W = {W} must divide 64 (conv3x3 weight gradient)")
    if (H * W) % 64 != 0:
        raise B200Error(f"ResBlock: H * W = {H * W} must be a multiple of 64 (conv3x3 weight gradient)")
    hb = min(H, 128 // W)
    if H % hb != 0 or 128 % (W * hb) != 0:
        raise B200Error(f"ResBlock: H = {H} must be a multiple of 128 / W (conv3x3 tiles of 128 pixels)")


# ------------------------------------------------------------------------------------------------------------------------------
# functional forward / backward on channels-last rows
# ------------------------------------------------------------------------------------------------------------------------------
def res_block_fwd(x: Tensor, time_net: Optional[Tensor], P: Sequence[Optional[Tensor]], eps: float) -> Tuple[Tensor, tuple]:
    """x: contiguous bf16 [B, H, W, Cin]; time_net: bf16 [B, tdim] or None (the reference then skips the add); P: the block's
    parameters (norm1 w / b, conv1 w / b, time_embedding w / b, norm2 w / b, conv2 w / b, shortcut w / b or None, None).
    Returns (out bf16 [B, H, W, Cout], the tensors backward needs)."""
    g1, be1, w1, b1, wt, bt, g2, be2, w2, b2, ws, bs = P
    B, H, W, Cin = x.shape
    Cout = w1.shape[0]
    HW, M = H * W, B * H * W
    g1f, be1f, g2f, be2f = (t.float().contiguous() for t in (g1, be1, g2, be2))  # the GroupNorm kernels read fp32 [C]
    y1, m1, r1 = ops.groupnorm_silu_fwd(x.view(B, HW, Cin), g1f, be1f, eps)
    w1p = ops.pack_conv3x3_weight(w1)
    ta = wtb = None
    if time_net is None:
        h = ops.conv3x3(y1.view(B, H, W, Cin), w1p, _bf(b1))
    else:
        ta = F.silu(time_net).contiguous()  # eager's F.silu on the bf16 tensor (fp32 maths, bf16 result)
        wtb = _bf(wt)
        t = ops.gemm(ta, wtb, bias=_bf(bt))  # [B, Cout]
        h = ops.conv3x3(y1.view(B, H, W, Cin), w1p, _bf(b1), epilogue=ops.EPI_BIAS_ADD_PER_IMAGE_BF16, aux=t)
    y2, m2, r2 = ops.groupnorm_silu_fwd(h.view(B, HW, Cout), g2f, be2f, eps)
    wsb = None
    if ws is None:
        inp = x
    else:  # 1x1 convolution on channels-last activations == a plain GEMM over the pixels
        wsb = _bf(ws.reshape(Cout, Cin))
        inp = ops.gemm(x.view(M, Cin), wsb, bias=_bf(bs))
    out = ops.conv3x3(y2.view(B, H, W, Cout), ops.pack_conv3x3_weight(w2), _bf(b2), epilogue=ops.EPI_BIAS_RESID_CLAMP_BF16, aux=inp)
    return out, (x, y1, h, y2, m1, r1, m2, r2, time_net, ta, g1f, be1f, g2f, be2f, w1, w2, wtb, wsb)


def res_block_bwd(saved: Sequence[Optional[Tensor]], dout: Tensor, pg: Optional[checkpoint.ParamGrads] = None
                  ) -> Tuple[Tensor, Optional[Tensor], List[Optional[Tensor]]]:
    """dout: contiguous bf16 [B, H, W, Cout].  Returns (dx bf16 [B, H, W, Cin], dtime bf16 [B, tdim] or None, the parameter
    gradients in ``res_block_fwd``'s P order: time-embedding ones None without a time input, shortcut ones None without one).
    ``pg``: where the parameter gradients go, numbered in P order (default: fresh tensors)."""
    x, y1, h, y2, m1, r1, m2, r2, time_net, ta, g1f, be1f, g2f, be2f, w1, w2, wtb, wsb = saved
    B, H, W, Cin = x.shape
    Cout = w1.shape[0]
    HW, M, dev = H * W, B * H * W, dout.device
    pg = pg or checkpoint.NO_GRADS
    f32 = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)  # noqa: E731
    d2 = dout.view(M, Cout)
    # conv2: weight, bias (= the shortcut's bias gradient too) and input gradients
    dw2 = pg.put(8, ops.conv3x3_weight_view(ops.conv3x3_wgrad(dout, y2.view(B, H, W, Cout)), Cout))
    shared_bias = wsb is not None and pg.dest(9) is not None  # one column sum feeds two arena views
    db2 = ops.colsum(d2, f32(Cout)) if shared_bias else ops.colsum(d2, pg.out(9, (Cout,), dev), **pg.mode)
    dy2 = ops.conv3x3(dout, ops.pack_conv3x3_weight_dgrad(w2))
    dh, dg2, dbe2 = ops.groupnorm_silu_bwd(h.view(B, HW, Cout), dy2.view(B, HW, Cout), g2f, be2f, m2, r2, **pg.norm_kw(6, 7))
    # one pass over dh: the time embedding's upstream gradient [B, Cout] and conv1's bias gradient
    if time_net is None:
        dt, db1 = None, ops.colsum(dh.view(M, Cout), pg.out(3, (Cout,), dev), **pg.mode)
    else:
        dt, db1 = ops.colsum_per_image(dh)
        db1 = pg.put(3, db1)
    dhv = dh.view(B, H, W, Cout)
    dw1 = pg.put(2, ops.conv3x3_weight_view(ops.conv3x3_wgrad(dhv, y1.view(B, H, W, Cin)), Cin))
    dy1 = ops.conv3x3(dhv, ops.pack_conv3x3_weight_dgrad(w1))
    dxg, dg1, dbe1 = ops.groupnorm_silu_bwd(x.view(B, HW, Cin), dy1.view(B, HW, Cin), g1f, be1f, m1, r1, **pg.norm_kw(0, 1))
    # the shortcut path, added to GroupNorm1's gradient in one bf16 add
    dws = dbs = None
    if wsb is None:
        dx = dxg.view(M, Cin) + d2
    else:
        dws = ops.wgrad(d2, x.view(M, Cin), pg.out(10, (Cout, Cin), dev), **pg.mode).view(Cout, Cin, 1, 1)
        if shared_bias:
            dbs, db2 = pg.put(11, db2), pg.put(9, db2)
        else:
            dbs = pg.put(11, db2.clone())
        dx = dxg.view(M, Cin) + ops.gemm(d2, wsb, b_mn_major=True)
    dtime = dwt = dbt = None
    if time_net is not None:  # [B, tdim] glue, the ops eager runs
        dwt = ops.wgrad(dt, ta, pg.out(4, tuple(wtb.shape), dev), **pg.mode)
        dbt = ops.colsum(dt, pg.out(5, (Cout,), dev), **pg.mode)
        dtime = torch.ops.aten.silu_backward(ops.gemm(dt, wtb, b_mn_major=True), time_net)
    return dx.view(B, H, W, Cin), dtime, [dg1, dbe1, dw1, db1, dwt, dbt, dg2, dbe2, dw2, db2, dws, dbs]


def res_block_forward(sd: Dict[str, Tensor], prefix: str, net: Tensor, time_net: Tensor) -> Tensor:
    """``net``: bf16 [B, H, W, Cin] channels-last; ``time_net``: bf16 [B, time_dim]; ``sd``: the reference's parameters of the
    block under ``prefix`` (fp32, NCHW conv weights).  Returns bf16 [B, H, W, Cout]."""
    if not net.is_cuda or net.dtype != torch.bfloat16 or net.dim() != 4:
        raise B200Error("res_block_forward: bf16 CUDA activations [B, H, W, C] (there is no CPU fallback)")
    p = prefix
    names = ("norm1.weight", "norm1.bias", "conv1.weight", "conv1.bias", "time_embedding.weight", "time_embedding.bias",
             "norm2.weight", "norm2.bias", "conv2.weight", "conv2.bias", "shortcut.weight", "shortcut.bias")
    out, _ = res_block_fwd(net.contiguous(), time_net, [sd.get(p + n) for n in names], 1e-5)
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# module
# ------------------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class _ResBlockOp:
    """ResidualBlockWithTimeEmbeddingB200 as a ``checkpoint.OpFn`` op on (net [B, Cin, H, W], time_net or None, *_params()):
    the NHWC kernels on net's channels-last view, the output [B, Cout, H, W] and dx with channels-last strides."""
    eps: float

    def forward(self, net: Tensor, time_net: Optional[Tensor], *params: Optional[Tensor]) -> Tuple[Tensor, tuple]:
        xt = net.permute(0, 2, 3, 1).contiguous()  # a view when net is channels-last
        out, saved = res_block_fwd(xt, time_net, params, self.eps)
        return out.permute(0, 3, 1, 2), saved

    def backward(self, saved: tuple, dout: Tensor, pg: Optional[checkpoint.ParamGrads] = None) -> tuple:
        pg = pg or checkpoint.NO_GRADS
        dx, dtime, grads = res_block_bwd(saved, dout.permute(0, 2, 3, 1).to(torch.bfloat16).contiguous(), pg.sub(2))
        return (dx.permute(0, 3, 1, 2), dtime, *grads)


class ResidualBlockWithTimeEmbeddingB200(nn.Module):
    """Drop-in for cflearn's ``ResidualBlockWithTimeEmbedding`` on the native kernels (bf16 activations, fp32 parameters; CUDA
    only).  ``forward(net, time_net=None)`` takes bf16 [B, Cin, H, W] (channels-last preferred: used without a copy) and a bf16
    [B, time_embedding_channels] time embedding, and returns bf16 [B, Cout, H, W] with channels-last strides.
    ``use_checkpoint=True`` keeps only the inputs for backward and recomputes the activations there (the same gradients)."""

    def __init__(self, in_channels: int, out_channels: Optional[int] = None, *, signal_dim: int = 2, dropout: float = 0.0,
                 norm_eps: float = 1.0e-6, use_conv_shortcut: bool = False, integrate_upsample: bool = False,
                 integrate_downsample: bool = False, time_embedding_channels: int = 512, use_scale_shift_norm: bool = False,
                 use_checkpoint: bool = False) -> None:
        super().__init__()
        out_channels = out_channels or in_channels
        if signal_dim != 2:
            raise NotImplementedError("ResidualBlockWithTimeEmbeddingB200: only 2-D signals are supported")
        if dropout > 0.0:
            raise NotImplementedError("ResidualBlockWithTimeEmbeddingB200: dropout > 0 is not supported")
        if use_scale_shift_norm:
            raise NotImplementedError("ResidualBlockWithTimeEmbeddingB200: use_scale_shift_norm is not supported")
        if integrate_upsample or integrate_downsample:
            raise NotImplementedError("ResidualBlockWithTimeEmbeddingB200: integrated up / down-sampling is not supported "
                                      "(SD-v1.5 resamples with separate convolutions)")
        if use_conv_shortcut and in_channels != out_channels:
            raise NotImplementedError("ResidualBlockWithTimeEmbeddingB200: the 3x3 convolution shortcut is not supported")
        if time_embedding_channels <= 0:
            raise NotImplementedError("ResidualBlockWithTimeEmbeddingB200: a block without a time embedding is not supported")
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.norm_eps = norm_eps
        self.use_checkpoint = use_checkpoint  # keep only the inputs and recompute the activations in backward
        # registration order of the reference (state_dict order): norm1, conv1, time_embedding, norm2, conv2, shortcut
        self.norm1 = nn.GroupNorm(32, in_channels, eps=norm_eps)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, 1, 1)
        self.time_embedding = nn.Linear(time_embedding_channels, out_channels)
        self.norm2 = nn.GroupNorm(32, out_channels, eps=norm_eps)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, 1, 1)
        with torch.no_grad():  # zero_module(conv2), as the reference
            self.conv2.weight.zero_()
            self.conv2.bias.zero_()
        self.shortcut = nn.Conv2d(in_channels, out_channels, 1, 1, 0) if in_channels != out_channels else None

    def _params(self) -> List[Optional[Tensor]]:
        s = self.shortcut
        return [self.norm1.weight, self.norm1.bias, self.conv1.weight, self.conv1.bias, self.time_embedding.weight,
                self.time_embedding.bias, self.norm2.weight, self.norm2.bias, self.conv2.weight, self.conv2.bias,
                None if s is None else s.weight, None if s is None else s.bias]

    def forward(self, net: Tensor, time_net: Optional[Tensor] = None) -> Tensor:
        what = "ResidualBlockWithTimeEmbeddingB200"
        if net.dim() != 4 or net.shape[1] != self.in_channels:
            raise B200Error(f"{what}: net must be [B, {self.in_channels}, H, W]")
        B, _, H, W = net.shape
        check_geometry(B, H, W, self.in_channels, self.out_channels)
        if time_net is not None:
            tdim = self.time_embedding.in_features
            if tuple(time_net.shape) != (B, tdim) or tdim % 8 != 0:
                raise B200Error(f"{what}: time_net must be [B, {tdim}] with a width that is a multiple of 8")
        _check_cuda(what, net, time_net)
        if any(t is not None and t.dtype != torch.bfloat16 for t in (net, time_net)):
            raise B200Error(f"{what}: net and time_net must be bf16 (the UNet's activations under bf16 autocast)")
        return checkpoint.OpFn.apply(_ResBlockOp(self.norm_eps), self.use_checkpoint, net, time_net, *self._params())


# ------------------------------------------------------------------------------------------------------------------------------
# resampling: ResDownsample / ResUpsample with use_conv (cflearn/modules/core/convs/residual.py:86-151)
# ------------------------------------------------------------------------------------------------------------------------------
def _tiles(what: str, h: int, w: int, wgrad: bool) -> None:
    """The tile rules of the implicit-GEMM convolutions on an h x w grid (``wgrad``: also those of the weight gradient)."""
    if w > 128 or 128 % w != 0 or h % min(h, 128 // w) != 0:
        raise B200Error(f"{what}: a {h} x {w} grid is not tiled by 128-pixel tiles of whole rows (the width must divide 128, the "
                        "height be a multiple of 128 / width)")
    if wgrad and (w > 64 or 64 % w != 0 or (h * w) % 64 != 0):
        raise B200Error(f"{what}: the weight gradient's {h} x {w} grid needs a width that divides 64 and h * w a multiple of 64")


def check_resample_geometry(what: str, up: bool, H: int, W: int, Cin: int, Cout: int) -> None:
    """Raise ``B200Error`` (with the reason) for shapes the resampling kernels do not take; H x W is the input's size."""
    for name, c in (("Cin", Cin), ("Cout", Cout)):
        if c <= 0 or c % 64 != 0:
            raise B200Error(f"{what}: {name} = {c} must be a positive multiple of 64 (the convolutions reduce over 64-channel blocks)")
    if up:  # fused forward on the H x W grid; backward: stride-1 input and weight gradients at 2H x 2W
        _tiles(what, H, W, False)
        _tiles(what, 2 * H, 2 * W, True)
    else:
        if H % 2 or W % 2:
            raise B200Error(f"{what}: H = {H} and W = {W} must be even")
        _tiles(what, H // 2, W // 2, True)


def _bias_rows(bias: Tensor, B: int) -> Tensor:
    """The bias as a per-image table [B, Cout] for the per-image epilogue with no bias of its own: bf16(bf16(conv) + bias), the
    two roundings of eager's biased convolution on CUDA (DESIGN.md section 2)."""
    return _bf(bias).expand(B, -1).contiguous()


def _nhwc(t: Tensor) -> Tensor:
    return t.permute(0, 2, 3, 1).to(torch.bfloat16).contiguous()  # a view when t is channels-last bf16


@dataclass(frozen=True)
class _DownsampleOp:
    """ResDownsampleB200 as a ``checkpoint.OpFn`` op on (net [B, Cin, H, W], weight, bias); keeps only its input (and the
    parameters) for backward."""

    def forward(self, net: Tensor, weight: Tensor, bias: Tensor) -> Tuple[Tensor, tuple]:
        out = ops.conv3x3_s2(_nhwc(net), ops.pack_conv3x3_weight(weight), epilogue=ops.EPI_BIAS_ADD_PER_IMAGE_BF16,
                             aux=_bias_rows(bias, net.shape[0]))
        return out.permute(0, 3, 1, 2), (net, weight)

    def backward(self, saved: tuple, dout: Tensor, pg: Optional[checkpoint.ParamGrads] = None) -> tuple:
        pg = pg or checkpoint.NO_GRADS
        net, weight = saved
        Cout, Cin = weight.shape[:2]
        d = _nhwc(dout)
        dw = pg.put(1, ops.conv3x3_weight_view(ops.conv3x3_s2_wgrad(d, _nhwc(net)), Cin))
        db = ops.colsum(d.view(-1, Cout), pg.out(2, (Cout,), d.device), **pg.mode)
        dx = ops.conv3x3_s2_dgrad(d, ops.pack_conv3x3_weight_s2_dgrad(weight))
        return dx.permute(0, 3, 1, 2), dw, db


@dataclass(frozen=True)
class _UpsampleOp:
    """ResUpsampleB200 as a ``checkpoint.OpFn`` op on (net [B, Cin, H, W], weight, bias); keeps only its low-resolution input (and
    the parameters) for backward.  Backward holds two transient 2H x 2W tensors: the upsampled input for the weight gradient and
    the input gradient before its 2x2 sum."""

    def forward(self, net: Tensor, weight: Tensor, bias: Tensor) -> Tuple[Tensor, tuple]:
        out = ops.conv3x3_up2(_nhwc(net), ops.pack_conv3x3_weight(weight), epilogue=ops.EPI_BIAS_ADD_PER_IMAGE_BF16,
                              aux=_bias_rows(bias, net.shape[0]))
        return out.permute(0, 3, 1, 2), (net, weight)

    def backward(self, saved: tuple, dout: Tensor, pg: Optional[checkpoint.ParamGrads] = None) -> tuple:
        pg = pg or checkpoint.NO_GRADS
        net, weight = saved
        Cout, Cin = weight.shape[:2]
        d = _nhwc(dout)
        dw = pg.put(1, ops.conv3x3_weight_view(ops.conv3x3_wgrad(d, ops.upsample_nearest2x(_nhwc(net))), Cin))
        db = ops.colsum(d.view(-1, Cout), pg.out(2, (Cout,), d.device), **pg.mode)
        dx = ops.sum2x2(ops.conv3x3(d, ops.pack_conv3x3_weight_dgrad(weight)))
        return dx.permute(0, 3, 1, 2), dw, db


def _resample_options(what: str, use_conv: bool, signal_dim: int, padding: int) -> None:
    if not use_conv:
        raise NotImplementedError(f"{what}: use_conv=False (average pooling / a bare interpolation) is not supported")
    if signal_dim != 2:
        raise NotImplementedError(f"{what}: signal_dim={signal_dim} is not supported (2-D signals only)")
    if padding != 1:
        raise NotImplementedError(f"{what}: padding={padding} is not supported (padding=1 only)")


class _Resample(nn.Module):
    """The forward of both resampling modules: bf16 [B, Cin, H, W] (either memory format; CUDA only) -> bf16 [B, Cout, H', W']
    with channels-last strides, through one ``checkpoint.OpFn`` node."""

    UP = False

    def _run(self, conv: nn.Conv2d, net: Tensor) -> Tensor:
        what = type(self).__name__
        if net.dim() != 4 or net.shape[1] != conv.in_channels:
            raise B200Error(f"{what}: net must be [B, {conv.in_channels}, H, W]")
        check_resample_geometry(what, self.UP, net.shape[2], net.shape[3], conv.in_channels, conv.out_channels)
        _check_cuda(what, net)
        if net.dtype != torch.bfloat16:
            raise B200Error(f"{what}: net must be bf16 (the UNet's activations under bf16 autocast)")
        op = _UpsampleOp() if self.UP else _DownsampleOp()
        return checkpoint.OpFn.apply(op, False, net, conv.weight, conv.bias)


class ResDownsampleB200(_Resample):
    """Drop-in for cflearn's ``ResDownsample`` with ``use_conv=True`` on the native kernels: a 3x3 convolution with stride 2 and
    padding 1 (``net`` is a Conv2d, as in the reference's state dict)."""

    def __init__(self, in_channels: int, use_conv: bool, *, signal_dim: int = 2, out_channels: Optional[int] = None,
                 padding: int = 1) -> None:
        super().__init__()
        _resample_options("ResDownsampleB200", use_conv, signal_dim, padding)
        self.net = nn.Conv2d(in_channels, out_channels or in_channels, 3, stride=2, padding=padding)

    def forward(self, net: Tensor) -> Tensor:
        return self._run(self.net, net)


class ResUpsampleB200(_Resample):
    """Drop-in for cflearn's ``ResUpsample`` with ``use_conv=True`` on the native kernels: nearest 2x upsampling and a 3x3 /
    padding 1 convolution (``conv``), fused so that the upsampled image is never written in the forward."""

    UP = True

    def __init__(self, in_channels: int, use_conv: bool, *, signal_dim: int = 2, out_channels: Optional[int] = None,
                 padding: int = 1) -> None:
        super().__init__()
        _resample_options("ResUpsampleB200", use_conv, signal_dim, padding)
        self.conv = nn.Conv2d(in_channels, out_channels or in_channels, 3, padding=padding)

    def forward(self, net: Tensor) -> Tensor:
        return self._run(self.conv, net)
