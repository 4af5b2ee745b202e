"""The SD-v1.5 UNet's ``SpatialTransformer`` and ``SpatialTransformerBlock`` (cflearn/modules/core/mixed_stacks/api.py:766-893)
on the native kernels, forward and backward.

    GroupNorm(32, eps 1e-6) -> 1x1 conv (to_latent) -> tokens [B, HW, C]            b200_groupnorm_silu_fwd(silu=0), GEMM
      per block:  x = attn1(LN1(x)) + x                                                b200_layernorm_bf16_fwd, attention_forward
                  x = attn2(LN2(x), context) + x                                       (out_linear with the bf16 residual epilogue)
                  x = ff(LN3(x)) + x,  ff = Linear(C, F) o (h * gelu(gate)) o Linear(C, 2F)   GEGLU epilogue, FF2 + bf16 residual
    -> 1x1 conv (from_latent) + input                                                  GEMM with the bf16 residual epilogue

Semantics are eager's under bf16 autocast (oracle/unet_oracle.py::transformer_block / ::spatial_transformer): the residual
stream is bf16, LayerNorm / GroupNorm run in fp32 and round once, every Linear / 1x1 conv output is bf16 and each residual add
is a bf16 add.  Rounding points that differ from eager: eager's 1x1 convolution rounds its product to bf16 before adding the
bias in a second bf16 op, ours adds the bias in fp32 and rounds once; in attention, see ``attention.py``.  In backward, GEGLU's
three elementwise gradients are eager's roundings (dh = bf16(da g), dg = bf16(da h), dgate = bf16(gelu'(gate) dg)), and each
LayerNorm gradient is rounded to bf16 before the bf16 add of the residual branch's gradient, as eager does.

Activations live channels-last: a ``torch.channels_last`` input is used with no copy (a contiguous NCHW one costs one permute),
and the output is [B, C, H, W] with channels-last strides.  A block is one ``checkpoint.OpFn`` node that keeps the activations
its backward reads, or with ``use_checkpoint=True`` only its inputs, rerunning its forward in backward: the same results bit for
bit, one block's activations held instead of every block's.  ``SpatialTransformerB200`` is a chain of such nodes: GroupNorm and
to_latent, each block as it runs standalone (with its own ``use_checkpoint``), then from_latent with the residual.  The outer
two keep their tensors either way, as the reference checkpoints the blocks alone.  Dropout > 0, hooks (ToMe / style
reference, inference features), ``use_linear=True`` and activations other than GEGLU are refused.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch
from torch import Tensor, nn

from . import checkpoint, ops
from ._cabi import B200Error
from .attention import CrossAttentionB200, _bf, _check_cuda, _Linear, _rows, attention_backward, attention_forward

LN_EPS = 1e-5  # nn.LayerNorm's default (api.py:792-794)
GN_EPS = 1e-6  # SpatialTransformer.norm (api.py:838)
BLOCK_PARAMS = 20  # tensors per block handed to _block_forward, in _block_params order


# ------------------------------------------------------------------------------------------------------------------------------
# one block: functional forward / backward on [M, C] bf16 token rows
# ------------------------------------------------------------------------------------------------------------------------------
def _block_forward(x0: Tensor, c: Optional[Tensor], P: Sequence[Tensor], B: int, heads: int) -> Tuple[Tensor, tuple]:
    """Returns (x3 bf16 [M, C], a flat tuple of 37 tensors / Nones for save_for_backward: 17 of its own + 10 per attention)."""
    a1, a2 = P[0:5], P[5:10]
    w1, b1, w2, b2 = P[10:14]
    g1, be1, g2, be2, g3, be3 = (t.float().contiguous() for t in P[14:BLOCK_PARAMS])  # the kernels read fp32 [C]
    y1, m1, r1 = ops.layernorm_bf16_fwd(x0, g1, be1, LN_EPS)
    x1, s1 = attention_forward(y1, None, *a1, B, heads, resid=x0)
    y2, m2, r2 = ops.layernorm_bf16_fwd(x1, g2, be2, LN_EPS)
    x2, s2 = attention_forward(y2, c, *a2, B, heads, resid=x1)
    y3, m3, r3 = ops.layernorm_bf16_fwd(x2, g3, be3, LN_EPS)
    w1b, w2b = _bf(w1), _bf(w2)
    hg, act = ops.geglu(y3, w1b, _bf(b1))
    x3 = ops.gemm(act, w2b, bias=_bf(b2), epilogue=ops.EPI_BIAS_RESID_BF16, aux=x2)
    return x3, (x0, x1, x2, m1, r1, m2, r2, m3, r3, y3, hg, act, w1b, w2b, g1, g2, g3, *s1, *s2)


def _block_backward(saved: tuple, dx3: Tensor, B: int, heads: int, pg: Optional[checkpoint.ParamGrads] = None
                    ) -> Tuple[Tensor, Optional[Tensor], List[Tensor]]:
    """dx3: bf16 [M, C], the gradient of the block's output.  Returns (dx0 bf16, dcontext bf16 or None, the BLOCK_PARAMS
    parameter gradients in _block_params order).  ``pg``: where they go, numbered in that order (default: fresh tensors)."""
    x0, x1, x2, m1, r1, m2, r2, m3, r3, y3, hg, act, w1b, w2b, g1, g2, g3 = saved[:17]
    s1, s2 = saved[17:27], saved[27:37]
    dev = dx3.device
    pg = pg or checkpoint.NO_GRADS
    # feed-forward: FF2's weight / bias gradients, its dgrad through GEGLU's backward (one epilogue), then FF1
    dw2 = ops.wgrad(dx3, act, pg.out(12, tuple(w2b.shape), dev), **pg.mode)
    db2 = ops.colsum(dx3, pg.out(13, (w2b.shape[0],), dev), **pg.mode)
    dhg = ops.gemm(dx3, w2b, b_mn_major=True, epilogue=ops.EPI_DGEGLU_BF16, aux=hg)
    dw1 = ops.wgrad(dhg, y3, pg.out(10, tuple(w1b.shape), dev), **pg.mode)
    db1 = ops.colsum(dhg, pg.out(11, (w1b.shape[0],), dev), **pg.mode)
    dy3 = ops.gemm(dhg, w1b, b_mn_major=True)
    dx2, dg3, dbe3 = ops.layernorm_bf16_bwd(dy3, x2, g3, m3, r3, dres=dx3, **pg.norm_kw(18, 19))
    dy2, dc, *ga2 = attention_backward(s2, dx2, B, heads, pg.sub(5))
    dx1, dg2, dbe2 = ops.layernorm_bf16_bwd(dy2, x1, g2, m2, r2, dres=dx2, **pg.norm_kw(16, 17))
    dy1, _, *ga1 = attention_backward(s1, dx1, B, heads, pg)
    dx0, dg1, dbe1 = ops.layernorm_bf16_bwd(dy1, x0, g1, m1, r1, dres=dx1, **pg.norm_kw(14, 15))
    return dx0, dc, [*ga1, *ga2, dw1, db1, dw2, db2, dg1, dbe1, dg2, dbe2, dg3, dbe3]


@dataclass(frozen=True)
class _BlockOp:
    """SpatialTransformerBlockB200 as a ``checkpoint.OpFn`` op on (net [B, T, C], context [B, Tk, Dc] or None, the
    BLOCK_PARAMS parameters in _block_params order)."""
    B: int
    heads: int

    def forward(self, net: Tensor, context: Optional[Tensor], *params: Tensor) -> Tuple[Tensor, tuple]:
        x3, saved = _block_forward(_rows(net), _rows(context), params, self.B, self.heads)
        return x3.view(net.shape), saved

    def backward(self, saved: tuple, dout: Tensor, pg: Optional[checkpoint.ParamGrads] = None) -> tuple:
        pg = pg or checkpoint.NO_GRADS
        dx, dc, grads = _block_backward(saved, _rows(dout), self.B, self.heads, pg.sub(2))
        return (dx, dc, *grads)


class _LatentIn:
    """SpatialTransformerB200's GroupNorm and to_latent as an op on (xt [B, H, W, C] channels-last, norm w / b, to_latent
    w / b): the tokens [B, H*W, L]."""

    def forward(self, xt: Tensor, gn_w: Tensor, gn_b: Tensor, w_in: Tensor, b_in: Tensor) -> Tuple[Tensor, tuple]:
        B, H, W, C = xt.shape
        L = w_in.shape[0]
        gn_w32, gn_b32 = gn_w.float().contiguous(), gn_b.float().contiguous()
        yn, gm, gr = ops.groupnorm_silu_fwd(xt.view(B, H * W, C), gn_w32, gn_b32, GN_EPS, silu=False)
        w_in_b = _bf(w_in.reshape(L, C))
        t = ops.gemm(yn.view(B * H * W, C), w_in_b, bias=_bf(b_in))
        return t.view(B, H * W, L), (xt, yn, gm, gr, gn_w32, gn_b32, w_in_b)

    def backward(self, saved: tuple, dout: Tensor, pg: Optional[checkpoint.ParamGrads] = None) -> tuple:
        pg = pg or checkpoint.NO_GRADS
        xt, yn, gm, gr, gn_w32, gn_b32, w_in_b = saved
        B, H, W, C = xt.shape
        L, M, dev = w_in_b.shape[0], B * H * W, dout.device
        dtl = _rows(dout)
        dw_in = ops.wgrad(dtl, yn.view(M, C), pg.out(3, (L, C), dev), **pg.mode)
        db_in = ops.colsum(dtl, pg.out(4, (L,), dev), **pg.mode)
        dyn = ops.gemm(dtl, w_in_b, b_mn_major=True)
        dxg, dgn_w, dgn_b = ops.groupnorm_silu_bwd(xt.view(B, H * W, C), dyn.view(B, H * W, C), gn_w32, gn_b32, gm, gr, silu=False,
                                                   **pg.norm_kw(1, 2))
        return dxg, dgn_w, dgn_b, dw_in, db_in


class _LatentOut:
    """SpatialTransformerB200's from_latent and the residual as an op on (t [B, H*W, L], xt [B, H, W, C], from_latent w / b):
    bf16(bf16(from_latent(t)) + xt) in the GEMM's epilogue, [B, C, H, W] with channels-last strides."""

    def forward(self, t: Tensor, xt: Tensor, w_out: Tensor, b_out: Tensor) -> Tuple[Tensor, tuple]:
        B, H, W, C = xt.shape
        w_out_b = _bf(w_out.reshape(C, t.shape[-1]))
        out = ops.gemm(_rows(t), w_out_b, bias=_bf(b_out), epilogue=ops.EPI_BIAS_RESID_BF16, aux=_rows(xt))
        return out.view(B, H, W, C).permute(0, 3, 1, 2), (t, w_out_b)

    def backward(self, saved: tuple, dout: Tensor, pg: Optional[checkpoint.ParamGrads] = None) -> tuple:
        pg = pg or checkpoint.NO_GRADS
        t, w_out_b = saved
        C, L = w_out_b.shape
        dev = dout.device
        dt = dout.permute(0, 2, 3, 1).to(torch.bfloat16).contiguous().view(-1, C)
        dw_out = ops.wgrad(dt, _rows(t), pg.out(2, (C, L), dev), **pg.mode)
        db_out = ops.colsum(dt, pg.out(3, (C,), dev), **pg.mode)
        return ops.gemm(dt, w_out_b, b_mn_major=True), dt, dw_out, db_out  # the residual's gradient is dt itself


# ------------------------------------------------------------------------------------------------------------------------------
# modules
# ------------------------------------------------------------------------------------------------------------------------------
class _GEGLUParams(nn.Module):
    """GEGLU's parameters (activations.py:157-164): ``net`` = Linear(in, 2 * out), h rows first, then the gate rows."""

    def __init__(self, in_dim: int, out_dim: int) -> None:
        super().__init__()
        self.net = _Linear(in_dim, 2 * out_dim, bias=True)


class _CustomLinearParams(nn.Module):
    """HijackCustomLinear's parameter names: ``linear.weight`` / ``linear.bias``."""

    def __init__(self, in_dim: int, out_dim: int) -> None:
        super().__init__()
        self.linear = _Linear(in_dim, out_dim, bias=True)


class _FeedForwardParams(nn.Module):
    """FeedForward(activation="geglu", add_last_dropout=False) (channel_mixers.py:15-36): net = [GEGLU, Dropout, Linear]."""

    def __init__(self, dim: int, latent_dim: int) -> None:
        super().__init__()
        self.net = nn.Sequential(_GEGLUParams(dim, latent_dim), nn.Dropout(0.0), _CustomLinearParams(latent_dim, dim))


class _Conv1x1Params(nn.Module):
    """A 1x1 Conv2d's parameters (HijackConv2d(in, out, 1, 1, 0)): weight [out, in, 1, 1], bias [out]."""

    def __init__(self, in_dim: int, out_dim: int, zero: bool = False) -> None:
        super().__init__()
        ref = nn.Conv2d(in_dim, out_dim, 1, 1, 0)
        self.weight = nn.Parameter(ref.weight.detach().clone())
        self.bias = nn.Parameter(ref.bias.detach().clone())
        if zero:  # zero_module (the reference's from_latent)
            with torch.no_grad():
                self.weight.zero_()
                self.bias.zero_()


class SpatialTransformerBlockB200(nn.Module):
    """Drop-in for cflearn's ``SpatialTransformerBlock`` on the native kernels (bf16 residual stream, fp32 parameters; CUDA
    only).  ``forward(net, context)`` takes bf16 tokens [B, T, query_dim] and a context [B, Tk, context_dim] (or None)."""

    def __init__(self, query_dim: int, num_heads: int, head_dim: int, *, dropout: float = 0.0, context_dim: Optional[int] = None,
                 feedforward_multiplier: float = 4.0, feedforward_activation: str = "geglu", use_checkpoint: bool = False,
                 hooks_kwargs: Optional[Dict[str, Any]] = None) -> None:
        super().__init__()
        if dropout > 0.0:
            raise NotImplementedError("SpatialTransformerBlockB200: dropout > 0 is not supported")
        if hooks_kwargs is not None:
            raise NotImplementedError("SpatialTransformerBlockB200: hooks (ToMe / style reference) are inference features, not supported")
        if feedforward_activation != "geglu":
            raise NotImplementedError("SpatialTransformerBlockB200: only the GEGLU feed-forward is supported")
        latent_dim = round(query_dim * feedforward_multiplier)
        if latent_dim % 8 != 0:
            raise NotImplementedError("SpatialTransformerBlockB200: the feed-forward width must be a multiple of 8")
        self.num_heads = num_heads
        self.use_checkpoint = use_checkpoint  # keep only the inputs and recompute the activations in backward
        # registration order of the reference: attn1, ff, attn2, norm1..3 (state_dict order)
        self.attn1 = CrossAttentionB200(query_dim=query_dim, num_heads=num_heads, head_dim=head_dim)
        self.ff = _FeedForwardParams(query_dim, latent_dim)
        self.attn2 = CrossAttentionB200(query_dim=query_dim, context_dim=context_dim, num_heads=num_heads, head_dim=head_dim)
        self.norm1 = nn.LayerNorm(query_dim)
        self.norm2 = nn.LayerNorm(query_dim)
        self.norm3 = nn.LayerNorm(query_dim)

    def _block_params(self) -> List[Tensor]:
        out: List[Tensor] = []
        for a in (self.attn1, self.attn2):
            lin = a.out_linear[0]
            out += [a.to_q.weight, a.to_k.weight, a.to_v.weight, lin.weight, lin.bias]
        g, f2 = self.ff.net[0].net, self.ff.net[2].linear
        out += [g.weight, g.bias, f2.weight, f2.bias]
        for n in (self.norm1, self.norm2, self.norm3):
            out += [n.weight, n.bias]
        return out

    def forward(self, net: Tensor, context: Optional[Tensor] = None) -> Tensor:
        _check_cuda("SpatialTransformerBlockB200", net, context)
        if net.dtype != torch.bfloat16:
            raise B200Error("SpatialTransformerBlockB200: the input must be bf16 (the residual stream of the UNet under bf16 autocast)")
        return checkpoint.OpFn.apply(_BlockOp(net.shape[0], self.num_heads), self.use_checkpoint, net, context, *self._block_params())


class SpatialTransformerB200(nn.Module):
    """Drop-in for cflearn's ``SpatialTransformer`` (conv form) on the native kernels.  ``forward(net, context)`` takes bf16
    [B, C, H, W] (channels-last preferred) and returns bf16 [B, C, H, W] with channels-last strides."""

    def __init__(self, in_channels: int, num_heads: int, head_dim: int, *, num_layers: int = 1, dropout: float = 0.0,
                 context_dim: Optional[int] = None, use_linear: bool = False, use_checkpoint: bool = False,
                 hooks_kwargs: Optional[Dict[str, Any]] = None) -> None:
        super().__init__()
        if use_linear:
            raise NotImplementedError("SpatialTransformerB200: use_linear=True is not supported (SD-v1.5 uses the 1x1 convolutions)")
        if hooks_kwargs is not None:
            raise NotImplementedError("SpatialTransformerB200: hooks (ToMe / style reference) are inference features, not supported")
        latent = num_heads * head_dim
        if latent != in_channels:
            # the reference reshapes the latent tokens with in_channels (api.py:874-879), so only this case runs there either
            raise NotImplementedError("SpatialTransformerB200: num_heads * head_dim must equal in_channels")
        self.num_heads = num_heads
        self.norm = nn.GroupNorm(32, in_channels, GN_EPS, affine=True)
        self.to_latent = _Conv1x1Params(in_channels, latent)
        self.blocks = nn.ModuleList([SpatialTransformerBlockB200(latent, num_heads, head_dim, dropout=dropout, context_dim=context_dim,
                                                                 use_checkpoint=use_checkpoint) for _ in range(num_layers)])
        self.from_latent = _Conv1x1Params(latent, in_channels, zero=True)

    def forward(self, net: Tensor, context: Optional[Tensor] = None) -> Tensor:
        _check_cuda("SpatialTransformerB200", net, context)
        if net.dtype != torch.bfloat16:
            raise B200Error("SpatialTransformerB200: the input must be bf16 (the residual stream of the UNet under bf16 autocast)")
        # a view when net is channels-last; autograd adds xt's two gradients (GroupNorm path, residual) and the blocks' context ones
        xt = net.permute(0, 2, 3, 1).contiguous()
        t = checkpoint.OpFn.apply(_LatentIn(), False, xt, self.norm.weight, self.norm.bias, self.to_latent.weight, self.to_latent.bias)
        for block in self.blocks:
            t = block(t, context)
        return checkpoint.OpFn.apply(_LatentOut(), False, t, xt, self.from_latent.weight, self.from_latent.bias)
