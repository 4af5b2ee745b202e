"""The SD-v1.5 UNet's ``CrossAttention`` (cflearn/modules/core/attentions.py:498-569) on the native kernels.

``CrossAttentionB200`` is a drop-in for the reference module: same constructor keywords, the same fp32 parameters under the
same ``state_dict`` keys (``to_q.weight``, ``to_k.weight``, ``to_v.weight``, ``out_linear.0.weight``, ``out_linear.0.bias``).
Its forward and backward are one ``checkpoint.OpFn`` node over ``attention_forward`` / ``attention_backward``, which the
SpatialTransformerBlock (``spatial_transformer.py``) calls as well; every product is the wgmma GEMM (``ops.gemm`` / ``ops.wgrad``) or the
streamed attention (``ops.cross_attention_fwd/_bwd``), which reads q / k / v as column slices of the projection outputs:

    self-attention (context None):  qkv = x [Wq; Wk; Wv]^T  (one GEMM, N = 3L)   dx = dqkv [Wq; Wk; Wv]  (one GEMM, K = 3L)
    cross-attention:                q = x Wq^T, kv = context [Wk; Wv]^T          dx = dq Wq, dcontext = dkv [Wk; Wv]
    then attention (scale Dh^-0.5), out_linear with bias; weight gradients by split-K wgrad, the bias gradient by a column sum.

Semantics are eager's under bf16 autocast: each input is cast to bf16 once, q / k / v, the attention output and the module
output are bf16, weight and bias gradients are rounded to bf16 like eager's, and input gradients come back in the input's
dtype.  Rounding points that differ from eager: in self-attention the three contributions to the input gradient are summed in
fp32 inside the packed dgrad GEMM and rounded once, where eager rounds each to bf16 and adds them (in bf16 for a bf16 input);
likewise the k and v contributions to the context gradient.  Dropout > 0 and attention masks are refused.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import torch
from torch import Tensor, nn

from . import checkpoint, ops
from ._cabi import B200Error


def _bf(t: Tensor) -> Tensor:
    return t.to(torch.bfloat16).contiguous()


def _rows(t: Optional[Tensor]) -> Optional[Tensor]:
    """[..., D] -> contiguous bf16 [rows, D] (a view of a contiguous bf16 tensor); None stays None."""
    return None if t is None else _bf(t.reshape(-1, t.shape[-1]))


def _check_cuda(what: str, *tensors: Optional[Tensor]) -> None:
    """Refuses CPU tensors before any launch: the native modules have no CPU fallback."""
    if any(t is not None and not t.is_cuda for t in tensors):
        raise B200Error(f"{what} needs CUDA tensors (there is no CPU fallback)")


def attention_forward(x: Tensor, c: Optional[Tensor], wq: Tensor, wk: Tensor, wv: Tensor, wo: Tensor, bo: Tensor, B: int, heads: int,
                      resid: Optional[Tensor] = None) -> Tuple[Tensor, tuple]:
    """Projections, attention and out_linear of one CrossAttention.  x: bf16 [B*Tq, Dq]; c: bf16 [B*Tk, Dc], or None for
    self-attention; fp32 weights.  ``resid`` (bf16 [B*Tq, Dq]): the module output is added to it in out_linear's epilogue,
    y = bf16(bf16(out_linear) + resid) -- the bf16 residual add that follows every attention of a SpatialTransformerBlock.
    Returns (y bf16 [B*Tq, Dq], what ``attention_backward`` needs: a flat tuple of tensors and Nones, for save_for_backward)."""
    L = wq.shape[0]
    if c is None:
        w_in = _bf(torch.cat([wq, wk, wv], 0))
        qkv = ops.gemm(x, w_in)
        q, k, v = qkv[:, :L], qkv[:, L:2 * L], qkv[:, 2 * L:]
        w_kv = None
    else:
        w_in, w_kv = _bf(wq), _bf(torch.cat([wk, wv], 0))
        q = ops.gemm(x, w_in)
        kv = ops.gemm(c, w_kv)
        k, v = kv[:, :L], kv[:, L:]
    o, lse = ops.cross_attention_fwd(q, k, v, B, heads)
    w_o = _bf(wo)
    if resid is None:
        y = ops.gemm(o, w_o, bias=_bf(bo))
    else:
        y = ops.gemm(o, w_o, bias=_bf(bo), epilogue=ops.EPI_BIAS_RESID_BF16, aux=resid)
    return y, (x, c, q, k, v, o, lse, w_in, w_kv, w_o)


def attention_backward(saved: tuple, dy: Tensor, B: int, heads: int, pg: Optional[checkpoint.ParamGrads] = None):
    """Backward of ``attention_forward`` for dy bf16 [B*Tq, Dq] (the gradient of y; with ``resid`` the residual's own
    gradient is dy as well, which the caller adds).  Returns (dx bf16, dc bf16 or None, dwq, dwk, dwv, dwo, dbo), the weight
    and bias gradients fp32 and rounded to bf16 like eager's.  ``pg``: where they go, numbered wq, wk, wv, wo, bo from 0
    (default: fresh tensors)."""
    x, c, q, k, v, o, lse, w_in, w_kv, w_o = saved
    M, Dq = x.shape
    L = q.shape[1]
    dev = dy.device
    pg = pg or checkpoint.NO_GRADS
    dwo = pg.out(3, tuple(w_o.shape), dev)
    dbo = pg.out(4, (Dq,), dev)
    ops.wgrad(dy, o, dwo, **pg.mode)
    ops.colsum(dy, dbo, **pg.mode)
    do = ops.gemm(dy, w_o, b_mn_major=True)
    if c is None:
        dqkv = torch.empty((M, 3 * L), dtype=torch.bfloat16, device=dev)
        ops.cross_attention_bwd(q, k, v, o, do, lse, B, heads, dq=dqkv[:, :L], dk=dqkv[:, L:2 * L], dv=dqkv[:, 2 * L:])
        dw, direct = pg.span((0, 1, 2), (3 * L, Dq), dev)  # the arena views of [Wq; Wk; Wv] when they are adjacent
        ops.wgrad(dqkv, x, dw, **(pg.mode if direct else {}))
        dwq, dwk, dwv = dw[:L], dw[L:2 * L], dw[2 * L:]
        if not direct:
            dwq, dwk, dwv = pg.put(0, dwq), pg.put(1, dwk), pg.put(2, dwv)
        dx = ops.gemm(dqkv, w_in, b_mn_major=True)
        dc = None
    else:
        dq = torch.empty((M, L), dtype=torch.bfloat16, device=dev)
        dkv = torch.empty((c.shape[0], 2 * L), dtype=torch.bfloat16, device=dev)
        ops.cross_attention_bwd(q, k, v, o, do, lse, B, heads, dq=dq, dk=dkv[:, :L], dv=dkv[:, L:])
        dwq = pg.out(0, (L, Dq), dev)
        dwkv, direct = pg.span((1, 2), (2 * L, c.shape[1]), dev)
        ops.wgrad(dq, x, dwq, **pg.mode)
        ops.wgrad(dkv, c, dwkv, **(pg.mode if direct else {}))
        dwk, dwv = dwkv[:L], dwkv[L:]
        if not direct:
            dwk, dwv = pg.put(1, dwk), pg.put(2, dwv)
        dx = ops.gemm(dq, w_in, b_mn_major=True)
        dc = ops.gemm(dkv, w_kv, b_mn_major=True)
    return dx, dc, dwq, dwk, dwv, dwo, dbo


@dataclass(frozen=True)
class _AttentionOp:
    """CrossAttentionB200 as a ``checkpoint.OpFn`` op on (net [B, Tq, Dq], context [B, Tk, Dc] or None, wq, wk, wv, wo, bo)."""
    B: int
    heads: int

    def forward(self, net: Tensor, context: Optional[Tensor], *params: Tensor) -> Tuple[Tensor, tuple]:
        y, saved = attention_forward(_rows(net), _rows(context), *params, self.B, self.heads)
        return y.view(net.shape), saved

    def backward(self, saved: tuple, dy: Tensor, pg: Optional[checkpoint.ParamGrads] = None) -> tuple:
        pg = pg or checkpoint.NO_GRADS
        return attention_backward(saved, _rows(dy), self.B, self.heads, pg.sub(2))


class _Linear(nn.Module):
    """Parameter holder with nn.Linear's parameter names and shapes (the reference's HijackLinear)."""

    def __init__(self, in_dim: int, out_dim: int, bias: bool) -> None:
        super().__init__()
        self.weight = nn.Parameter(torch.empty(out_dim, in_dim))
        self.bias = nn.Parameter(torch.empty(out_dim)) if bias else None
        ref = nn.Linear(in_dim, out_dim, bias=bias)  # nn.Linear's initialisation
        with torch.no_grad():
            self.weight.copy_(ref.weight)
            if bias:
                self.bias.copy_(ref.bias)


class CrossAttentionB200(nn.Module):
    """Drop-in for cflearn's ``CrossAttention`` on the native kernels (bf16 compute, fp32 parameters; CUDA only)."""

    def __init__(self, *, query_dim: int, context_dim: Optional[int] = None, num_heads: int = 8, head_dim: int = 64,
                 dropout: float = 0.0) -> None:
        super().__init__()
        if dropout > 0.0:
            raise NotImplementedError("CrossAttentionB200: dropout > 0 is not supported")
        self.has_context = context_dim is not None
        latent_dim = head_dim * num_heads
        context_dim = context_dim or query_dim
        self.num_heads = num_heads
        self.to_q = _Linear(query_dim, latent_dim, bias=False)
        self.to_k = _Linear(context_dim, latent_dim, bias=False)
        self.to_v = _Linear(context_dim, latent_dim, bias=False)
        self.out_linear = nn.Sequential(_Linear(latent_dim, query_dim, bias=True), nn.Dropout(dropout))

    def forward(self, net: Tensor, *, context: Optional[Tensor] = None, mask: Optional[Tensor] = None) -> Tensor:
        if mask is not None:
            raise NotImplementedError("CrossAttentionB200: attention masks are not supported")
        _check_cuda("CrossAttentionB200", net, context)
        B, _, _ = net.shape  # tokens [B, Tq, query_dim]
        lin = self.out_linear[0]
        return checkpoint.OpFn.apply(_AttentionOp(B, self.num_heads), False, net, context, self.to_q.weight, self.to_k.weight,
                                     self.to_v.weight, lin.weight, lin.bias)
