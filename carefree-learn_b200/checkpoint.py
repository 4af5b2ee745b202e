"""The autograd Function of the SD-UNet's native modules, with the activation checkpointing that ``use_checkpoint`` asks for (the
reference hands that keyword to ``gradient_checkpoint``, which keeps a block's inputs and reruns the block in backward).

A module describes one node of the graph as an op: an object that carries the node's non-tensor configuration (``B``,
``heads``, ``eps``, ...) and two functions,

    op.forward(*inputs) -> (out, saved)    launches the forward kernels; ``saved``: the tensors (or Nones) backward reads
    op.backward(saved, dout) -> grads      one gradient (or None) per input

and applies it as ``OpFn.apply(op, use_checkpoint, *inputs)``.  Without checkpointing the node keeps ``saved`` for backward;
with it, it keeps ``inputs`` alone and reruns ``op.forward`` on them into fresh buffers when backward starts.  The forward
kernels are deterministic (the GEMM's static persistent schedule, the streamed attention, fixed-order GroupNorm / LayerNorm
statistics), so the rebuilt tensors, and with them every gradient, equal the stored path's bit for bit.  Checkpointing trades
the activations held between forward and backward for one more run of the forward's launches in backward.

Everything is kept through ``save_for_backward``, so ``retain_graph``, saved-tensor hooks and autograd's in-place checks apply
as for any other op.  Each gradient comes back in its input's dtype, and is reshaped to the input's shape only where the
shapes differ: a gradient the op returns as a permuted view (NCHW with channels-last strides) keeps its strides.  A module
made of several nodes is a chain of ``OpFn`` applications, and autograd sums the gradients of an input that several nodes
read.  The Function itself touches no device; the ops do.
"""
from __future__ import annotations

from typing import Any, Optional

import torch
from torch import Tensor


def _like(g: Optional[Tensor], meta) -> Optional[Tensor]:
    if g is None:
        return None
    dtype, shape = meta
    if g.dtype != dtype:
        g = g.to(dtype)
    return g if g.shape == shape else g.reshape(shape)


class OpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx: Any, op: Any, use_checkpoint: bool, *inputs: Optional[Tensor]) -> Tensor:  # type: ignore[override]
        out, saved = op.forward(*inputs)
        ctx.save_for_backward(*(inputs if use_checkpoint else saved))
        ctx.op, ctx.use_checkpoint = op, use_checkpoint
        ctx.meta = [None if t is None else (t.dtype, t.shape) for t in inputs]
        return out

    @staticmethod
    def backward(ctx: Any, dout: Tensor):  # type: ignore[override]
        kept = ctx.saved_tensors
        saved = ctx.op.forward(*kept)[1] if ctx.use_checkpoint else kept
        grads = ctx.op.backward(saved, dout)
        return (None, None, *(_like(g, m) for g, m in zip(grads, ctx.meta)))
