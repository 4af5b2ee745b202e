"""The autograd Function of the SD-UNet's native modules, with the activation checkpointing that ``use_checkpoint`` asks for (the
reference hands that keyword to ``gradient_checkpoint``, which keeps a block's inputs and reruns the block in backward).

A module describes one node of the graph as an op: an object that carries the node's non-tensor configuration (``B``,
``heads``, ``eps``, ...) and two functions,

    op.forward(*inputs) -> (out, saved)        launches the forward kernels; ``saved``: the tensors (or Nones) backward reads
    op.backward(saved, dout[, pg]) -> grads    one gradient (or None) per input; parameter gradients go through ``pg``

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

A parameter may carry a ``GradSlot`` (``unet.enable_grad_arena``): its view of a flat gradient arena and its all-reduce bucket.
The op's backward then writes that parameter's gradient straight into the view, with the kernel that produces it (``pg.out``
is the view, ``pg.mode`` adds ``accumulate`` when the arena already holds a gradient, ``ParamArena.claim_grads``), and autograd
receives None for it: no allocation per gradient and no accumulation pass.  Without slots ``pg`` hands out fresh tensors and the
op's kernel calls are exactly those of a plain op.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import torch
from torch import Tensor


def _like(g: Optional[Tensor], meta) -> Optional[Tensor]:
    if g is None:
        return None
    dtype, shape = meta
    if g.dtype != dtype:
        g = g.to(dtype)
    return g if g.shape == shape else g.reshape(shape)


class Bucket:
    """One all-reduce bucket of a gradient arena: ``done(n)`` after n of its ``size`` parameter gradients are written; the one
    that completes it calls ``ready(name)``.  ``reset`` starts a backward; after it ``left`` is 0 exactly when every gradient of
    the bucket was written once (negative: some twice, and the bucket was handed over before the last write)."""

    def __init__(self, name: str, size: int, ready: Callable[[str], None]) -> None:
        self.name, self.ready = name, ready
        self.reset(size)

    def reset(self, size: Optional[int] = None) -> None:
        if size is not None:
            self.size = size
        self.left = self.size

    def done(self, n: int) -> None:
        self.left -= n
        if self.left == 0:
            self.ready(self.name)


class GradSlot:
    """Where a parameter's gradient goes: key ``key`` of the ``ParamArena`` ``arena``, in ``bucket``."""

    def __init__(self, arena: Any, key: str, bucket: Bucket) -> None:
        self.arena, self.key, self.bucket = arena, key, bucket


SLOT_ATTR = "_b200_grad_slot"


class ParamGrads:
    """The parameter-gradient destinations of one op's backward, by input index: ``dest(i)`` the arena view of input i, or None
    (a fresh tensor).  ``mode``: the keyword arguments that make a kernel add to its output ({"accumulate": ...}), empty
    without an arena so the calls stay those of a plain op."""

    def __init__(self, dests: Sequence[Optional[Tensor]] = (), accumulate: bool = False) -> None:
        self.dests = list(dests)
        self.accumulate = accumulate
        self.mode: Dict[str, bool] = {"accumulate": accumulate} if any(d is not None for d in self.dests) else {}

    def dest(self, i: int) -> Optional[Tensor]:
        return self.dests[i] if i < len(self.dests) else None

    def sub(self, start: int) -> "ParamGrads":
        """The destinations of inputs start, start + 1, ... (for a helper that numbers its parameters from 0)."""
        return ParamGrads(self.dests[start:], self.accumulate)

    def out(self, i: int, shape: Tuple[int, ...], device: torch.device) -> Tensor:
        """The fp32 tensor the kernel producing input i's gradient writes (with ``mode``)."""
        d = self.dest(i)
        return torch.empty(shape, dtype=torch.float32, device=device) if d is None else d.view(shape)

    def put(self, i: int, g: Tensor) -> Tensor:
        """Input i's gradient ``g`` computed elsewhere: copied into (or added to) its view, else returned (contiguous)."""
        d = self.dest(i)
        if d is None:
            return g.contiguous()
        with torch.no_grad():
            if self.accumulate:
                d.add_(g.reshape(d.shape))
            else:
                d.copy_(g.reshape(d.shape))
        return d

    def norm_kw(self, i_gamma: int, i_beta: int) -> Dict[str, Any]:
        """``dgamma`` / ``dbeta`` / ``accumulate`` of a normalisation backward whose two affine gradients are inputs i_gamma, i_beta."""
        dg, db = self.dest(i_gamma), self.dest(i_beta)
        if dg is None or db is None:
            return {}
        return dict(dgamma=dg, dbeta=db, accumulate=self.accumulate)

    def span(self, idx: Sequence[int], shape: Tuple[int, ...], device: torch.device) -> Tuple[Tensor, bool]:
        """One fp32 tensor for the gradients of inputs ``idx`` stacked along dim 0 (e.g. [Wq; Wk; Wv]): their arena views when
        these are adjacent, else a fresh tensor (second value False: hand its rows to ``put``)."""
        views = [self.dest(i) for i in idx]
        if all(v is not None for v in views):
            base = views[0]
            n = sum(v.numel() for v in views)
            if all(v.data_ptr() == base.data_ptr() + 4 * sum(u.numel() for u in views[:k]) for k, v in enumerate(views)):
                return base.as_strided((n,), (1,)).view(shape), True
        return torch.empty(shape, dtype=torch.float32, device=device), False


NO_GRADS = ParamGrads()  # every gradient a fresh tensor: a plain op


def _slots(inputs: Sequence[Optional[Tensor]]) -> List[Optional[GradSlot]]:
    return [None if t is None or not t.requires_grad else getattr(t, SLOT_ATTR, None) for t in inputs]


class OpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx: Any, op: Any, use_checkpoint: bool, *inputs: Optional[Tensor]) -> Tensor:  # type: ignore[override]
        out, saved = op.forward(*inputs)
        ctx.save_for_backward(*(inputs if use_checkpoint else saved))
        ctx.op, ctx.use_checkpoint = op, use_checkpoint
        ctx.meta = [None if t is None else (t.dtype, t.shape) for t in inputs]
        ctx.slots = _slots(inputs)
        return out

    @staticmethod
    def backward(ctx: Any, dout: Tensor):  # type: ignore[override]
        kept = ctx.saved_tensors
        saved = ctx.op.forward(*kept)[1] if ctx.use_checkpoint else kept
        slots = ctx.slots
        used = [s for s in slots if s is not None]
        if used:
            arena = used[0].arena
            keys = [s.key for s in used]
            pg = ParamGrads([None if s is None else arena.g(s.key) for s in slots], arena.claim_grads(keys))
        grads = ctx.op.backward(saved, dout, pg) if used else ctx.op.backward(saved, dout)
        if used:
            arena.publish_grads(keys)
            counts: Dict[Bucket, int] = {}
            for s in used:
                counts[s.bucket] = counts.get(s.bucket, 0) + 1
            for b, n in counts.items():
                b.done(n)
        return (None, None, *(None if s is not None else _like(g, m) for g, m, s in zip(grads, ctx.meta, slots)))
