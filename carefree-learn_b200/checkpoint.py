"""Activation checkpointing for the native autograd Functions: what ``use_checkpoint`` does in the SD-UNet blocks (the reference
hands that keyword to ``gradient_checkpoint``, which keeps a block's inputs and reruns the block in backward).

A Function's forward is a builder ``build(*inputs) -> (out, saved)``: it launches the forward kernels and returns, with the
output, the tensors its backward reads.  Without checkpointing the Function keeps ``saved`` for backward; with it, it keeps
``inputs`` alone and reruns ``build`` on them into fresh buffers when backward starts.  The forward kernels are deterministic (the
GEMM's static persistent schedule, the streamed attention, fixed-order GroupNorm / LayerNorm statistics), so the rebuilt tensors,
and with them every gradient, equal the stored path's bit for bit.  Checkpointing trades the activations held between forward
and backward for one more run of the forward's launches in backward.
"""
from __future__ import annotations

from typing import Callable, Sequence, Tuple

from torch import Tensor

Build = Callable[..., Tuple[Tensor, tuple]]


def run(build: Build, inputs: Sequence, enabled: bool) -> Tuple[Tensor, tuple]:
    """Runs ``build(*inputs)``.  Returns (its output, what to keep for backward: its saved tensors, or ``inputs`` when
    ``enabled``, in which case the saved tensors are released on return)."""
    out, saved = build(*inputs)
    return out, tuple(inputs) if enabled else tuple(saved)


def rebuild(build: Build, kept: Sequence, enabled: bool) -> tuple:
    """``build``'s saved tensors from what ``run`` kept: ``kept`` itself, or when ``enabled`` those of ``build`` rerun on it."""
    return tuple(build(*kept)[1]) if enabled else tuple(kept)
