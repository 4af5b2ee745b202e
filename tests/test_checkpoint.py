"""checkpoint.OpFn, the autograd Function of the SD-UNet's native modules, on CPU toy ops: what each mode keeps for backward,
that checkpointed backward reruns the op's forward exactly once, and how gradients are handed back (the input's dtype and shape,
a permuted gradient's strides, None inputs)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cflearn_b200  # noqa: F401,E402
from cflearn_b200.checkpoint import OpFn  # noqa: E402


class _Affine:
    """y = x * w (+ b) over the last dim, in fp32 on [rows, D] and returned in x's dtype; the gradients come back as fp32 rows."""

    def __init__(self) -> None:
        self.forwards = 0

    def forward(self, x, w, b):
        self.forwards += 1
        xr = x.reshape(-1, x.shape[-1]).float()
        y = xr * w if b is None else xr * w + b
        return y.to(x.dtype).view(x.shape), (xr, w, b)

    def backward(self, saved, dy):
        xr, w, b = saved
        dyr = dy.reshape(-1, dy.shape[-1]).float()
        return dyr * w, (dyr * xr).sum(0), None if b is None else dyr.sum(0)


def _case(with_bias):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 3, 8, generator=g).to(torch.bfloat16).requires_grad_(True)
    w = torch.randn(8, generator=g).requires_grad_(True)
    b = torch.randn(8, generator=g).requires_grad_(True) if with_bias else None
    dy = torch.randn(2, 3, 8, generator=g).to(torch.bfloat16)
    return x, w, b, dy


def _run(flag, with_bias=True, retain=False):
    """Forward and backward(s) under a packing hook: (op, output, the tensors autograd packed, the inputs with their grads)."""
    op = _Affine()
    x, w, b, dy = _case(with_bias)
    packed = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: packed.append(t) or t, lambda t: t):
        y = OpFn.apply(op, flag, x, w, b)
    y.backward(dy, retain_graph=retain)
    if retain:
        y.backward(dy)
    return op, y, packed, (x, w, b)


def _same(a, b):
    return a.data_ptr() == b.data_ptr() and a.shape == b.shape


def test_each_mode_keeps_what_its_contract_says():
    op, _, packed, (x, w, b) = _run(False)
    assert len(packed) == 3 and packed[0].dtype == torch.float32 and packed[0].shape == (6, 8)  # saved: xr, w, b
    assert _same(packed[1], w) and _same(packed[2], b)
    op, _, packed, (x, w, b) = _run(True)
    assert len(packed) == 3 and all(_same(t, s) for t, s in zip(packed, (x, w, b)))  # the inputs alone


@pytest.mark.parametrize("retain", [False, True])
def test_checkpointed_backward_reruns_forward_once(retain):
    backwards = 2 if retain else 1
    stored, y_s, _, inputs_s = _run(False, retain=retain)
    ckpt, y_c, _, inputs_c = _run(True, retain=retain)
    assert stored.forwards == 1 and ckpt.forwards == 1 + backwards
    assert torch.equal(y_s, y_c)
    for s, c in zip(inputs_s, inputs_c):
        assert s.grad.stride() == c.grad.stride() and torch.equal(s.grad, c.grad)


@pytest.mark.parametrize("flag", [False, True])
def test_gradients_come_back_in_the_inputs_dtype_and_shape(flag):
    _, _, _, (x, w, b) = _run(flag)
    _, _, _, dy = _case(True)
    dyr = dy.reshape(-1, 8).float()
    assert x.grad.dtype == torch.bfloat16 and x.grad.shape == x.shape
    assert torch.equal(x.grad, (dyr * w.detach()).to(torch.bfloat16).view(x.shape))
    assert w.grad.dtype == torch.float32 and torch.equal(b.grad, dyr.sum(0))


@pytest.mark.parametrize("flag", [False, True])
def test_none_inputs(flag):
    op, y, _, (x, w, b) = _run(flag, with_bias=False)
    assert b is None and x.grad is not None and w.grad is not None
    assert op.forwards == (2 if flag else 1)


class _ChannelsLast:
    """Doubles an NCHW tensor through its NHWC view, and returns the gradient as a permuted NHWC tensor."""

    def forward(self, x):
        return (x.permute(0, 2, 3, 1).contiguous() * 2).permute(0, 3, 1, 2), ()

    def backward(self, saved, dy):
        return ((dy.permute(0, 2, 3, 1).contiguous() * 2).permute(0, 3, 1, 2),)


@pytest.mark.parametrize("flag", [False, True])
def test_a_permuted_gradient_keeps_its_strides(flag):
    leaf = torch.randn(2, 16, 4, 4, requires_grad=True)
    x = leaf * 1  # a contiguous NCHW non-leaf: the hook sees the gradient as OpFn returns it
    seen = []
    x.register_hook(lambda g: seen.append(g))
    y = OpFn.apply(_ChannelsLast(), flag, x)
    y.backward(torch.ones_like(y))
    cl = torch.empty(2, 16, 4, 4).contiguous(memory_format=torch.channels_last)
    assert seen[0].shape == x.shape and seen[0].stride() == cl.stride()
    assert torch.equal(seen[0], torch.full_like(x, 2.0))
