"""CPU: the exact operands of test_fcnn_exact_gpu.py.  For every case of that sweep, every sum the fused FCNN step computes -- each
forward pre-activation, the loss, each output gradient, each weight and bias gradient over all rows, each input gradient -- comes
out of fp32 additions in forward, reverse and pairwise order equal to its float64 value, so no order of the kernel's (or of the
block reduction's) can change a bit.  The planted zeros are where the generator says, and it refuses operands over its budget."""
import pytest
import torch

from _refs import FCNN_BUDGET, exact_fcnn_operands, fcnn_forward, fcnn_layers
import test_fcnn_exact_gpu as sweep

F64 = torch.float64


def sweep_operands():
    """(name, dims, operands, loss weights) of every exact case the GPU sweep runs."""
    def case(dims, M, bias, seed, **kw):
        L = len(dims) - 1
        yield f"dims {dims} M {M} loss_mode 0", dims, exact_fcnn_operands(dims, M, sweep._bias(bias, L), seed, **kw), (1.0, 1.0)
        n = M * dims[-1]
        if n & (n - 1) == 0:
            for i, w in enumerate(sweep.LOSS_WEIGHTS):
                o = exact_fcnn_operands(dims, M, sweep._bias(bias, L), seed + 100 + i, y=True, w_mae=w[0], w_mse=w[1], **kw)
                yield f"dims {dims} M {M} loss_mode 1 w {w}", dims, o, w

    for dims, M, bias in sweep.CASES:
        yield from case(dims, M, bias, M + 7 * len(dims))
    for dims, floats in sweep.SMEM_CASES:
        for M, bias in ((256, "all"), (257, "alt")):
            yield from case(dims, M, bias, floats + M, arena_len=floats - sweep.ACT_LD * sum(dims))


def sums(o, dims, w):
    """(what, terms [..., n]) of every sum of the step, in float64; each term is one fp32 product (or, for the loss and the output
    gradient, one of the two products of an element)."""
    layers = fcnn_layers(o["params"], dims, o["woff"], o["boff"])
    _, acts = fcnn_forward(o["x"], layers)
    M = acts[0].shape[0]
    for l, (W, b) in enumerate(layers):
        terms = acts[l][:, None, :] * W[None]
        if b is not None:
            terms = torch.cat([b.expand(M, -1)[..., None], terms], -1)
        yield f"layer {l} forward", terms
    if "y" in o:
        d = acts[-1] - o["y"].to(F64)
        yield "loss", torch.stack([w[0] * d.abs(), w[1] * d * d], -1).reshape(1, -1)
        grad = torch.stack([w[0] * torch.sign(d), 2 * w[1] * d], -1)
        yield "output gradient", grad
        g = grad.sum(-1) / d.numel()
    else:
        g = o["dpred"].to(F64)
    for l in reversed(range(len(layers))):
        W, _ = layers[l]
        yield f"layer {l} weight gradient", (g[:, :, None] * acts[l][:, None, :]).permute(1, 2, 0)
        yield f"layer {l} bias gradient", g.t()
        if l > 0:
            t = g[:, :, None] * W[None]  # [M, out, in]
            yield f"layer {l} input gradient", t.transpose(1, 2)
            g = torch.where(acts[l] > 0, t.sum(1), torch.zeros_like(acts[l]))


def fp32_orders(terms):
    """fp32 sums over the last dim: forward, reverse and pairwise."""
    t = terms.to(torch.float32)
    fwd, rev = torch.zeros(t.shape[:-1]), torch.zeros(t.shape[:-1])
    n = t.shape[-1]
    for i in range(n):
        fwd = fwd + t[..., i]
        rev = rev + t[..., n - 1 - i]
    pw = t
    while pw.shape[-1] > 1:
        if pw.shape[-1] % 2:
            pw = torch.cat([pw, torch.zeros_like(pw[..., :1])], -1)
        pw = pw[..., 0::2] + pw[..., 1::2]
    return {"forward": fwd, "reverse": rev, "pairwise": pw[..., 0]}


def test_sums_are_exact_in_any_order():
    for name, dims, o, w in sweep_operands():
        assert sweep.smem_floats(dims, o["params"].numel()) <= sweep.SMEM_CAP, f"{name}: the kernel would refuse it"
        for what, terms in sums(o, dims, w):
            assert torch.equal(terms.to(torch.float32).to(F64), terms), f"{name} {what}: a term is not exact in fp32"
            exact = terms.sum(-1)
            for order, s in fp32_orders(terms).items():
                assert torch.equal(s.to(F64), exact), f"{name} {what}: the fp32 sum in {order} order is not exact"


def test_planted_zeros_are_there():
    """Every planted ReLU input and residual is exactly 0, and every case with a hidden layer or the fused loss plants some."""
    for name, dims, o, _ in sweep_operands():
        pre, acts = fcnn_forward(o["x"], fcnn_layers(o["params"], dims, o["woff"], o["boff"]))
        for l, r, j in o["relu_zeros"]:
            assert pre[l][r, j].item() == 0.0, f"{name}: layer {l} row {r} unit {j} pre-activation {pre[l][r, j].item()}"
        if any(n > 1 for n in dims[1:-1]):
            assert o["relu_zeros"], f"{name}: no ReLU input planted at 0"
        if "y" in o:
            d = acts[-1] - o["y"].to(F64)
            for r, j in o["residual_zeros"]:
                assert d[r, j].item() == 0.0, f"{name}: residual ({r}, {j}) = {d[r, j].item()}"
            assert (d == 0).sum().item() == len(o["residual_zeros"]), f"{name}: residuals are 0 only where planted"
            assert o["residual_zeros"] or d.numel() < 3


def test_generator_refuses_operands_over_budget():
    dense = dict(dims=[129] * 9, M=256, bias=[True] * 8, seed=0)
    with pytest.raises(AssertionError, match="budget"):
        exact_fcnn_operands(**dense, fan=129.0)
    with pytest.raises(AssertionError, match="power of two"):
        exact_fcnn_operands([10, 32, 1], 129, [True, True], 0, y=True)
    with pytest.raises(AssertionError, match="arena_len"):
        exact_fcnn_operands([10, 32, 1], 128, [True, True], 0, arena_len=100)
    # the densest weights that fit: the same network refused at the density above is accepted, under the budget
    o = exact_fcnn_operands(**dense)
    assert o["params"].numel() >= 8 * (129 * 129 + 129) and FCNN_BUDGET == 2 ** 24
