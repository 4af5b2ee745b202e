"""The fused FCNN step (b200_fcnn_step, csrc/mlp.cu) bit for bit, on operands whose every product and partial sum is exact in fp32.

The kernel is plain fp32 FFMA in a fixed order, one thread per sample, so on ``_refs.exact_fcnn_operands`` (small integers times a
power of two per layer, every sum under 2^24 units of its quantum) the only right pred, loss and gradient is the float64 one of
``_refs.fcnn_step``, to the bit.  A wrong ReLU mask at an exact zero, sign(0) != 0 in the L1 gradient, a missed ``valid`` guard on
the loss or the output gradient, a bias read from or written to the wrong offset, a row dropped from a block's sum, a stale
activation buffer, or a mean taken over the wrong count each change some bit.  The operands plant ReLU inputs and residuals that are
exactly 0.  The fused loss runs where M nout is a power of two (the kernel's fp32 1 / (M nout) is exact only then); every other M
runs with a given dpred.

Every call goes through ``ops.fcnn_step`` and through the raw C-ABI, with the arena's gaps, the block partials, the predictions and
the reduced gradients all NaN until the kernel writes them.  The sweep covers M across the 128-row block edges and more blocks than
SMs, 1 to 8 layers, widths 1, 31, 32, 33 and 129, bias on every layer, on none and alternating, the four loss weightings, inference
alone and no predictions, shared memory on both sides of 48 KB and exactly at the 220 KB cap (one float more is refused).  Random
Gaussian inputs are held, element by element, to ``_refs.fcnn_bounds``, a first-order fp32 error bound; two runs must be
bit-identical.  The FCNNB200 module's train_step and autograd route are checked against the same reference.  Run on an H100:
pytest -m gpu."""
import ctypes
import math

import pytest
import torch

import cflearn_b200  # noqa: F401  (registers the package)
from cflearn_b200 import _cabi, ops
from cflearn_b200._cabi import B200Error
from cflearn_b200.fcnn import FCNNB200
from _refs import FCNN_C, exact_fcnn_operands, fcnn_bounds, fcnn_step

DEV = "cuda"
ROWS = 128                     # samples per block (MLP_ROWS)
ACT_LD = ROWS + 1              # floats per unit of an activation buffer
SMEM_CAP = 220 * 1024 // 4     # floats of parameters + activations the kernel admits
SMEM_STATIC = 48 * 1024 // 4   # above this the launch raises the dynamic shared-memory limit first
B200_ERR_ARG = -1
LOSS_WEIGHTS = [(1.0, 1.0), (1.0, 0.0), (0.0, 1.0), (0.5, 2.0)]
NAN = float("nan")


def _bias(pattern, L):
    return {"all": [True] * L, "none": [False] * L, "alt": [l % 2 == 0 for l in range(L)]}[pattern]


# (dims, M, bias): every M of {1, 2, 127, 128, 129, 255, 256, 257, 1000} and one of more 128-row blocks than the 132 SMs; 1 to 8
# layers; widths 1, 31, 32, 33 and 129, input and output widths of 1 and more
CASES = [
    ([1, 1], 1, "all"),
    ([33, 1], 2, "none"),
    ([1, 129, 1], 127, "alt"),
    ([31, 32, 33, 32], 128, "all"),
    ([10, 32, 32, 1], 129, "all"),
    ([129, 33, 1, 31, 2], 255, "alt"),
    ([32, 129, 31, 33, 1, 32], 256, "none"),
    ([7, 33, 32, 31, 129, 1, 33, 1], 257, "alt"),
    ([2, 31, 32, 33, 31, 32, 33, 31, 1], 1000, "all"),
    ([1, 1, 1, 1, 1, 1, 1, 1, 1], 128, "all"),
    ([129, 129, 4], 2, "alt"),
    ([10, 32, 32, 1], 133 * ROWS + 5, "alt"),
]


def smem_floats(dims, P):
    return P + ACT_LD * sum(dims)


def _bits(t):
    return t.contiguous().view(torch.int32)


def assert_exact(got, want, what):
    """fp32 ``got`` equals float64 ``want`` (exact in fp32) bit for bit; names the first bad element."""
    got, want = got.reshape(got.shape or (1,)), want.reshape(want.shape or (1,))
    want32 = want.to(torch.float32).to(got.device)
    assert torch.equal(want32.double(), want.to(got.device)), f"{what}: the reference is not exact in fp32"
    bad = _bits(got) != _bits(want32)
    if bad.any():
        i = tuple(torch.nonzero(bad)[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ, first at {i}: got {got[i].item()!r}, "
                             f"expected {want32[i].item()!r}")


def _ptr(t):
    return None if t is None else t.data_ptr()


def _ints(v):
    return (ctypes.c_int * len(v))(*v)


def raw_step(x, params, dims, woff, boff, *, y=None, dpred=None, w=(1.0, 1.0), with_pred=True, with_part=True, P=None):
    """One b200_fcnn_step call with NaN-filled pred and partials, then b200_colsum_finish of the partials into NaN-filled
    gradients and loss.  Returns the status and {pred, grads, loss} of what was asked for."""
    M, nout = x.shape[0], dims[-1]
    P = params.numel() if P is None else P
    nblk = -(-M // ROWS)
    pred = torch.full((M, nout), NAN, device=DEV) if with_pred else None
    part = torch.full((nblk, P + 1), NAN, device=DEV) if with_part else None
    nb = ctypes.c_int(-1)
    stream = torch.cuda.current_stream().cuda_stream
    status = _cabi.lib().b200_fcnn_step(x.data_ptr(), _ptr(y), _ptr(dpred), params.data_ptr(), _ptr(pred), _ptr(part), M, len(dims) - 1,
                                        _ints(dims), _ints(woff), _ints(boff), P, int(y is not None), w[0], w[1], ctypes.byref(nb),
                                        stream)
    out = {"status": status, "pred": pred}
    if status == 0:
        assert nb.value == nblk
        if part is not None:
            out["grads"] = torch.full((P,), NAN, device=DEV)
            out["loss"] = torch.full((), NAN, device=DEV)
            _cabi.call("b200_colsum_finish", part.data_ptr(), P + 1, nblk, P, out["grads"].data_ptr(), 0, 0, stream)
            _cabi.call("b200_colsum_finish", part.data_ptr() + 4 * P, P + 1, nblk, 1, out["loss"].data_ptr(), 0, 0, stream)
    torch.cuda.synchronize()
    return out


def check_exact_step(o, dims, what, w=(1.0, 1.0)):
    """Every route of one exact case against fcnn_step: ops training and inference, raw with and without pred or partials."""
    x, params = o["x"].to(DEV), o["params"].to(DEV)
    y = o["y"].to(DEV) if "y" in o else None
    dpred = o["dpred"].to(DEV) if "dpred" in o else None
    woff, boff = o["woff"], o["boff"]
    pred, loss, grads = fcnn_step(x, params, dims, woff, boff, y=y, dpred=dpred, w_mae=w[0], w_mse=w[1])
    what = f"{what} {'loss_mode 1 w ' + str(w) if y is not None else 'loss_mode 0'}"

    G = torch.full_like(params, NAN)
    got_pred, got_loss = ops.fcnn_step(x, params, dims, woff, boff, y=y, dpred=dpred, grads=G, loss_weights=w)
    torch.cuda.synchronize()
    assert_exact(got_pred, pred, f"{what} ops pred")
    assert_exact(G, grads, f"{what} ops grads")
    if y is not None:
        assert_exact(got_loss, loss, f"{what} ops loss")
    else:
        assert got_loss is None

    inf_pred, inf_loss = ops.fcnn_step(x, params, dims, woff, boff)
    torch.cuda.synchronize()
    assert_exact(inf_pred, pred, f"{what} ops inference pred")
    assert inf_loss is None

    r = raw_step(x, params, dims, woff, boff, y=y, dpred=dpred, w=w)
    assert r["status"] == 0, _cabi.last_error()
    assert_exact(r["pred"], pred, f"{what} raw pred")
    assert_exact(r["grads"], grads, f"{what} raw grads")
    assert_exact(r["loss"], loss if y is not None else torch.zeros((), dtype=torch.float64), f"{what} raw loss column")

    r = raw_step(x, params, dims, woff, boff, y=y, dpred=dpred, w=w, with_pred=False)
    assert r["status"] == 0 and r["pred"] is None
    assert_exact(r["grads"], grads, f"{what} raw grads without pred")

    r = raw_step(x, params, dims, woff, boff, y=y, dpred=dpred, w=w, with_part=False)
    assert r["status"] == 0
    assert_exact(r["pred"], pred, f"{what} raw inference pred")


def run_case(dims, M, bias, seed, what, **kw):
    """loss_mode 0 with an exact dpred; where M nout is a power of two also the fused loss under every weighting."""
    L = len(dims) - 1
    check_exact_step(exact_fcnn_operands(dims, M, _bias(bias, L), seed, **kw), dims, what)
    n = M * dims[-1]
    if n & (n - 1) == 0:
        for i, w in enumerate(LOSS_WEIGHTS):
            o = exact_fcnn_operands(dims, M, _bias(bias, L), seed + 100 + i, y=True, w_mae=w[0], w_mse=w[1], **kw)
            check_exact_step(o, dims, what, w)


@pytest.mark.gpu
@pytest.mark.parametrize("dims,M,bias", CASES, ids=lambda v: str(v))
def test_fcnn_step_exact(dims, M, bias):
    run_case(dims, M, bias, seed=M + 7 * len(dims), what=f"dims {dims} M {M} bias {bias}")


# networks padded to fill shared memory exactly: 48 KB (the launch keeps the default limit), 48 KB + 4 bytes (it raises the
# limit first) and the 220 KB cap
SMEM_CASES = [([8, 32, 32, 4], SMEM_STATIC), ([8, 32, 32, 4], SMEM_STATIC + 1), ([16, 129, 129, 1], SMEM_CAP)]


@pytest.mark.gpu
@pytest.mark.parametrize("dims,floats", SMEM_CASES, ids=lambda v: str(v))
def test_fcnn_step_exact_at_shared_memory_edges(dims, floats):
    arena_len = floats - ACT_LD * sum(dims)
    for M, bias in ((256, "all"), (257, "alt")):
        run_case(dims, M, bias, seed=floats + M, what=f"dims {dims} smem {4 * floats} B M {M} bias {bias}", arena_len=arena_len)


@pytest.mark.gpu
def test_fcnn_step_refuses_one_float_past_the_cap():
    """The 220 KB network with an arena one float longer: B200_ERR_ARG naming the shared-memory limit, from the C-ABI and from
    ops, and nothing written."""
    dims = [16, 129, 129, 1]
    P = SMEM_CAP - ACT_LD * sum(dims) + 1
    o = exact_fcnn_operands(dims, 129, _bias("all", 3), 5, arena_len=P)
    x, params, dpred = o["x"].to(DEV), o["params"].to(DEV), o["dpred"].to(DEV)
    assert smem_floats(dims, P) == SMEM_CAP + 1
    r = raw_step(x, params, dims, o["woff"], o["boff"], dpred=dpred)
    assert r["status"] == B200_ERR_ARG and "shared-memory" in _cabi.last_error(), (r["status"], _cabi.last_error())
    assert torch.isnan(r["pred"]).all(), "a refused call wrote predictions"
    G = torch.full_like(params, NAN)
    with pytest.raises(B200Error, match="shared-memory"):
        ops.fcnn_step(x, params, dims, o["woff"], o["boff"], dpred=dpred, grads=G)
    torch.cuda.synchronize()
    assert torch.isnan(G).all()


# ---- random inputs against the first-order bound ------------------------------------------------------------------------------
def _random_network(dims, M, seed):
    g = torch.Generator().manual_seed(seed)
    L = len(dims) - 1
    woff, boff, cur = [], [], 0
    for l in range(L):
        woff.append(cur)
        boff.append(cur + dims[l] * dims[l + 1])
        cur += dims[l] * dims[l + 1] + dims[l + 1]
    params = torch.empty(cur)
    for l in range(L):
        params[woff[l]:boff[l]] = torch.randn(dims[l] * dims[l + 1], generator=g) * math.sqrt(2.0 / dims[l])
        params[boff[l]:boff[l] + dims[l + 1]] = torch.randn(dims[l + 1], generator=g) * 0.1
    x = torch.randn(M, dims[0], generator=g)
    y = torch.randn(M, dims[-1], generator=g)
    return x.to(DEV), params.to(DEV), woff, boff, y.to(DEV)


# the BASELINE 10 -> 32 -> 32 -> 1 network at batch 128 and on 1000 rows; an 8-layer network of width 44 at 215 KB of shared memory
RANDOM_CASES = [([10, 32, 32, 1], 128), ([10, 32, 32, 1], 1000), ([16] + [44] * 7 + [4], 1000)]


@pytest.mark.gpu
@pytest.mark.parametrize("dims,M", RANDOM_CASES, ids=lambda v: str(v))
def test_fcnn_step_random_within_bound(dims, M):
    """Gaussian inputs, the fused loss: every element of pred, the loss and every gradient within fcnn_bounds (C = FCNN_C); a second
    run is bit-identical."""
    x, params, woff, boff, y = _random_network(dims, M, seed=M + len(dims))
    w = (1.0, 1.0)
    (pred, loss, grads), (tol_pred, tol_loss, tol_grads) = fcnn_bounds(x, params, dims, woff, boff, y=y, w_mae=w[0], w_mse=w[1])
    runs = []
    for _ in range(2):
        G = torch.full_like(params, NAN)
        p, l = ops.fcnn_step(x, params, dims, woff, boff, y=y, grads=G, loss_weights=w)
        torch.cuda.synchronize()
        runs.append((p, l, G))
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(_bits(a), _bits(b)), f"dims {dims} M {M}: two runs differ"
    for name, got, ref, tol in (("pred", runs[0][0], pred, tol_pred), ("loss", runs[0][1], loss, tol_loss),
                                ("grads", runs[0][2], grads, tol_grads)):
        err = (got.double() - ref).abs()
        bad = ~(err <= tol)
        if bad.any():
            i = tuple(torch.nonzero(bad.reshape(bad.shape or (1,)))[0].tolist())
            raise AssertionError(f"dims {dims} M {M} {name}: {int(bad.sum())} elements outside the bound, first at {i}: "
                                 f"error {err.reshape(err.shape or (1,))[i].item():.3g} > {tol.reshape(tol.shape or (1,))[i].item():.3g}")
        ratio = (err / tol.clamp_min(1e-300)).max().item()
        print(f"fcnn random dims {dims} M {M} {name}: worst error / bound {ratio:.3e} (C = {FCNN_C})")


# ---- the module ----------------------------------------------------------------------------------------------------------------------
def _exact_module(dims, bias, M, seed, **kw):
    """FCNNB200 on the device whose arena holds exact operands (NaN in its alignment gaps), and those operands."""
    m = FCNNB200(dims[0], dims[-1], dims[1:-1], bias=bias).to(DEV)
    m.arena.ensure()
    o = exact_fcnn_operands(dims, M, [bias] * (len(dims) - 1), seed, layout=(m._woff, m._boff, m.arena.total), **kw)
    with torch.no_grad():
        m.arena.flat.copy_(o["params"].to(DEV))
    return m, o


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [True, False])
def test_module_train_step_exact(bias):
    """FCNNB200.train_step with loss_weights (0.5, 2): loss, predictions and every parameter's .grad bit for bit."""
    dims, M, w = [10, 33, 32, 31, 2], 256, (0.5, 2.0)
    m, o = _exact_module(dims, bias, M, seed=11 + bias, y=True, w_mae=w[0], w_mse=w[1])
    x, y = o["x"].to(DEV), o["y"].to(DEV)
    pred, loss, grads = fcnn_step(x, m.arena.flat, dims, m._woff, m._boff, y=y, w_mae=w[0], w_mse=w[1])
    got_loss, got_pred = m.train_step(x, y, loss_weights=w)
    torch.cuda.synchronize()
    assert_exact(got_pred, pred, "train_step pred")
    assert_exact(got_loss, loss, "train_step loss")
    for k, p in m.named_parameters():
        assert_exact(p.grad, m.arena.view(grads, k), f"train_step {k}.grad")


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [True, False])
def test_module_autograd_exact(bias):
    """forward, then a user loss sum(pred * dpred): the backward re-runs the kernel with loss_mode 0; every .grad bit for bit."""
    dims, M = [10, 33, 32, 31, 2], 1000
    m, o = _exact_module(dims, bias, M, seed=21 + bias)
    x, dpred = o["x"].to(DEV), o["dpred"].to(DEV)
    pred, _, grads = fcnn_step(x, m.arena.flat, dims, m._woff, m._boff, dpred=dpred)
    out = m(x)
    (out * dpred).sum().backward()
    torch.cuda.synchronize()
    assert_exact(out.detach(), pred, "forward")
    for k, p in m.named_parameters():
        assert_exact(p.grad, m.arena.view(grads, k), f"autograd {k}.grad")


@pytest.mark.gpu
def test_module_default_hidden_units_past_the_cap():
    """The reference's default hidden_units, 2 x [max(32, min(1024, 2 input_dim))]: input_dim 56 is the widest that fits the 220 KB
    of shared memory and runs; 57 and 600 ([1024, 1024]) are refused with the shared-memory message on the first forward."""
    x = torch.ones(3, 56, device=DEV)
    assert FCNNB200(56, 1).to(DEV)(x).shape == (3, 1)
    for input_dim, output_dim in ((57, 1), (600, 3)):
        m = FCNNB200(input_dim, output_dim).to(DEV)
        with pytest.raises(B200Error, match="shared-memory"):
            m(torch.randn(4, input_dim, device=DEV))
        with torch.no_grad(), pytest.raises(B200Error, match="shared-memory"):
            m(torch.randn(4, input_dim, device=DEV))
