"""Per-op checks of the SD-UNet's native blocks (tests/test_unet_ops_gpu.py): each block's op table, the float64 check of every
entry point, and the two ways a table is run.

An op table is the list of calls a block's module makes, in order: the ``ops`` entry point, every argument (where each tensor
comes from, every non-tensor value: epilogue, ``eps``, ``silu``, ``B``, ``heads``, ``b_mn_major``), the names of the results and,
for each result, eager's value of the same tensor.  A few rows are the torch glue between kernels (eager's own ops, which the
modules call as eager does).  A table is run two ways:

``teacher_forced``  each op on eager's own inputs of that op: the eager bf16-autocast oracle's activation and upstream gradient,
                    and the statistics our own forward op computed on eager's input.  Every output is checked element by
                    element against float64 of the same op, and against eager's output of the op.
``wiring``          the module's real forward and backward, with ``ops`` replaced by a ``Recorder`` that logs each call.  The
                    log must be the table: the same entry points and non-tensor arguments, every tensor argument bit-equal to
                    the table's source (an earlier call's output, a module input or a cast parameter), every output within the
                    float64 bound of the op on the inputs it received, and the module's outputs and gradients bit-equal to the
                    table's.

Element-wise bounds.  u = 2^-24 (fp32), a sum of n exact bf16 x bf16 products in any order is off by at most n u sum|terms| (the
worst-case bound of recursive summation, which holds for any order and any split, so c = 1 there).  A bf16 output must be
within ``assert_ulp(..., ulps=1.01)`` of float64 at our documented rounding points, the fp32 error passed through assert_ulp's
``mag``; an fp32 gradient within that error, plus 2^-8 |ref| where it is rounded to bf16 as eager's.  Elementwise fp32 chains
(a GroupNorm / LayerNorm output, SiLU) use c = 8 per operation: each of their few fp32 operations and fast-math functions
(exp, rsqrt, reciprocal) is within 2 u, and 8 leaves a margin of 4 without hiding a wrong constant or operand.  Attention uses
``_refs.attention_bounds_rows``, one head at a time."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from _refs import (FP32_U, GELU_ATOL, assert_ulp, attention_bounds_rows, colsum_per_image, conv3x3, conv3x3_s2, conv3x3_s2_dgrad,
                   conv3x3_s2_wgrad, conv3x3_up2, conv3x3_wgrad, gelu, gelu_grad, relerr)

from cflearn_b200 import ops

F64 = torch.float64
BF = torch.bfloat16
U16 = 2.0 ** -8   # one bf16 rounding, relative
C_EW = 8          # elementwise fp32 chains: see the module docstring
TOL = 1e-3        # against eager's output of the same op (test_taps_gpu.TOL)
TOL_ATTN = 2e-3   # the attention ops (test_taps_gpu.TOL_ATTN: both round the probabilities to bf16, at different points)
TWICE = "2x"      # ops whose rounding point the modules document as different from eager's: 2 x relerr(eager, float64)

# every kernel entry point the blocks call (the weight-packing helpers are plain torch and checked through their outputs)
KERNELS = {"gemm", "geglu", "wgrad", "colsum", "colsum_per_image", "layernorm_bf16_fwd", "layernorm_bf16_bwd", "cross_attention_fwd",
           "cross_attention_bwd", "groupnorm_silu_fwd", "groupnorm_silu_bwd", "conv3x3", "conv3x3_wgrad", "conv3x3_s2", "conv3x3_up2",
           "conv3x3_s2_dgrad", "conv3x3_s2_wgrad", "upsample_nearest2x", "sum2x2"}


# ---- bounds ------------------------------------------------------------------------------------------------------------------
class Report:
    """The worst element-wise error / bound ratio and the eager comparisons of one test."""

    def __init__(self) -> None:
        self.worst: Tuple[float, str] = (0.0, "")
        self.eager: List[Tuple[str, float, float, str]] = []  # (what, relerr vs eager, its bound, rule)

    def ratio(self, r: float, what: str) -> None:
        self.worst = max(self.worst, (r, what))


REPORT = Report()


def d(t):
    return t.to(F64)


def within(got, ref, err, what, kind="bf16"):
    """``kind`` "bf16": a bf16 output, assert_ulp(ulps=1.01) of ``ref`` plus ``err``; "grad": an fp32 sum rounded to bf16, 2^-8 |ref| +
    ``err``; "f32": ``err``.  Records the worst |got - ref| / bound."""
    g, r = d(got).reshape(ref.shape), ref
    err = torch.broadcast_to(err, r.shape)
    if kind == "bf16":
        ulps = 1.01
        mag = r.abs() + err / (ulps * 2.0 ** -7)
        tol = ulps * 2.0 ** -7 * mag + 1e-6 * r.abs().max().clamp_min(1e-30)
        assert_ulp(g, r, what, ulps=ulps, mag=mag)
    else:
        tol = err + (U16 * r.abs() if kind == "grad" else 0.0) + 1e-30
        bad = ~((g - r).abs() <= tol)
        pos = tuple(torch.nonzero(bad)[0].tolist()) if bad.any() else None
        assert pos is None, f"{what}: element {pos} = {g[pos].item()} vs reference {r[pos].item()} (bound {tol[pos].item()})"
    REPORT.ratio(((g - r).abs() / tol).max().item(), what)


def sums(a, b):
    """(a b^T, |a| |b|^T) in float64 for a [M, K], b [N, K]."""
    a, b = d(a), d(b)
    return a @ b.t(), a.abs() @ b.abs().t()


# ---- float64 checks, one per entry point: (args, kwargs, outputs, what) -> float64 value of each output ----------------------
def _epilogue(out, acc, err, kw, what, rows=None):
    """The bias / residual epilogues on acc (float64) with fp32 error ``err``; ``rows``: the image of each row (per-image aux)."""
    bias = kw.get("bias")
    epi = kw.get("epilogue", 0)
    if bias is not None:
        acc = acc + d(bias)
        err = err + FP32_U * (acc.abs() + d(bias).abs())
    if epi == 0:
        within(out, acc, err, what)
        return acc
    aux = d(kw["aux"]).reshape(-1, acc.shape[1])
    if epi == 10:
        aux = aux[rows]
    assert epi in (9, 10, 11), epi
    ref = acc + aux  # bf16(bf16(acc + bias) + aux): the inner rounding is part of the error
    within(out, ref, U16 * (acc.abs() + err) + err, what)
    return ref


def chk_gemm(a, kw, out, what):
    A, W = a[0], a[1]
    if kw.get("b_mn_major"):
        W = W.t()
    acc, s = sums(A, W)
    err = A.shape[1] * FP32_U * s
    if kw.get("epilogue", 0) != 8:
        return [_epilogue(out[0], acc, err, kw, what)]
    # dGEGLU: da = bf16(acc); dh = bf16(da g), g = bf16(gelu(gate)); dgate = bf16(gelu'(gate) bf16(da h))
    hg = d(kw["aux"])
    Fd = acc.shape[1]
    h, gate = hg[:, :Fd], hg[:, Fd:]
    g = gelu(gate).to(torch.float32).to(BF).to(F64)
    eda = U16 * acc.abs() + err
    dh, e_dh = acc * g, eda * g.abs() + GELU_ATOL * acc.abs()
    gg = gelu_grad(gate)
    dgate = gg * acc * h
    e_dg = gg.abs() * (U16 * (acc * h).abs() + eda * h.abs()) + GELU_ATOL * (acc * h).abs()
    ref = torch.cat([dh, dgate], 1)
    within(out[0], ref, torch.cat([e_dh, e_dg], 1), what)
    return [ref]


def chk_geglu(a, kw, out, what):
    acc, s = sums(a[0], a[1])
    hg = _epilogue(out[0], acc, a[0].shape[1] * FP32_U * s, {"bias": a[2]}, what + " hg")
    Fd = acc.shape[1] // 2
    h, gate = d(out[0])[:, :Fd], d(out[0])[:, Fd:]  # the product reads the kernel's own rounded hg
    ref = h * gelu(gate).to(torch.float32).to(BF).to(F64)
    within(out[1], ref, GELU_ATOL * h.abs(), what + " act")
    return [hg, ref]


def chk_wgrad(a, kw, out, what):
    dy, x = a[0], a[1]
    ref, s = sums(dy.t(), x.t())
    within(out[0], ref, dy.shape[0] * FP32_U * s, what, "grad")
    return [ref]


def chk_colsum(a, kw, out, what):
    x = d(a[0])
    within(out[0], x.sum(0), x.shape[0] * FP32_U * x.abs().sum(0), what, "grad")
    return [x.sum(0)]


def chk_colsum_per_image(a, kw, out, what):
    x = a[0]
    per, tot = colsum_per_image(x)
    aper, atot = colsum_per_image(x.abs())
    n = x.numel() // (x.shape[0] * x.shape[-1])
    within(out[0], per, n * FP32_U * aper, what + " per image")
    within(out[1], tot, x.shape[0] * n * FP32_U * atot, what + " total", "grad")
    return [per, tot]


def _norm_stats(xg, mean, what):
    """xg: float64 [..., G, K] (K the elements of a group); checks the kernel's mean [..., G] (a K-term sum) against float64 and
    returns the two-pass variance.  The callers hold rstd to c = 4 on its K-term sum of squares: room for a shifted one-pass sum,
    whose error grows with mean((x - shift)^2) / var, about 2 for a shift inside the data."""
    K = xg.shape[-1]
    mu = xg.mean(-1)
    var = ((xg - mu[..., None]) ** 2).mean(-1)
    within(mean, mu, K * FP32_U * xg.abs().mean(-1) + FP32_U * mu.abs(), what + " mean", "f32")
    return var


def chk_layernorm_bf16_fwd(a, kw, out, what):
    x, g, b, eps = d(a[0]), d(a[1]), d(a[2]), a[3]
    y, mean, rstd = out
    var = _norm_stats(x[:, None, :], mean[:, None], what)[:, 0]
    r64 = (var + eps).rsqrt()
    within(rstd, r64, (4 * x.shape[1] + C_EW) * FP32_U * r64, what + " rstd", "f32")
    m, r = d(mean)[:, None], d(rstd)[:, None]  # y on the kernel's own statistics
    ref = (x - m) * r * g + b
    within(y, ref, C_EW * FP32_U * ((x.abs() + m.abs()) * r * g.abs() + b.abs()), what + " y")
    return [ref, None, None]


def _ln_grad(dy, xh, dxh, r, K):
    """LayerNorm's input gradient r (dy - mean(dy) - xh mean(dy xh)) over the last dim (dy already times gamma), with its fp32
    error: C_EW u per element, K u on the two K-term means, and the error dxh of the fp32 xh."""
    A, Bm = dy.mean(-1, keepdim=True), (dy * xh).mean(-1, keepdim=True)
    ref = r * (dy - A - xh * Bm)
    mA, mB = dy.abs().mean(-1, keepdim=True), (dy * xh).abs().mean(-1, keepdim=True)
    err = r * (C_EW * FP32_U * (dy.abs() + mA + xh.abs() * mB) + K * FP32_U * (mA + xh.abs() * mB)
               + dxh * Bm.abs() + xh.abs() * (dy.abs() * dxh).mean(-1, keepdim=True))
    return ref, err


def chk_layernorm_bf16_bwd(a, kw, out, what):
    dy, x, g, mean, rstd = (d(t) for t in a[:5])
    dres = kw.get("dres")
    dx, dgamma, dbeta = out
    K = x.shape[1]
    m, r = mean[:, None], rstd[:, None]
    xh = (x - m) * r
    dxh = 2 * FP32_U * (x.abs() + m.abs()) * r
    lng, err = _ln_grad(dy * g, xh, dxh, r, K)
    if dres is None:
        ref = lng
    else:  # bf16(dres + bf16(LN'(dy))): the LayerNorm gradient is rounded before the bf16 residual add, as eager's
        ref, err = lng + d(dres), U16 * (lng.abs() + err) + err
    within(dx, ref, err, what + " dx")
    R = x.shape[0]
    gref, bref = (dy * xh).sum(0), dy.sum(0)
    within(dgamma, gref, R * FP32_U * (dy * xh).abs().sum(0) + (dy.abs() * dxh).sum(0), what + " dgamma", "f32")
    within(dbeta, bref, R * FP32_U * dy.abs().sum(0), what + " dbeta", "f32")
    return [ref, gref, bref]


def _groups(t, C):
    B = t.shape[0]
    return d(t).reshape(B, -1, 32, C // 32).permute(0, 2, 1, 3).reshape(B, 32, -1)  # [B, 32, HW Cg]


def _ungroup(t, shape):
    B, HW, C = shape
    return t.reshape(B, 32, HW, C // 32).permute(0, 2, 1, 3).reshape(B, HW, C)


def chk_groupnorm_silu_fwd(a, kw, out, what):
    x, g, b, eps = a[0], d(a[1]), d(a[2]), a[3]
    silu = kw.get("silu", True)
    y, mean, rstd = out
    B, HW, C = x.shape
    xg = _groups(x, C)
    var = _norm_stats(xg, mean, what)
    r64 = (var + eps).rsqrt()
    within(rstd, r64, (4 * xg.shape[-1] + C_EW) * FP32_U * r64, what + " rstd", "f32")
    m, r = _ungroup(d(mean)[..., None].expand(xg.shape), x.shape), _ungroup(d(rstd)[..., None].expand(xg.shape), x.shape)
    xd = d(x)
    z = (xd - m) * r * g + b  # on the kernel's own statistics
    ez = C_EW * FP32_U * ((xd.abs() + m.abs()) * r * g.abs() + b.abs())
    ref, err = z, ez
    if silu:  # |silu'| <= 1.1
        ref, err = F.silu(z), 1.1 * ez + C_EW * FP32_U * F.silu(z).abs()
    within(y, ref, err, what + " y")
    return [ref, None, None]


def chk_groupnorm_silu_bwd(a, kw, out, what):
    x, dy, g, b, mean, rstd = a[:6]
    silu = kw.get("silu", True)
    dx, dgamma, dbeta = out
    B, HW, C = x.shape
    shape = x.shape
    xd, dyd, g, b = d(x), d(dy), d(g), d(b)
    ex = lambda s: _ungroup(d(s)[..., None].expand(B, 32, HW * C // 32), shape)  # noqa: E731
    m, r = ex(mean), ex(rstd)
    xh = (xd - m) * r
    dxh = 2 * FP32_U * (xd.abs() + m.abs()) * r
    dz, edz = dyd, torch.zeros_like(dyd)
    if silu:  # dz = dy silu'(z) with z recomputed in fp32: |silu''| <= 0.5
        z = xh * g + b
        sg = torch.sigmoid(z)
        sp = sg * (1 + z * (1 - sg))
        ez = C_EW * FP32_U * ((xd.abs() + m.abs()) * r * g.abs() + b.abs())
        dz, edz = dyd * sp, dyd.abs() * (C_EW * FP32_U * sp.abs() + 0.5 * ez)
    gd = dz * g
    K = HW * C // 32
    lng, err = _ln_grad(_groups(gd, C), _groups(xh, C), _groups(dxh, C), _groups(r, C), K)
    egd = _groups(edz * g.abs(), C)
    rr = _groups(r, C)
    err = err + rr * (egd + egd.mean(-1, keepdim=True) + _groups(xh, C).abs() * (egd * _groups(xh, C).abs()).mean(-1, keepdim=True))
    ref = _ungroup(lng, shape)
    within(dx, ref, _ungroup(err, shape), what + " dx")
    n = B * HW
    gref, bref = (dz * xh).sum((0, 1)), dz.sum((0, 1))
    within(dgamma, gref, n * FP32_U * (dz * xh).abs().sum((0, 1)) + (edz * xh.abs() + dz.abs() * dxh).sum((0, 1)), what + " dgamma", "f32")
    within(dbeta, bref, n * FP32_U * dz.abs().sum((0, 1)) + edz.sum((0, 1)), what + " dbeta", "f32")
    return [ref, gref, bref]


def unpack(wp):
    """The kernels' packed [Cout, 9 Cin] (tap-major) -> [Cout, Cin, 3, 3]."""
    co = wp.shape[0]
    return wp.reshape(co, 3, 3, -1).permute(0, 3, 1, 2)


def _rows_image(B, n):
    return torch.arange(B, device="cuda").repeat_interleave(n)


def chk_conv3x3(a, kw, out, what):
    x, wp = a[0], a[1]
    kw = dict(kw, bias=a[2] if len(a) > 2 else kw.get("bias"))
    w = unpack(wp)
    B, H, W, Cin = x.shape
    acc, s = conv3x3(x, w), conv3x3(d(x).abs(), d(w).abs())
    return [_epilogue(out[0].reshape(acc.shape), acc, 9 * Cin * FP32_U * s, kw, what, rows=_rows_image(B, H * W))]


def chk_conv3x3_wgrad(a, kw, out, what):
    dy, x = a[0], a[1]
    dyr = dy.reshape(-1, dy.shape[-1])
    ref, s = conv3x3_wgrad(dyr, x), conv3x3_wgrad(d(dyr).abs(), d(x).abs())
    within(out[0], ref, dyr.shape[0] * FP32_U * s, what, "grad")
    return [ref]


def _resample(fn, a, kw, out, what):
    x, wp = a[0], a[1]
    w = unpack(wp)
    acc, s = fn(x, w), fn(d(x).abs(), d(w).abs())
    B, Ho, Wo, Cout = acc.shape
    ref = _epilogue(out[0].reshape(-1, Cout), acc.reshape(-1, Cout), 9 * x.shape[3] * FP32_U * s.reshape(-1, Cout), kw, what,
                    rows=_rows_image(B, Ho * Wo))
    return [ref]


def chk_conv3x3_s2(a, kw, out, what):
    return _resample(conv3x3_s2, a, kw, out, what)


def chk_conv3x3_up2(a, kw, out, what):
    return _resample(conv3x3_up2, a, kw, out, what)


def chk_conv3x3_s2_wgrad(a, kw, out, what):
    dy, x = a[0], a[1]
    ref, s = conv3x3_s2_wgrad(dy, x), conv3x3_s2_wgrad(d(dy).abs(), d(x).abs())
    within(out[0], ref, dy.shape[0] * dy.shape[1] * dy.shape[2] * FP32_U * s, what, "grad")
    return [ref]


def chk_conv3x3_s2_dgrad(a, kw, out, what):
    dy, wd = a[0], a[1]
    Cout = dy.shape[3]
    w = torch.empty(Cout, wd.shape[0], 3, 3, dtype=wd.dtype, device=wd.device)
    for j, (ky, kx) in enumerate(ops._S2_DGRAD_TAPS):  # the inverse of pack_conv3x3_weight_s2_dgrad
        w[:, :, ky, kx] = wd[:, j * Cout:(j + 1) * Cout].t()
    B, h, ww, _ = dy.shape
    ref = conv3x3_s2_dgrad(dy, w, 2 * h, 2 * ww)
    s = conv3x3_s2_dgrad(d(dy).abs(), d(w).abs(), 2 * h, 2 * ww)
    within(out[0], ref, 4 * Cout * FP32_U * s, what)  # at most 4 taps per parity class
    return [ref]


def chk_upsample_nearest2x(a, kw, out, what):
    ref = a[0].repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert torch.equal(out[0], ref), what
    return [d(ref)]


def chk_sum2x2(a, kw, out, what):
    x = d(a[0])
    B, H2, W2, C = x.shape
    q = x.reshape(B, H2 // 2, 2, W2 // 2, 2, C)
    ref = q.sum((2, 4))
    within(out[0], ref, 3 * FP32_U * q.abs().sum((2, 4)), what)
    return [ref]


def _heads(q, k, v, dout, o, B, H, what):
    """attention_bounds_rows one head at a time (a float64 [B, Tq, Tk] per head fits at 64 x 64); yields (h, cols, refs, tols)."""
    L = q.shape[1]
    Dh = L // H
    for h in range(H):
        c = slice(h * Dh, (h + 1) * Dh)
        refs, tols = attention_bounds_rows(q[:, c], k[:, c], v[:, c], dout[:, c], B, 1, Dh ** -0.5, False, o[:, c])
        yield h, c, refs, tols


def chk_cross_attention_fwd(a, kw, out, what):
    q, k, v, B, H = a[:5]
    o, lse = out
    ref = torch.empty(o.shape, dtype=F64, device=o.device)
    for h, c, (o64, lse64, *_), (tol_o, *_) in _heads(q, k, v, torch.zeros_like(o), o, B, H, what):
        g = d(o[:, c])
        bad = ~((g - o64).abs() <= tol_o)
        assert not bad.any(), f"{what} out head {h}: {bad.sum().item()} elements outside the attention bound"
        REPORT.ratio(((g - o64).abs() / tol_o).max().item(), what + " out")
        # lse: as test_attention_elementwise_gpu holds it, 1e-4 of (1 + |lse|)
        within(lse[:, h], lse64[:, 0], 1e-4 * (1 + lse64[:, 0].abs()), what + f" lse head {h}", "f32")
        ref[:, c] = o64
    return [ref, None]


def chk_cross_attention_bwd(a, kw, out, what):
    q, k, v, o, do, lse, B, H = a[:8]
    refs = [torch.empty(t.shape, dtype=F64, device=t.device) for t in out]
    for h, c, (_, _, dq, dk, dv), (_, tq, tk, tv) in _heads(q, k, v, do, o, B, H, what):
        for i, (name, ref, tol) in enumerate((("dq", dq, tq), ("dk", dk, tk), ("dv", dv, tv))):
            g = d(out[i][:, c])
            bad = ~((g - ref).abs() <= tol)
            assert not bad.any(), f"{what} {name} head {h}: {bad.sum().item()} elements outside the attention bound"
            REPORT.ratio(((g - ref).abs() / tol).max().item(), f"{what} {name}")
            refs[i][:, c] = ref
    return refs


# the torch glue between kernels: eager's own ops on the same tensors
def glue_silu(x):
    return F.silu(x)


def glue_silu_bwd(dy, x):
    return torch.ops.aten.silu_backward(dy, x)


def glue_add(a, b):
    return a + b


def chk_glue_silu(a, kw, out, what):
    x = d(a[0])
    ref = F.silu(x)
    within(out[0], ref, C_EW * FP32_U * (ref.abs() + x.abs()), what)
    return [ref]


def chk_glue_silu_bwd(a, kw, out, what):
    dy, x = d(a[0]), d(a[1])
    s = torch.sigmoid(x)
    ref = dy * s * (1 + x * (1 - s))
    within(out[0], ref, C_EW * FP32_U * dy.abs() * (1 + x.abs()), what)
    return [ref]


def chk_glue_add(a, kw, out, what):
    ref = d(a[0]) + d(a[1])
    within(out[0], ref, 0.0 * ref, what)
    return [ref]


CHECKS: Dict[str, Callable] = {n[4:]: f for n, f in globals().items() if n.startswith("chk_")}
GLUE: Dict[str, Callable] = {"glue_silu": glue_silu, "glue_silu_bwd": glue_silu_bwd, "glue_add": glue_add}


# ---- op tables ---------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Out:
    """An output buffer the call fills: fp32 / bf16 of ``shape``, or (``packed``) columns [lo, hi) of a packed buffer."""
    shape: Tuple[int, ...]
    dtype: torch.dtype = torch.float32
    packed: Optional[Tuple[str, int, int, int]] = None  # (env key of the buffer, its width, lo, hi)

    def make(self, env):
        if self.packed is None:
            return torch.empty(self.shape, dtype=self.dtype, device="cuda")
        key, width, lo, hi = self.packed
        if key not in env:
            env[key] = torch.empty((self.shape[0], width), dtype=self.dtype, device="cuda")
        return env[key][:, lo:hi]


@dataclass
class Row:
    """One call: ``name`` (an ``ops`` entry point, or glue_*), its arguments (str: an env key; callable: f(env); Out: a buffer;
    anything else: a value the call must get as is), the env keys of its results (None: not kept) and, per result, eager's value
    of it: f(E, G) on the oracle's boundary values / gradients."""
    name: str
    args: tuple
    kw: Dict[str, Any]
    outs: Tuple[Optional[str], ...]
    eager: Dict[str, Callable] = field(default_factory=dict)
    rule: Any = TOL

    @property
    def glue(self) -> bool:
        return self.name.startswith("glue_")


def R(name, *args, outs, eager=None, rule=TOL, **kw):
    return Row(name, args, kw, tuple(outs), eager or {}, rule)


def resolve(src, env):
    if isinstance(src, str):
        return env[src]
    if callable(src):
        return src(env)
    if isinstance(src, Out):
        return src.make(env)
    return src


def V(key, *shape):
    """env[key] viewed as ``shape``."""
    return lambda env: env[key].reshape(*shape)


def cat(*keys):
    return lambda env: torch.cat([env[k] for k in keys], 1)


def call_row(r, a, kw):
    fn = GLUE[r.name] if r.glue else getattr(ops, r.name)
    res = fn(*a, **kw)
    return res if isinstance(res, tuple) else (res,)


def teacher_forced(rows, env, E, G, tag):
    """Run every row on eager's inputs (see the module docstring); returns the rows held to the 2x-eager bound."""
    twice = []
    for r in rows:
        a = [resolve(s, env) for s in r.args]
        kw = {k: resolve(s, env) for k, s in r.kw.items()}
        out = call_row(r, a, kw)
        what = f"{tag} {r.name} -> {','.join(o for o in r.outs if o)}"
        refs = CHECKS[r.name](a, kw, out, what)
        for name, o, ref in zip(r.outs, out, refs):
            if name is None:
                continue
            env[name] = o
            if name not in r.eager:
                continue
            e = r.eager[name](E, G)
            e = e.to(o.dtype).reshape(o.shape).contiguous()
            err = relerr(o, e)
            if r.rule == TWICE:
                bound = 2 * relerr(e.reshape(ref.shape), ref)
                twice.append(f"{r.name} -> {name}")
            elif r.rule == "attn":
                # eager's SDPA rounds the probabilities to bf16 as ours does, at other points: two independent bf16-P noises.  At
                # the SD head dims (40, 80, 160) each is ~1.7e-3 of float64, so the two are ~2.4e-3 apart; then the bound is
                # 2 x relerr(eager, float64), and every element is within the float64 attention bound above in any case
                bound = max(TOL_ATTN, 2 * relerr(e.reshape(ref.shape), ref))
            else:
                bound = r.rule
            REPORT.eager.append((f"{tag} {name}", err, bound, str(r.rule)))
            assert err <= bound, (f"{what}: {name} is {err:.3e} from eager's, over {bound:.3e} ({r.rule}); float64 is "
                                  f"{relerr(o, ref):.3e} from ours, {relerr(e.reshape(ref.shape), ref):.3e} from eager's")
            env[name] = e
    return twice


@dataclass
class Call:
    name: str
    args: list
    kw: dict
    out: tuple


class Recorder:
    """Stands in for ``ops`` in the module files: logs each kernel call's name, arguments (a copy, as they were when called) and
    outputs, then calls through; everything else is ``ops``' own."""

    def __init__(self) -> None:
        self.calls: List[Call] = []

    def __getattr__(self, name):
        real = getattr(ops, name)
        if name not in KERNELS:
            return real

        def rec(*args, **kw):
            snap = lambda v: v.detach().clone() if torch.is_tensor(v) else v  # noqa: E731
            a, k = [snap(v) for v in args], {n: snap(v) for n, v in kw.items()}
            res = real(*args, **kw)
            outs = res if isinstance(res, tuple) else (res,)
            self.calls.append(Call(name, a, k, tuple(o.detach().clone() for o in outs)))
            return res
        return rec


def _same_arg(got, src, env, what):
    if isinstance(src, Out):
        assert torch.is_tensor(got) and tuple(got.shape) == tuple(src.shape) and got.dtype == src.dtype, what
        return
    if isinstance(src, str) or callable(src):
        want = resolve(src, env)
        assert torch.is_tensor(got), what
        assert tuple(got.shape) == tuple(want.shape) and got.dtype == want.dtype, \
            f"{what}: {tuple(got.shape)} {got.dtype}, the table's source is {tuple(want.shape)} {want.dtype}"
        assert torch.equal(got, want), f"{what}: not the tensor the table says feeds it"
        return
    assert not torch.is_tensor(got) and got == src and type(got) is type(src), f"{what}: {got!r}, the table has {src!r}"


def wiring(rows, env, calls, tag):
    """Check a module's recorded calls against its op table (see the module docstring); fills ``env`` with the recorded outputs."""
    table = [r.name for r in rows if not r.glue]
    assert [c.name for c in calls] == table, f"{tag}: the module called {[c.name for c in calls]}, the table is {table}"
    it = iter(calls)
    for r in rows:
        what = f"{tag} {r.name} -> {','.join(o for o in r.outs if o)}"
        if r.glue:
            a = [resolve(s, env) for s in r.args]
            kw = {}
            out = call_row(r, a, kw)
        else:
            c = next(it)
            assert len(c.args) == len(r.args) and set(c.kw) == set(r.kw), \
                f"{what}: called with {len(c.args)} arguments and keywords {sorted(c.kw)}, the table has {len(r.args)} and {sorted(r.kw)}"
            for i, (got, src) in enumerate(zip(c.args, r.args)):
                _same_arg(got, src, env, f"{what}: argument {i}")
            for k, src in r.kw.items():
                _same_arg(c.kw[k], src, env, f"{what}: {k}=")
            a, kw, out = c.args, c.kw, c.out
        CHECKS[r.name](a, kw, out, what)
        for name, o in zip(r.outs, out):
            if name is not None:
                env[name] = o


# ---- layouts -----------------------------------------------------------------------------------------------------------------
def nhwc(t):
    """[B, C, H, W] -> contiguous [B, H, W, C]."""
    return t.permute(0, 2, 3, 1).contiguous()


def rows_(t):
    return t.reshape(-1, t.shape[-1])


def bf(t):
    return t.detach().to(BF).contiguous()


def pack(w):
    return ops.pack_conv3x3_weight(w)


# ---- the tables --------------------------------------------------------------------------------------------------------------
def res_block_table(B, H, W, Cin, Cout, tdim, eps=1e-5):
    """ResidualBlockWithTimeEmbeddingB200: res_block_fwd then res_block_bwd (unet_blocks.py).  env: x [B, H, W, Cin], time [B, tdim],
    dout [B, H, W, Cout] and the cast parameters (see ``res_block_env``)."""
    HW, M = H * W, B * H * W
    sc = Cin != Cout
    P = lambda k: lambda E, G: G["p:" + k]  # noqa: E731  eager's gradient of a parameter
    pk = lambda k: lambda E, G: pack(G["p:" + k])  # noqa: E731
    n = lambda k, val=True: (lambda E, G: nhwc((E if val else G)[k]))  # noqa: E731
    rows = [
        R("groupnorm_silu_fwd", V("x", B, HW, Cin), "g1", "be1", eps, outs=("y1", "m1", "r1"), eager={"y1": n("silu1")}),
        R("glue_silu", "time", outs=("ta",), eager={"ta": lambda E, G: E["time_silu"]}),
        R("gemm", "ta", "wt", bias="bt", outs=("t",), eager={"t": lambda E, G: E["t"]}),
        # conv1 adds its bias in fp32 and rounds once, eager rounds the product and adds the bias in a second bf16 op
        R("conv3x3", V("y1", B, H, W, Cin), "w1p", "b1", epilogue=ops.EPI_BIAS_ADD_PER_IMAGE_BF16, aux="t", outs=("h",),
          eager={"h": n("h")}, rule=TWICE),
        R("groupnorm_silu_fwd", V("h", B, HW, Cout), "g2", "be2", eps, outs=("y2", "m2", "r2"), eager={"y2": n("silu2")}),
    ]
    if sc:  # the same bias rounding as conv1
        rows.append(R("gemm", V("x", M, Cin), "ws", bias="bs", outs=("inp",), eager={"inp": n("shortcut")}, rule=TWICE))
    rows += [
        R("conv3x3", V("y2", B, H, W, Cout), "w2p", "b2", epilogue=ops.EPI_BIAS_RESID_CLAMP_BF16, aux="inp" if sc else "x",
          outs=("out",), eager={"out": n("out")}, rule=TWICE),
        # backward: the clamp is the identity (eager's too: no sum overflows here)
        R("conv3x3_wgrad", "dout", V("y2", B, H, W, Cout), outs=("dw2p",), eager={"dw2p": pk("conv2.weight")}),
        R("colsum", V("dout", M, Cout), Out((Cout,)), outs=("db2",), eager={"db2": P("conv2.bias")}),
        R("conv3x3", "dout", "w2d", outs=("dy2",), eager={"dy2": n("silu2", False)}),
        R("groupnorm_silu_bwd", V("h", B, HW, Cout), V("dy2", B, HW, Cout), "g2", "be2", "m2", "r2", outs=("dh", "dg2", "dbe2"),
          eager={"dh": n("h", False), "dg2": P("norm2.weight"), "dbe2": P("norm2.bias")}),
        R("colsum_per_image", "dh", outs=("dt", "db1"), eager={"dt": lambda E, G: G["t"], "db1": P("conv1.bias")}),
        R("conv3x3_wgrad", V("dh", B, H, W, Cout), V("y1", B, H, W, Cin), outs=("dw1p",), eager={"dw1p": pk("conv1.weight")}),
        R("conv3x3", V("dh", B, H, W, Cout), "w1d", outs=("dy1",), eager={"dy1": n("silu1", False)}),
        R("groupnorm_silu_bwd", V("x", B, HW, Cin), V("dy1", B, HW, Cin), "g1", "be1", "m1", "r1", outs=("dxg", "dg1", "dbe1"),
          eager={"dxg": n("x_gn", False), "dg1": P("norm1.weight"), "dbe1": P("norm1.bias")}),
    ]
    if sc:
        rows += [
            R("wgrad", V("dout", M, Cout), V("x", M, Cin), Out((Cout, Cin)), outs=("dws",),
              eager={"dws": lambda E, G: G["p:shortcut.weight"].reshape(Cout, Cin)}),
            R("gemm", V("dout", M, Cout), "ws", b_mn_major=True, outs=("dsc",), eager={"dsc": n("x_sc", False)}),
        ]
    rows += [
        R("glue_add", V("dxg", M, Cin), "dsc" if sc else V("dout", M, Cout), outs=("dx",), eager={"dx": n("x", False)}),
        R("wgrad", "dt", "ta", Out((Cout, tdim)), outs=("dwt",), eager={"dwt": P("time_embedding.weight")}),
        R("colsum", "dt", Out((Cout,)), outs=("dbt",), eager={"dbt": P("time_embedding.bias")}),
        R("gemm", "dt", "wt", b_mn_major=True, outs=("dta",), eager={"dta": lambda E, G: G["time_silu"]}),
        R("glue_silu_bwd", "dta", "time", outs=("dtime",), eager={"dtime": lambda E, G: G["time"]}),
    ]
    return rows


def res_block_env(sd, x, time, dout):
    """The table's sources for the module inputs (channels-last bf16) and the parameters as the module casts them."""
    f = lambda k: sd[k].to("cuda").float().contiguous()  # noqa: E731
    b = lambda k: bf(sd[k].to("cuda"))  # noqa: E731
    env = {"x": x, "time": time, "dout": dout, "g1": f("norm1.weight"), "be1": f("norm1.bias"), "g2": f("norm2.weight"),
           "be2": f("norm2.bias"), "b1": b("conv1.bias"), "b2": b("conv2.bias"), "wt": b("time_embedding.weight"),
           "bt": b("time_embedding.bias")}
    for i in (1, 2):
        w = sd[f"conv{i}.weight"].to("cuda")
        env[f"w{i}p"], env[f"w{i}d"] = ops.pack_conv3x3_weight(w), ops.pack_conv3x3_weight_dgrad(w)
    if "shortcut.weight" in sd:
        w = sd["shortcut.weight"]
        env["ws"], env["bs"] = bf(w.reshape(w.shape[0], -1).to("cuda")), b("shortcut.bias")
    return env


def attention_fwd_table(p, e, B, heads, L, x, c, resid, out, out_eager):
    """attention_forward (attention.py) on env[x] [B Tq, Dq] and env[c] [B Tk, Dc] (None: self-attention); ``resid``: the env key
    of the bf16 residual its out_linear adds.  ``p``: the env prefix of its keys; ``e``: eager's key prefix of the
    CrossAttention's boundaries; ``out_eager``: eager's value of the output."""
    E_ = lambda k: lambda E, G: rows_(E[e + k])  # noqa: E731
    rows = []
    if c is None:
        rows.append(R("gemm", x, p + "wqkv", outs=(p + "qkv",),
                      eager={p + "qkv": lambda E, G: torch.cat([rows_(E[e + k]) for k in "qkv"], 1)}))
        q, k, v = (lambda env, i=i: env[p + "qkv"][:, i * L:(i + 1) * L] for i in range(3))
    else:
        rows.append(R("gemm", x, p + "wq", outs=(p + "q",), eager={p + "q": E_("q")}))
        rows.append(R("gemm", c, p + "wkv", outs=(p + "kv",), eager={p + "kv": lambda E, G: torch.cat([rows_(E[e + "k"]), rows_(E[e + "v"])], 1)}))
        q = p + "q"
        k, v = (lambda env, i=i: env[p + "kv"][:, i * L:(i + 1) * L] for i in range(2))
    rows.append(R("cross_attention_fwd", q, k, v, B, heads, outs=(p + "o", p + "lse"), eager={p + "o": E_("attn")}, rule="attn"))
    if resid is None:
        rows.append(R("gemm", p + "o", p + "wo", bias=p + "bo", outs=(out,), eager={out: out_eager}))
    else:  # eager: bf16(bf16(out_linear) + resid), as ours
        rows.append(R("gemm", p + "o", p + "wo", bias=p + "bo", epilogue=ops.EPI_BIAS_RESID_BF16, aux=resid, outs=(out,),
                      eager={out: out_eager}))
    return rows


def attention_bwd_table(p, e, B, heads, L, Tq, Tk, Dq, Dc, x, c, dy, dx, dc, dx_eager, dc_eager):
    """attention_backward on the upstream gradient env[dy] of the forward on env[x] / env[c]; writes env[dx] (and env[dc] for
    cross-attention), whose eager values are ``dx_eager`` / ``dc_eager``.  The packed input
    gradients (self-attention's dx, cross-attention's dcontext) sum their two or three products in fp32 and round once, where eager
    rounds each and adds them: held to the 2x-eager bound."""
    Ge = lambda k: lambda E, G: rows_(G[e + k])  # noqa: E731
    Pg = lambda *ks: lambda E, G: torch.cat([G["p:" + e + k] for k in ks], 0)  # noqa: E731
    M, Mk = B * Tq, B * Tk
    rows = [
        R("wgrad", dy, p + "o", Out((Dq, L)), outs=(p + "dwo",), eager={p + "dwo": Pg("out_linear.0.weight")}),
        R("colsum", dy, Out((Dq,)), outs=(p + "dbo",), eager={p + "dbo": Pg("out_linear.0.bias")}),
        R("gemm", dy, p + "wo", b_mn_major=True, outs=(p + "do",), eager={p + "do": Ge("attn")}),
    ]
    if c is None:
        q, k, v = (lambda env, i=i: env[p + "qkv"][:, i * L:(i + 1) * L] for i in range(3))
        bufs = [Out((M, L), BF, (p + "dqkv_buf", 3 * L, i * L, (i + 1) * L)) for i in range(3)]
        rows += [
            R("cross_attention_bwd", q, k, v, p + "o", p + "do", p + "lse", B, heads, dq=bufs[0], dk=bufs[1], dv=bufs[2],
              outs=(p + "dq", p + "dk", p + "dv"), eager={p + "dq": Ge("q"), p + "dk": Ge("k"), p + "dv": Ge("v")}, rule="attn"),
            R("wgrad", cat(p + "dq", p + "dk", p + "dv"), x, Out((3 * L, Dq)), outs=(p + "dw",),
              eager={p + "dw": Pg("to_q.weight", "to_k.weight", "to_v.weight")}),
            R("gemm", cat(p + "dq", p + "dk", p + "dv"), p + "wqkv", b_mn_major=True, outs=(dx,), eager={dx: dx_eager}, rule=TWICE),
        ]
    else:
        q = p + "q"
        k, v = (lambda env, i=i: env[p + "kv"][:, i * L:(i + 1) * L] for i in range(2))
        bufs = [Out((Mk, L), BF, (p + "dkv_buf", 2 * L, i * L, (i + 1) * L)) for i in range(2)]
        rows += [
            R("cross_attention_bwd", q, k, v, p + "o", p + "do", p + "lse", B, heads, dq=Out((M, L), BF), dk=bufs[0], dv=bufs[1],
              outs=(p + "dq", p + "dk", p + "dv"), eager={p + "dq": Ge("q"), p + "dk": Ge("k"), p + "dv": Ge("v")}, rule="attn"),
            R("wgrad", p + "dq", x, Out((L, Dq)), outs=(p + "dwq",), eager={p + "dwq": Pg("to_q.weight")}),
            R("wgrad", cat(p + "dk", p + "dv"), c, Out((2 * L, Dc)), outs=(p + "dwkv",), eager={p + "dwkv": Pg("to_k.weight", "to_v.weight")}),
            R("gemm", p + "dq", p + "wq", b_mn_major=True, outs=(dx,), eager={dx: dx_eager}),
            R("gemm", cat(p + "dk", p + "dv"), p + "wkv", b_mn_major=True, outs=(dc,), eager={dc: dc_eager}, rule=TWICE),
        ]
    return rows


def res_block_finals(Cin, Cout):
    """The module's results -> the env values they must equal bit for bit: (what, f(module tensors), f(env))."""
    sc = Cin != Cout
    g = lambda k: (lambda m: m["p:" + k])  # noqa: E731
    out = [("out", lambda m: nhwc(m["out"]), "out"), ("dx", lambda m: nhwc(m["x"]), "dx"), ("dtime", lambda m: m["time"], "dtime"),
           ("norm1.weight", g("norm1.weight"), "dg1"), ("norm1.bias", g("norm1.bias"), "dbe1"),
           ("conv1.weight", g("conv1.weight"), lambda env: ops.unpack_conv3x3_weight(env["dw1p"], Cin)),
           ("conv1.bias", g("conv1.bias"), "db1"), ("time_embedding.weight", g("time_embedding.weight"), "dwt"),
           ("time_embedding.bias", g("time_embedding.bias"), "dbt"), ("norm2.weight", g("norm2.weight"), "dg2"),
           ("norm2.bias", g("norm2.bias"), "dbe2"),
           ("conv2.weight", g("conv2.weight"), lambda env: ops.unpack_conv3x3_weight(env["dw2p"], Cout)),
           ("conv2.bias", g("conv2.bias"), "db2")]
    if sc:  # the shortcut's bias gradient is conv2's: both are the column sums of dout
        out += [("shortcut.weight", g("shortcut.weight"), lambda env: env["dws"].view(Cout, Cin, 1, 1)),
                ("shortcut.bias", g("shortcut.bias"), "db2")]
    return out


def check_finals(finals, module, env, tag):
    for what, got, src in finals:
        a, b = got(module), resolve(src, env)
        assert a.numel() == b.numel() and a.dtype == b.dtype, f"{tag}: the module's {what} is {tuple(a.shape)} {a.dtype}"
        assert torch.equal(a.reshape(b.shape), b), f"{tag}: the module's {what} is not the table's"


def attention_env(sd, p, e, self_attn):
    """The cast parameters of the CrossAttention ``e`` (state-dict prefix) under env prefix ``p``, as attention_forward casts them."""
    w = lambda k: sd[e + k].to("cuda")  # noqa: E731
    env = {p + "wo": bf(w("out_linear.0.weight")), p + "bo": bf(w("out_linear.0.bias"))}
    if self_attn:
        env[p + "wqkv"] = bf(torch.cat([w("to_q.weight"), w("to_k.weight"), w("to_v.weight")], 0))
    else:
        env[p + "wq"], env[p + "wkv"] = bf(w("to_q.weight")), bf(torch.cat([w("to_k.weight"), w("to_v.weight")], 0))
    return env


def attention_finals(p, L, self_attn):
    g = lambda k: (lambda m: m["p:" + k])  # noqa: E731
    if self_attn:
        w = [(lambda env, i=i: env[p + "dw"][i * L:(i + 1) * L]) for i in range(3)]
    else:
        w = [p + "dwq"] + [(lambda env, i=i: env[p + "dwkv"][i * L:(i + 1) * L]) for i in range(2)]
    return [("to_q.weight", g("to_q.weight"), w[0]), ("to_k.weight", g("to_k.weight"), w[1]), ("to_v.weight", g("to_v.weight"), w[2]),
            ("out_linear.0.weight", g("out_linear.0.weight"), p + "dwo"), ("out_linear.0.bias", g("out_linear.0.bias"), p + "dbo")]


def spatial_transformer_table(B, H, W, C, heads, layers, Tk, Dc):
    """SpatialTransformerB200: _LatentIn, each block's _block_forward, _LatentOut, then their backwards in autograd's order
    (spatial_transformer.py, attention.py).  env: x [B, H, W, C], ctx [B Tk, Dc], dout [B, H, W, C] and ``spatial_transformer_env``."""
    HW, M, L, Fd = H * W, B * H * W, C, 4 * C
    Pg = lambda k: lambda E, G: G["p:" + k]  # noqa: E731
    Er = lambda k: lambda E, G: rows_(E[k])  # noqa: E731
    Gr = lambda k: lambda E, G: rows_(G[k])  # noqa: E731
    rows = [
        R("groupnorm_silu_fwd", V("x", B, HW, C), "gnw", "gnb", 1e-6, silu=False, outs=("yn", "gm", "gr"),
          eager={"yn": lambda E, G: nhwc(E["gn"])}),
        # the 1x1 convolutions add their bias in fp32 and round once, eager rounds the product and adds the bias in bf16
        R("gemm", V("yn", M, C), "w_in", bias="b_in", outs=("tok0",), eager={"tok0": Er("tokens")}, rule=TWICE),
    ]
    for i in range(layers):
        b, e = f"b{i}.", f"blocks.{i}."
        x0 = f"tok{i}"
        rows.append(R("layernorm_bf16_fwd", x0, b + "g1", b + "be1", 1e-5, outs=(b + "y1", b + "m1", b + "r1"), eager={b + "y1": Er(e + "ln1")}))
        rows += attention_fwd_table(b + "a1.", e + "attn1.", B, heads, L, b + "y1", None, x0, b + "x1", Er(e + "x1"))
        rows.append(R("layernorm_bf16_fwd", b + "x1", b + "g2", b + "be2", 1e-5, outs=(b + "y2", b + "m2", b + "r2"), eager={b + "y2": Er(e + "ln2")}))
        rows += attention_fwd_table(b + "a2.", e + "attn2.", B, heads, L, b + "y2", "ctx", b + "x1", b + "x2", Er(e + "x2"))
        rows += [
            R("layernorm_bf16_fwd", b + "x2", b + "g3", b + "be3", 1e-5, outs=(b + "y3", b + "m3", b + "r3"), eager={b + "y3": Er(e + "ln3")}),
            R("geglu", b + "y3", b + "w1", b + "fb1", outs=(b + "hg", b + "act"), eager={b + "hg": Er(e + "hg"), b + "act": Er(e + "prod")}),
            R("gemm", b + "act", b + "w2", bias=b + "fb2", epilogue=ops.EPI_BIAS_RESID_BF16, aux=b + "x2", outs=(f"tok{i + 1}",),
              eager={f"tok{i + 1}": Er(e + "out")}),
        ]
    n = f"tok{layers}"
    rows += [
        R("gemm", n, "w_out", bias="b_out", epilogue=ops.EPI_BIAS_RESID_BF16, aux=V("x", M, C), outs=("out",),
          eager={"out": lambda E, G: nhwc(E["out"])}, rule=TWICE),
        R("wgrad", V("dout", M, C), n, Out((C, L)), outs=("dw_out",), eager={"dw_out": lambda E, G: G["p:from_latent.weight"].reshape(C, L)}),
        R("colsum", V("dout", M, C), Out((C,)), outs=("db_out",), eager={"db_out": Pg("from_latent.bias")}),
        R("gemm", V("dout", M, C), "w_out", b_mn_major=True, outs=("d" + n,), eager={"d" + n: Gr(f"blocks.{layers - 1}.out")}),
    ]
    for i in reversed(range(layers)):
        b, e = f"b{i}.", f"blocks.{i}."
        dx3, x0 = f"dtok{i + 1}", f"tok{i}"
        rows += [
            R("wgrad", dx3, b + "act", Out((C, Fd)), outs=(b + "dw2",), eager={b + "dw2": Pg(e + "ff.net.2.linear.weight")}),
            R("colsum", dx3, Out((C,)), outs=(b + "db2",), eager={b + "db2": Pg(e + "ff.net.2.linear.bias")}),
            # GEGLU's three backward roundings (documented in spatial_transformer.py)
            R("gemm", dx3, b + "w2", b_mn_major=True, epilogue=ops.EPI_DGEGLU_BF16, aux=b + "hg", outs=(b + "dhg",),
              eager={b + "dhg": Gr(e + "hg")}, rule=TWICE),
            R("wgrad", b + "dhg", b + "y3", Out((2 * Fd, C)), outs=(b + "dw1",), eager={b + "dw1": Pg(e + "ff.net.0.net.weight")}),
            R("colsum", b + "dhg", Out((2 * Fd,)), outs=(b + "db1",), eager={b + "db1": Pg(e + "ff.net.0.net.bias")}),
            R("gemm", b + "dhg", b + "w1", b_mn_major=True, outs=(b + "dy3",), eager={b + "dy3": Gr(e + "ln3")}),
            # each LayerNorm gradient rounded to bf16 before the bf16 add of the residual's gradient (documented)
            R("layernorm_bf16_bwd", b + "dy3", b + "x2", b + "g3", b + "m3", b + "r3", dres=dx3, outs=(b + "dx2", b + "dg3", b + "dbe3"),
              eager={b + "dx2": Gr(e + "x2"), b + "dg3": Pg(e + "norm3.weight"), b + "dbe3": Pg(e + "norm3.bias")}, rule=TWICE),
        ]
        rows += attention_bwd_table(b + "a2.", e + "attn2.", B, heads, L, HW, Tk, C, Dc, b + "y2", "ctx", b + "dx2", b + "dy2", b + "dc",
                                    Gr(e + "ln2"), Gr(e + "context"))
        rows.append(R("layernorm_bf16_bwd", b + "dy2", b + "x1", b + "g2", b + "m2", b + "r2", dres=b + "dx2", outs=(b + "dx1", b + "dg2", b + "dbe2"),
                      eager={b + "dx1": Gr(e + "x1"), b + "dg2": Pg(e + "norm2.weight"), b + "dbe2": Pg(e + "norm2.bias")}, rule=TWICE))
        rows += attention_bwd_table(b + "a1.", e + "attn1.", B, heads, L, HW, HW, C, C, b + "y1", None, b + "dx1", b + "dy1", None,
                                    Gr(e + "ln1"), None)
        rows.append(R("layernorm_bf16_bwd", b + "dy1", x0, b + "g1", b + "m1", b + "r1", dres=b + "dx1", outs=(f"dtok{i}", b + "dg1", b + "dbe1"),
                      eager={f"dtok{i}": Gr("tokens" if i == 0 else f"blocks.{i - 1}.out"), b + "dg1": Pg(e + "norm1.weight"),
                             b + "dbe1": Pg(e + "norm1.bias")}, rule=TWICE))
    rows += [
        R("wgrad", "dtok0", V("yn", M, C), Out((L, C)), outs=("dw_in",), eager={"dw_in": lambda E, G: G["p:to_latent.weight"].reshape(L, C)}),
        R("colsum", "dtok0", Out((L,)), outs=("db_in",), eager={"db_in": Pg("to_latent.bias")}),
        R("gemm", "dtok0", "w_in", b_mn_major=True, outs=("dyn",), eager={"dyn": lambda E, G: nhwc(G["gn"])}),
        R("groupnorm_silu_bwd", V("x", B, HW, C), V("dyn", B, HW, C), "gnw", "gnb", "gm", "gr", silu=False, outs=("dxg", "dgnw", "dgnb"),
          eager={"dxg": lambda E, G: nhwc(G["x_gn"]), "dgnw": Pg("norm.weight"), "dgnb": Pg("norm.bias")}),
        # autograd adds x's two gradients (GroupNorm path, residual) and the blocks' context gradients, in bf16
        R("glue_add", V("dxg", M, C), V("dout", M, C), outs=("dx",), eager={"dx": lambda E, G: nhwc(G["x"])}),
    ]
    dc = "b0.dc"
    for i in range(1, layers):
        last = i == layers - 1  # eager's context gradient is the sum over all blocks
        rows.append(R("glue_add", f"b{i}.dc", dc, outs=(f"dctx{i}",), eager={f"dctx{i}": lambda E, G: rows_(G["context"])} if last else None))
        dc = f"dctx{i}"
    return rows, dc


def spatial_transformer_env(sd, layers, x, ctx, dout):
    f = lambda k: sd[k].to("cuda").float().contiguous()  # noqa: E731
    b = lambda k: bf(sd[k].to("cuda"))  # noqa: E731
    C = sd["norm.weight"].shape[0]
    env = {"x": x, "ctx": ctx, "dout": dout, "gnw": f("norm.weight"), "gnb": f("norm.bias"),
           "w_in": bf(sd["to_latent.weight"].reshape(C, -1).to("cuda")), "b_in": b("to_latent.bias"),
           "w_out": bf(sd["from_latent.weight"].reshape(C, -1).to("cuda")), "b_out": b("from_latent.bias")}
    for i in range(layers):
        p, e = f"b{i}.", f"blocks.{i}."
        for j in (1, 2, 3):
            env[p + f"g{j}"], env[p + f"be{j}"] = f(e + f"norm{j}.weight"), f(e + f"norm{j}.bias")
        env[p + "w1"], env[p + "fb1"] = b(e + "ff.net.0.net.weight"), b(e + "ff.net.0.net.bias")
        env[p + "w2"], env[p + "fb2"] = b(e + "ff.net.2.linear.weight"), b(e + "ff.net.2.linear.bias")
        env.update(attention_env(sd, p + "a1.", e + "attn1.", True))
        env.update(attention_env(sd, p + "a2.", e + "attn2.", False))
    return env


def spatial_transformer_finals(C, layers, dc):
    g = lambda k: (lambda m: m["p:" + k])  # noqa: E731
    out = [("out", lambda m: nhwc(m["out"]), "out"), ("dx", lambda m: nhwc(m["x"]), "dx"), ("dcontext", lambda m: rows_(m["context"]), dc),
           ("norm.weight", g("norm.weight"), "dgnw"), ("norm.bias", g("norm.bias"), "dgnb"),
           ("to_latent.weight", g("to_latent.weight"), lambda env: env["dw_in"].view(C, C, 1, 1)), ("to_latent.bias", g("to_latent.bias"), "db_in"),
           ("from_latent.weight", g("from_latent.weight"), lambda env: env["dw_out"].view(C, C, 1, 1)),
           ("from_latent.bias", g("from_latent.bias"), "db_out")]
    for i in range(layers):
        b, e = f"b{i}.", f"blocks.{i}."
        out += [(e + k, g(e + k), v) for k, v in (("ff.net.0.net.weight", b + "dw1"), ("ff.net.0.net.bias", b + "db1"),
                                                    ("ff.net.2.linear.weight", b + "dw2"), ("ff.net.2.linear.bias", b + "db2"),
                                                    ("norm1.weight", b + "dg1"), ("norm1.bias", b + "dbe1"), ("norm2.weight", b + "dg2"),
                                                    ("norm2.bias", b + "dbe2"), ("norm3.weight", b + "dg3"), ("norm3.bias", b + "dbe3"))]
        for a, self_attn in (("a1.", True), ("a2.", False)):
            name = "attn1." if self_attn else "attn2."
            out += [(e + name + w, (lambda m, k=e + name + w: m["p:" + k]), src) for w, _, src in attention_finals(b + a, C, self_attn)]
    return out


def resample_table(up, B, H, W, Cin, Cout):
    """ResDownsampleB200 / ResUpsampleB200: _DownsampleOp / _UpsampleOp (unet_blocks.py); H x W is the input's size.  env: x
    [B, H, W, Cin], dout (the output's shape), wp (packed weight), wd (the input-gradient packing), brows (bf16 bias per image)."""
    w = "conv." if up else "net."
    Pg = lambda k: lambda E, G: G["p:" + w + k]  # noqa: E731
    out = "conv3x3_up2" if up else "conv3x3_s2"
    rows = [R(out, "x", "wp", epilogue=ops.EPI_BIAS_ADD_PER_IMAGE_BF16, aux="brows", outs=("out",), eager={"out": lambda E, G: nhwc(E["out"])})]
    db = R("colsum", V("dout", -1, Cout), Out((Cout,)), outs=("db",), eager={"db": Pg("bias")})
    dx = {"dx": lambda E, G: nhwc(G["x"])}
    if up:
        rows += [
            R("upsample_nearest2x", "x", outs=("xu",), eager={"xu": lambda E, G: nhwc(E["up"])}),
            R("conv3x3_wgrad", "dout", "xu", outs=("dwp",), eager={"dwp": lambda E, G: pack(G["p:conv.weight"])}),
            db,
            R("conv3x3", "dout", "wd", outs=("dxu",), eager={"dxu": lambda E, G: nhwc(G["up"])}),
            R("sum2x2", "dxu", outs=("dx",), eager=dx),
        ]
    else:
        rows += [
            R("conv3x3_s2_wgrad", "dout", "x", outs=("dwp",), eager={"dwp": lambda E, G: pack(G["p:net.weight"])}),
            db,
            R("conv3x3_s2_dgrad", "dout", "wd", outs=("dx",), eager=dx),
        ]
    return rows


def resample_env(sd, up, B, x, dout):
    w = "conv." if up else "net."
    weight = sd[w + "weight"].to("cuda")
    wd = ops.pack_conv3x3_weight_dgrad(weight) if up else ops.pack_conv3x3_weight_s2_dgrad(weight)
    return {"x": x, "dout": dout, "wp": ops.pack_conv3x3_weight(weight), "wd": wd,
            "brows": bf(sd[w + "bias"].to("cuda")).expand(B, -1).contiguous()}


def resample_finals(up, Cin):
    w = "conv." if up else "net."
    return [("out", lambda m: nhwc(m["out"]), "out"), ("dx", lambda m: nhwc(m["x"]), "dx"),
            ("weight", lambda m: m["p:" + w + "weight"], lambda env: ops.unpack_conv3x3_weight(env["dwp"], Cin)),
            ("bias", lambda m: m["p:" + w + "bias"], "db")]
