"""Memory footprint of every C-ABI kernel: each call writes exactly its outputs and reads nothing outside its inputs.

Every buffer a call sees is a ``Guarded`` allocation ``[front guard | rows x ld | back guard]`` whose view starts 16 mod 256
bytes (the ABI promises 16-byte alignment and no more).  Around outputs, the guards and the ``[width, ld)`` padding hold a
NaN payload no kernel produces (the kernels turn NaN into 0x7FFF when they round to bf16); around inputs they hold a different
NaN, so a report can tell "never written" from "read the poison".  After a call:
  - outputs: guards and padding are bit-identical, and no element of the view still holds the sentinel;
  - outputs the contract says are read (accumulate, in-place aux, caller-zeroed rows) equal the documented update;
  - inputs, guards included, are bit-identical, and no output holds a NaN;
  - workspaces are exactly the advertised size, NaN-filled, and the sentinel behind them survives;
  - every value matches a float64 CPU reference of the same operation.
Every case runs twice, the second time with a different sentinel, and both results must be bit-identical.

The calls go straight to the C-ABI (the ``ops`` wrappers pick leading dims and workspaces themselves).  The entry points of the
companion header include/b200_cflearn_ext.h have their cases beside their other tests (EXT_CASE_MODULES); the coverage check
imports those modules, so one ``@covers`` table spans both headers."""
import ctypes
import importlib
import math

import pytest
import torch
import torch.nn.functional as F

import cflearn_b200  # noqa: F401  (registers the package)
from cflearn_b200 import _cabi
from _refs import (adam, assert_ulp, attention_rows, bf16, conv3x3, conv3x3_wgrad, first_bad, gelu, gelu_grad, groupnorm, layernorm,
                   packed_attention, relerr, with_grads)

DEV = "cuda"
GUARD_BYTES = 65536

_BITS = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int32: torch.int32, torch.int64: torch.int64,
         torch.uint8: torch.uint8}
SENTINEL = {torch.bfloat16: 0x7FA5, torch.float32: 0x7FA5A5A5, torch.int32: 0x7FA5A5A5, torch.int64: 0x7FA5A5A5A5A5A5A5,
            torch.uint8: 0xA5}
SENTINEL2 = {torch.bfloat16: 0x7FA6, torch.float32: 0x7FA6A6A6, torch.int32: 0x7FA6A6A6, torch.int64: 0x7FA6A6A6A6A6A6A6,
             torch.uint8: 0xA6}
POISON = {torch.bfloat16: 0x7FC0, torch.float32: 0x7FC00000, torch.int32: 0x7FC00000, torch.int64: 0x7FC0000000000000,
          torch.uint8: 0xC0}


def rup(n, m=8):
    return (n + m - 1) // m * m


# ------------------------------------------------------------------------------------------------------------------------
# guarded buffers
# ------------------------------------------------------------------------------------------------------------------------
class Guarded:
    """One flat allocation [front guard | rows x ld | back guard]; ``view`` is [rows, width] with row stride ld, its base
    16 mod 256 bytes.  Both guards are at least 64 KB and the back guard at least ``back_rows`` rows of ld."""

    def __init__(self, rows, width, ld=None, dtype=torch.float32, device=DEV, back_rows=0):
        ld = width if ld is None else ld
        assert ld >= width and rows >= 1 and width >= 1
        es = torch.empty((), dtype=dtype).element_size()
        self.rows, self.width, self.ld, self.dtype = rows, width, ld, dtype
        body = rows * ld
        front_min = GUARD_BYTES // es
        back = max(GUARD_BYTES // es, back_rows * ld)
        self.flat = torch.empty(front_min + 256 // es + body + back, dtype=dtype, device=device)
        skew = (16 - (self.flat.data_ptr() + front_min * es)) % 256
        assert skew % es == 0
        self.front = front_min + skew // es
        self.bits = self.flat.view(_BITS[dtype])
        self.view = self.flat[self.front:self.front + body].view(rows, ld)[:, :width]
        inside = torch.zeros(self.flat.numel(), dtype=torch.bool, device=device)
        inside[self.front:self.front + body].view(rows, ld)[:, :width] = True
        self.inside = inside

    def ptr(self):
        return self.view.data_ptr()

    def fill_outside(self, pattern):
        keep = self.view.clone()
        self.bits.fill_(_as_signed(pattern, self.bits.dtype))
        self.view.copy_(keep)

    def fill_view_bits(self, pattern):
        self.view.view(_BITS[self.dtype]).fill_(_as_signed(pattern, self.bits.dtype))

    def where(self, flat_index):
        """(row, col) of a flat index relative to the view (negative rows: front guard; rows >= self.rows: back guard)."""
        return divmod(int(flat_index) - self.front, self.ld)

    def outside_changed(self, before):
        """First (row, col) outside the view whose bits differ from ``before`` (a ``bits`` snapshot), or None."""
        bad = (self.bits != before) & ~self.inside
        idx = torch.nonzero(bad)
        return None if idx.numel() == 0 else self.where(idx[0, 0])

    def unwritten(self, pattern):
        """First (row, col) of the view that still holds ``pattern``, or None."""
        hit = self.view.view(_BITS[self.dtype]) == _as_signed(pattern, self.bits.dtype)
        idx = torch.nonzero(hit)
        return None if idx.numel() == 0 else (int(idx[0, 0]), int(idx[0, 1]))


def _as_signed(pattern, bits_dtype):
    width = torch.iinfo(bits_dtype).bits
    if bits_dtype == torch.uint8:
        return pattern
    return pattern - (1 << width) if pattern >= 1 << (width - 1) else pattern


class Case:
    """The buffers of one C-ABI call.  ``run(launch)`` checks the footprint rules, runs a second time with another sentinel,
    and returns the CPU copies of every output by name."""

    def __init__(self, name):
        self.name = name
        self.bufs = []  # (kind, name, Guarded, prior)

    def _add(self, kind, name, g, prior=None):
        self.bufs.append((kind, name, g, prior))
        return g

    def input(self, name, data, ld=None):
        data = data.reshape(1, -1) if data.dim() == 1 else data.reshape(data.shape[0], -1)
        g = Guarded(data.shape[0], data.shape[1], ld, data.dtype)
        g.bits.fill_(_as_signed(POISON[data.dtype], g.bits.dtype))
        g.view.copy_(data.to(DEV))
        return self._add("in", name, g)

    def output(self, name, rows, width, ld=None, dtype=torch.float32, back_rows=0):
        return self._add("out", name, Guarded(rows, width, ld, dtype, back_rows=back_rows))

    def inout(self, name, prior, ld=None, back_rows=0):
        prior = prior.reshape(1, -1) if prior.dim() == 1 else prior.reshape(prior.shape[0], -1)
        g = Guarded(prior.shape[0], prior.shape[1], ld, prior.dtype, back_rows=back_rows)
        return self._add("inout", name, g, prior.to(DEV))

    def scratch(self, name, n, dtype=torch.float32):
        """Workspace of exactly n elements: NaN-filled, contents free, guards must survive."""
        g = Guarded(1, n, None, dtype)
        return self._add("scratch", name, g)

    def _prepare(self, sent):
        for kind, _, g, prior in self.bufs:
            if kind == "out":
                g.bits.fill_(_as_signed(sent[g.dtype], g.bits.dtype))
            elif kind == "inout":
                g.view.copy_(prior)
                g.fill_outside(sent[g.dtype])
            elif kind == "scratch":
                g.bits.fill_(_as_signed(sent[g.dtype], g.bits.dtype))
                g.fill_view_bits(POISON[g.dtype])

    def _check(self, sent, before, nan_ok):
        for (kind, name, g, _), snap in zip(self.bufs, before):
            what = f"{self.name}: {name}"
            if kind == "in":
                changed = torch.nonzero(g.bits != snap)
                assert changed.numel() == 0, f"{what}: input modified at (row, col) {g.where(changed[0, 0])}"
                continue
            pos = g.outside_changed(snap)
            assert pos is None, f"{what}: write outside the view at (row, col) {pos}"
            if kind == "out":
                pos = g.unwritten(sent[g.dtype])
                assert pos is None, f"{what}: element (row, col) {pos} never written"
            if kind in ("out", "inout") and g.dtype in (torch.float32, torch.bfloat16) and name not in nan_ok:
                nan = torch.nonzero(torch.isnan(g.view))
                assert nan.numel() == 0, f"{what}: NaN at (row, col) {tuple(nan[0].tolist())} (poison read?)"

    def run(self, launch, by_value=(), nan_ok=()):
        results = []
        for sent in (SENTINEL, SENTINEL2):
            self._prepare(sent)
            before = [g.bits.clone() for _, _, g, _ in self.bufs]
            torch.cuda.synchronize()
            launch()
            torch.cuda.synchronize()
            self._check(sent, before, nan_ok)
            results.append({name: g.view.clone() for kind, name, g, _ in self.bufs if kind in ("out", "inout")})
        first, second = results
        for name, t in first.items():
            if name in by_value:
                assert torch.allclose(t.double(), second[name].double(), rtol=1e-6, atol=1e-6), f"{self.name}: {name} differs on a rerun"
            else:
                same = t.view(_BITS[t.dtype]) == second[name].view(_BITS[t.dtype])
                bad = torch.nonzero(~same)
                assert bad.numel() == 0, f"{self.name}: {name} not bit-identical on a rerun at {tuple(bad[0].tolist())}"
        return {name: t.cpu() for name, t in first.items()}


def S():
    return torch.cuda.current_stream().cuda_stream


def call(name, *args):
    _cabi.check(getattr(_cabi.lib(), name)(*args), name)


# ------------------------------------------------------------------------------------------------------------------------
# value checks (the float64 references of _refs.py, on the CPU)
# ------------------------------------------------------------------------------------------------------------------------
def within(got, ref, rtol, atol_rel=0.0):
    """Elementwise |got - ref| <= rtol |ref| + atol_rel max |ref| (+ 1e-30), the bound of assert_close."""
    g, r = got.double(), ref.double()
    tol = rtol * r.abs() + atol_rel * r.abs().max().clamp_min(1e-30) + 1e-30
    return (g - r).abs() <= tol


def assert_close(got, ref, what, rtol, atol_rel=0.0):
    pos = first_bad(~within(got, ref, rtol, atol_rel))
    assert pos is None, f"{what}: element {pos} = {got.double()[pos].item()} vs reference {ref.double()[pos].item()}"


def grad_err(got, ref, whole):
    """Relative L2 error of one attention gradient, measured against 1e-2 of the whole gradient where this one vanishes (one
    key: the softmax is constant, dq and dk are zero up to rounding)."""
    return ((got.double() - ref).norm() / max(ref.norm().item(), 1e-2 * whole.norm().item(), 1e-30)).item()


def assert_equal(got, ref, what):
    g = got.view(_BITS[got.dtype]) if got.dtype in _BITS and got.dtype != torch.int64 else got
    r = ref.view(_BITS[ref.dtype]) if ref.dtype in _BITS and ref.dtype != torch.int64 else ref
    pos = first_bad(g != r)
    assert pos is None, f"{what}: element {pos} = {got[pos].item()} vs reference {ref[pos].item()}"


def rand(shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * scale).to(dtype)


# ------------------------------------------------------------------------------------------------------------------------
# coverage: every compute entry point has a case here
# ------------------------------------------------------------------------------------------------------------------------
COVERED = set()


def covers(*names):
    COVERED.update(names)
    return lambda fn: fn


NOT_FOOTPRINT = {
    # switches and setters: no device memory
    "b200_set_gemm_multicast", "b200_set_attention_fwd_version", "b200_set_attention_bwd_version", "b200_set_attention_prefetch",
    "b200_set_persistent_ctas",
    # queries
    "b200_abi_version", "b200_last_error", "b200_launch_count", "b200_gemm_pick_splits", "b200_colsum_per_image_workspace_floats",
    "b200_attention_long_bwd_workspace_floats", "b200_cross_attention_bwd_workspace_floats", "b200_groupnorm_workspace_floats",
    # the NCCL exchange needs two GPUs (tools/dp_check.py)
    "b200_comm_unique_id", "b200_comm_init", "b200_comm_allreduce_bucket", "b200_comm_async_error", "b200_comm_finalize",
    "b200_comm_nccl_version",
}


# ------------------------------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------------------------------
GEMM_SHAPES = [(1, 8, 8), (129, 1003, 200), (300, 264, 72)]
GEMM_CASES = ([(0, a, b) for a in (0, 1) for b in (0, 1)] + [(e, 0, 0) for e in (1, 2, 5, 7, 9)] + [(e, 0, 1) for e in (3, 6, 8)]
              + [(4, 1, 1)])


def _gemm_case(M, N, K, epi, a_mn, b_mn, inplace=False, max_ctas=0, splits=1):
    geglu = epi in (7, 8)
    if geglu:
        N = 400  # N = 2F, F = 200
    cols = N // 2 if epi == 8 else N  # the width of the product itself
    A = rand((M, K), 1)
    Bm = rand((cols, K), 2, 0.5)
    c = Case(f"gemm epi {epi} majors ({a_mn}, {b_mn}) {M}x{N}x{K}" + (" in place" if inplace else "") + (f" max_ctas {max_ctas}" if max_ctas else ""))
    ga = c.input("A", A.t().contiguous() if a_mn else A, ld=rup(M if a_mn else K) + 8)
    gb = c.input("B", Bm.t().contiguous() if b_mn else Bm, ld=rup(cols if b_mn else K) + 8)
    acc = A.double() @ Bm.double().t()
    bias = rand((N,), 3) if epi not in (3, 4, 6, 8) else None
    gbias = c.input("bias", bias) if bias is not None else None
    ldo = rup(N) + 8
    f32 = epi in (2, 4)
    out_dtype = torch.float32 if f32 else torch.bfloat16
    aux = out1 = None
    if epi == 4:
        nkb = (K + 63) // 64
        splits = min(splits, nkb)  # the kernel runs at most one split per 64-deep k-block
        out0 = c.output("out0", splits * M, N, ldo, out_dtype, back_rows=128)
    elif epi in (2, 9) and inplace:
        prior = rand((M, N), 4, dtype=out_dtype)
        out0 = c.inout("out0", prior, ldo, back_rows=128)
        aux = out0
    else:
        out0 = c.output("out0", M, N, ldo, out_dtype, back_rows=128)
    if epi in (2, 9) and not inplace:
        aux = c.input("aux", rand((M, N), 4, dtype=out_dtype), ldo)
    if epi in (3, 6):
        aux = c.input("aux", rand((M, N), 5), ldo)
    if epi == 8:
        aux = c.input("aux", rand((M, N), 5), ldo)
    if epi in (1, 5):
        out1 = c.output("out1", M, N, ldo, torch.bfloat16, back_rows=128)
    if epi == 7:
        out1 = c.output("out1", M, N // 2, None, torch.bfloat16, back_rows=128)
    lda = ga.ld
    ldb = gb.ld

    def launch():
        call("b200_gemm_bf16", ga.ptr(), lda, a_mn, gb.ptr(), ldb, b_mn, M, N, K, epi, gbias.ptr() if gbias else None, out0.ptr(),
             out1.ptr() if out1 else None, aux.ptr() if aux else None, ldo, splits, max_ctas, S())

    r = c.run(launch)
    o0 = r["out0"]
    b64 = bias.double() if bias is not None else 0.0
    if epi == 0:
        assert_ulp(o0, acc + b64, c.name)
    elif epi in (1, 5, 7):
        assert_ulp(o0, acc + b64, c.name + " out0")
        h = o0.double()
        if epi == 1:
            assert_ulp(r["out1"], gelu(h), c.name + " out1")
        elif epi == 5:  # eager's three bf16 roundings: 1.702 * h, sigmoid, product
            s = bf16(torch.sigmoid(bf16(1.702 * h).double())).double()
            assert_ulp(r["out1"], h * s, c.name + " out1", ulps=2.01, floor=1e-3)
        else:
            F_ = N // 2
            g = bf16(gelu(h[:, F_:])).double()
            assert_ulp(r["out1"], h[:, :F_] * g, c.name + " out1")
    elif epi == 2:
        prior = (rand((M, N), 4, dtype=out_dtype)).double()
        term = bf16(acc + b64).double()
        err = (o0.double() - prior - term).abs()
        ok = err <= 2.0 ** -7 * (acc + b64).abs() + 1e-6 * (acc + b64).abs().max()
        assert first_bad(~ok) is None, f"{c.name}: element {first_bad(~ok)}"
    elif epi == 9:
        prior = rand((M, N), 4, dtype=out_dtype).double()
        assert_ulp(o0, bf16(acc + b64).double() + prior, c.name, ulps=1.01, floor=1e-3)
    elif epi == 3:
        assert_ulp(o0, bf16(acc).double() * gelu_grad(rand((M, N), 5).double()), c.name, ulps=2.01, floor=1e-3)
    elif epi == 6:
        # autograd of h * sigmoid(1.702 h) on bf16 CUDA tensors, one rounding per kernel: the two products' gradients, sigmoid's
        # backward (evaluated in bf16 arithmetic, one rounding per operator), the 1.702 scaling, and the sum of both paths into
        # h.  The sum cancels, so the bound is relative to its terms.
        h = rand((M, N), 5).double()
        d = bf16(acc).double()
        s = bf16(torch.sigmoid(bf16(1.702 * h).double())).double()
        gh1 = bf16(d * s).double()
        gt = bf16(bf16(bf16(d * h).double() * bf16(1 - s).double()).double() * s).double()
        gh2 = bf16(1.702 * gt).double()
        assert_ulp(o0, gh1 + gh2, c.name, ulps=3.01, floor=1e-3, mag=gh1.abs() + gh2.abs())
    elif epi == 8:
        F_ = N // 2
        hg = rand((M, N), 5).double()
        da = bf16(acc).double()
        h, gate = hg[:, :F_], hg[:, F_:]
        g = bf16(gelu(gate)).double()
        dh = da * g
        dg = bf16(da * h).double()
        assert_ulp(o0, torch.cat([dh, gelu_grad(gate) * dg], 1), c.name, ulps=2.01, floor=1e-3)
    elif epi == 4:
        nkb = (K + 63) // 64
        planes = o0.double().view(splits, M, N)
        absacc = A.double().abs() @ Bm.double().abs().t()
        for sp in range(splits):
            k0, k1 = nkb * sp // splits * 64, min(K, nkb * (sp + 1) // splits * 64)
            ref = A.double()[:, k0:k1] @ Bm.double()[:, k0:k1].t()
            bad = (planes[sp] - ref).abs() > 1e-5 * absacc + 1e-30
            assert first_bad(bad) is None, f"{c.name}: split {sp} element {first_bad(bad)}"
    return r


@covers("b200_gemm_bf16")
@pytest.mark.gpu
@pytest.mark.parametrize("epi,a_mn,b_mn", GEMM_CASES)
@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_footprint(M, N, K, epi, a_mn, b_mn):
    _gemm_case(M, N, K, epi, a_mn, b_mn, splits=3 if epi == 4 else 1)


@pytest.mark.gpu
@pytest.mark.parametrize("epi", [2, 9])
@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_in_place_equals_out_of_place(M, N, K, epi):
    fresh = _gemm_case(M, N, K, epi, 0, 0)["out0"]
    inplace = _gemm_case(M, N, K, epi, 0, 0, inplace=True)["out0"]
    assert_equal(inplace, fresh, f"gemm epi {epi} in place vs out of place")


@pytest.mark.gpu
def test_gemm_one_cta():
    r1 = _gemm_case(129, 1003, 200, 0, 0, 0, max_ctas=1)["out0"]
    r0 = _gemm_case(129, 1003, 200, 0, 0, 0)["out0"]
    assert_equal(r1, r0, "gemm max_ctas = 1 vs all SMs")


# ------------------------------------------------------------------------------------------------------------------------
# 3x3 convolution
# ------------------------------------------------------------------------------------------------------------------------
CONV_SHAPES = [(3, 8, 8, 64, 200), (1, 16, 32, 128, 72)]


@covers("b200_conv3x3_nhwc_bf16")
@pytest.mark.gpu
@pytest.mark.parametrize("epi", [0, 2, 10, 11])
@pytest.mark.parametrize("B,H,W,Cin,Cout", CONV_SHAPES)
def test_conv3x3_footprint(B, H, W, Cin, Cout, epi):
    x = rand((B, H, W, Cin), 11)
    w = rand((Cout, Cin, 3, 3), 12, 0.7 / math.sqrt(9 * Cin))
    bias = rand((Cout,), 13, 0.1)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    M = B * H * W
    ldo = Cout + 8
    c = Case(f"conv3x3 epi {epi} {B}x{H}x{W}x{Cin}->{Cout}")
    gx = c.input("x", x.reshape(1, -1))  # NaN on both sides: the halo must come from the TMA zero fill
    gw = c.input("w", wp)
    dtype = torch.float32 if epi == 2 else torch.bfloat16
    aux = None
    if epi == 2:
        aux_v = rand((M, Cout), 14, dtype=torch.float32)
    elif epi == 10:
        aux_v = rand((B, Cout), 14)
    elif epi == 11:
        aux_v = rand((M, Cout), 14)
        # huge bias columns 0 and Cout - 1: the fp32 sums of pixel 0 / the last pixel overflow and are clamped to +-bf16 max
        bias[0], bias[Cout - 1] = 2e38, -2e38
        aux_v[0, 0], aux_v[M - 1, Cout - 1] = 3e38, -3e38
    gb = c.input("bias", bias)
    if epi:
        aux = c.input("aux", aux_v, ldo)
    out = c.output("out0", M, Cout, ldo, dtype, back_rows=128)
    r = c.run(lambda: call("b200_conv3x3_nhwc_bf16", gx.ptr(), gw.ptr(), gb.ptr(), out.ptr(), aux.ptr() if aux else None, ldo, B, H, W,
                           Cin, Cout, epi, S()))
    o = r["out0"]
    acc = conv3x3(x, w) + bias.double()
    if epi == 0:
        assert_ulp(o, acc, c.name)
    elif epi == 2:
        term = bf16(acc).double()
        ok = (o.double() - aux_v.double() - term).abs() <= 2.0 ** -7 * acc.abs() + 1e-6 * acc.abs().max()
        assert first_bad(~ok) is None, f"{c.name}: element {first_bad(~ok)}"
    elif epi == 10:
        per_pixel = aux_v.double().repeat_interleave(H * W, 0)
        assert_ulp(o, bf16(acc).double() + per_pixel, c.name, ulps=1.01, floor=1e-3)
    else:
        big = torch.finfo(torch.bfloat16).max
        ref = (bf16(acc).double() + aux_v.double()).clamp(-big, big)
        assert_ulp(o[:, 1:Cout - 1], ref[:, 1:Cout - 1], c.name, ulps=1.01, floor=1e-3)
        assert_ulp(o[1:, 0], ref[1:, 0], c.name + " column 0", floor=0.0)
        assert_ulp(o[:M - 1, Cout - 1], ref[:M - 1, Cout - 1], c.name + " last column", floor=0.0)
        assert o[0, 0].item() == big and o[M - 1, Cout - 1].item() == -big


@covers("b200_conv3x3_wgrad_nhwc_bf16")
@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,Cin,Cout", CONV_SHAPES)
def test_conv3x3_wgrad_footprint(B, H, W, Cin, Cout):
    x = rand((B, H, W, Cin), 21)
    M = B * H * W
    dy = rand((M, Cout), 22)
    splits = 2
    c = Case(f"conv3x3 wgrad {B}x{H}x{W}x{Cin}->{Cout}")
    gdy = c.input("dy", dy, ld=Cout + 8)
    gx = c.input("x", x.reshape(1, -1))
    part = c.output("partials", splits * Cout, 9 * Cin, back_rows=128)
    r = c.run(lambda: call("b200_conv3x3_wgrad_nhwc_bf16", gdy.ptr(), Cout + 8, gx.ptr(), part.ptr(), B, H, W, Cin, Cout, splits, S()))
    nkb = M // 64
    planes = r["partials"].double().view(splits, Cout, 9 * Cin)
    for sp in range(splits):
        p0, p1 = nkb * sp // splits * 64, nkb * (sp + 1) // splits * 64
        dy_sp = torch.zeros(M, Cout, dtype=torch.float64)  # the split's pixels only
        dy_sp[p0:p1] = dy.double()[p0:p1]
        ref = conv3x3_wgrad(dy_sp, x)
        absref = conv3x3_wgrad(dy_sp.abs(), x.abs())
        bad = (planes[sp] - ref).abs() > 1e-5 * absref + 1e-30
        assert first_bad(bad) is None, f"{c.name}: split {sp} element {first_bad(bad)}"


# ------------------------------------------------------------------------------------------------------------------------
# reductions
# ------------------------------------------------------------------------------------------------------------------------
@covers("b200_splitk_reduce")
@pytest.mark.gpu
@pytest.mark.parametrize("round_bf16,accumulate", [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("n", [4, 1028])
def test_splitk_reduce_footprint(n, round_bf16, accumulate):
    splits = 3
    part = rand((splits, n), 31, dtype=torch.float32)
    prior = rand((n,), 32, dtype=torch.float32)
    c = Case(f"splitk_reduce n {n} round {round_bf16} accumulate {accumulate}")
    gp = c.input("partial", part.reshape(1, -1))
    out = c.inout("out", prior) if accumulate else c.output("out", 1, n)
    r = c.run(lambda: call("b200_splitk_reduce", gp.ptr(), splits, n, out.ptr(), round_bf16, accumulate, S()))
    s = part[0].clone()
    for k in range(1, splits):
        s = s + part[k]  # fp32, the kernel's order: bit-exact
    if round_bf16:
        s = bf16(s).float()
    if accumulate:
        s = s + prior
    assert_equal(r["out"].view(-1), s, "splitk_reduce")


def _natural_parts_colsum(rows, cols):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return max(1, min(sms * 4 // ((cols + 255) // 256), (rows + 7) // 8))


@covers("b200_colsum_bf16")
@pytest.mark.gpu
@pytest.mark.parametrize("cols", [13, 1000])
@pytest.mark.parametrize("rows", [4, 1028])
def test_colsum_bf16_footprint(rows, cols):
    x = rand((rows, cols), 41)
    natural = _natural_parts_colsum(rows, cols)
    max_parts = max(1, natural - 1) if natural > 1 else 1
    c = Case(f"colsum_bf16 {rows}x{cols}")
    gx = c.input("x", x, ld=rup(cols) + 8)  # NaN in [cols, roundup(cols, 8)), which the kernel reads
    part = c.output("part", max_parts, cols)
    nparts = ctypes.c_int(-1)
    r = c.run(lambda: call("b200_colsum_bf16", gx.ptr(), gx.ld, rows, cols, part.ptr(), max_parts, ctypes.byref(nparts), S()))
    assert nparts.value == max_parts
    got = r["part"].double().sum(0)
    ref = x.double().sum(0)
    assert_close(got, ref, c.name, rtol=1e-6, atol_rel=1e-6)


@covers("b200_colsum_finish", "b200_colsum_finish2")
@pytest.mark.gpu
@pytest.mark.parametrize("round_bf16,accumulate", [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("cols", [13, 1000])
@pytest.mark.parametrize("nparts", [4, 1028])
def test_colsum_finish_footprint(nparts, cols, round_bf16, accumulate):
    part = rand((nparts, cols), 51, dtype=torch.float32)
    prior = rand((cols,), 52, dtype=torch.float32)
    c = Case(f"colsum_finish {nparts}x{cols} round {round_bf16} accumulate {accumulate}")
    gp = c.input("part", part, ld=cols + 5)
    out = c.inout("out", prior) if accumulate else c.output("out", 1, cols)
    r = c.run(lambda: call("b200_colsum_finish", gp.ptr(), gp.ld, nparts, cols, out.ptr(), round_bf16, accumulate, S()))
    _check_finish(r["out"].view(-1), part.double().sum(0), prior, round_bf16, accumulate, c.name)
    # two destinations: (13, 7) columns of the same parts
    c0, c1 = 13, 7
    part2 = rand((nparts, c0 + c1), 53, dtype=torch.float32)
    c = Case(f"colsum_finish2 {nparts} round {round_bf16} accumulate {accumulate}")
    gp = c.input("part", part2, ld=c0 + c1 + 3)
    o0 = c.inout("out0", prior[:c0]) if accumulate else c.output("out0", 1, c0)
    o1 = c.inout("out1", prior[:c1]) if accumulate else c.output("out1", 1, c1)
    r = c.run(lambda: call("b200_colsum_finish2", gp.ptr(), gp.ld, nparts, c0, o0.ptr(), round_bf16, c1, o1.ptr(), 1 - round_bf16,
                           accumulate, S()))
    ref = part2.double().sum(0)
    _check_finish(r["out0"].view(-1), ref[:c0], prior[:c0], round_bf16, accumulate, c.name + " out0")
    _check_finish(r["out1"].view(-1), ref[c0:], prior[:c1], 1 - round_bf16, accumulate, c.name + " out1")


def _check_finish(got, ref, prior, round_bf16, accumulate, what):
    got = got.double() - (prior.double() if accumulate else 0.0)  # prior + t in fp32: exact to half an fp32 ulp of the sum
    if round_bf16:
        assert_ulp(got, ref, what, floor=1e-5)
    else:
        assert_close(got, ref, what, rtol=1e-5, atol_rel=1e-5)


@covers("b200_colsum_per_image_bf16")
@pytest.mark.gpu
@pytest.mark.parametrize("B,HW,C", [(5, 72, 8), (2, 4096, 328)])
def test_colsum_per_image_footprint(B, HW, C):
    x = rand((B * HW, C), 61)
    ws = int(_cabi.lib().b200_colsum_per_image_workspace_floats(B, HW, C))
    c = Case(f"colsum_per_image {B}x{HW}x{C}")
    gx = c.input("x", x)
    per = c.output("per_image", B, C, dtype=torch.bfloat16)
    tot = c.output("total", 1, C)
    w = c.scratch("workspace", ws)
    r = c.run(lambda: call("b200_colsum_per_image_bf16", gx.ptr(), B, HW, C, per.ptr(), tot.ptr(), w.ptr(), S()))
    ref = x.double().view(B, HW, C).sum(1)
    assert_ulp(r["per_image"], ref, c.name + " per_image", floor=1e-5)
    assert_ulp(r["total"].view(-1), ref.sum(0), c.name + " total", floor=1e-5)


# ------------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------------------------------
def _ln_natural_parts(rows):
    return min(2 * torch.cuda.get_device_properties(0).multi_processor_count, (rows + 7) // 8)


@covers("b200_layernorm_fwd")
@pytest.mark.gpu
@pytest.mark.parametrize("with_f32", [False, True])
@pytest.mark.parametrize("dim", [8, 1000, 1024])
@pytest.mark.parametrize("rows", [1, 333])
def test_layernorm_fwd_footprint(rows, dim, with_f32):
    x = rand((rows, dim), 71, 1.5, torch.float32) + 0.3
    gam, bet = rand((dim,), 72, dtype=torch.float32), rand((dim,), 73, dtype=torch.float32)
    c = Case(f"layernorm_fwd {rows}x{dim} y_f32 {with_f32}")
    gx = c.input("x", x, ld=dim + 4)
    gg, gb = c.input("gamma", gam), c.input("beta", bet)
    y = c.output("y", rows, dim, dtype=torch.bfloat16)
    y32 = c.output("y_f32", rows, dim) if with_f32 else None
    mean, rstd = c.output("mean", 1, rows), c.output("rstd", 1, rows)
    r = c.run(lambda: call("b200_layernorm_fwd", gx.ptr(), gx.ld, gg.ptr(), gb.ptr(), y.ptr(), y32.ptr() if y32 else None, mean.ptr(),
                           rstd.ptr(), rows, dim, 1e-6, S()))
    ref, m, rs, _ = layernorm(x, gam, bet, 1e-6)
    assert_ulp(r["y"], ref, c.name + " y", floor=1e-5)
    if with_f32:
        assert_close(r["y_f32"], ref, c.name + " y_f32", rtol=1e-5, atol_rel=1e-5)
        assert_equal(r["y"], r["y_f32"].to(torch.bfloat16), c.name + " y == bf16(y_f32)")
    assert_close(r["mean"].view(-1), m, c.name + " mean", rtol=1e-5, atol_rel=1e-6)
    assert_close(r["rstd"].view(-1), rs, c.name + " rstd", rtol=1e-5)


@covers("b200_layernorm_bwd")
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "bf16_colsum", "bf16_dres", "f32_dy"])
@pytest.mark.parametrize("dim", [8, 1000, 1024])
@pytest.mark.parametrize("rows", [1, 333])
def test_layernorm_bwd_footprint(rows, dim, mode):
    x = rand((rows, dim), 81, 1.5, torch.float32) + 0.3
    gam, bet = rand((dim,), 82, dtype=torch.float32), rand((dim,), 83, dtype=torch.float32)
    _, m, rs, _ = layernorm(x, gam, bet, 1e-6)
    dy_is_f32 = mode == "f32_dy"
    dy = rand((rows, dim), 84, dtype=torch.float32 if dy_is_f32 else torch.bfloat16)
    dres = rand((rows, dim), 85, dtype=torch.float32) if mode == "bf16_dres" else None  # row stride ld_dx, like dx_out
    colsum = mode == "bf16_colsum"
    want_bf16 = not dy_is_f32
    nw = 3 if colsum else 2
    natural = _ln_natural_parts(rows)
    max_parts = max(1, min(5, natural - 1)) if natural > 1 else 1
    c = Case(f"layernorm_bwd {rows}x{dim} {mode}")
    gdy = c.input("dy", dy)
    gx = c.input("x", x, ld=dim + 4)
    gg = c.input("gamma", gam)
    gm, gr = c.input("mean", m.float()), c.input("rstd", rs.float())
    gres = c.input("dres", dres, ld=3 * dim) if dres is not None else None
    dx = c.output("dx", rows, dim, ld=3 * dim)  # the head LN scatters into token 0 of a wider row
    dxb = c.output("dx_bf16", rows, dim, dtype=torch.bfloat16) if want_bf16 else None
    part = c.output("dgb_part", max_parts, nw * dim)
    nparts = ctypes.c_int(-1)
    r = c.run(lambda: call("b200_layernorm_bwd", gdy.ptr(), int(dy_is_f32), gx.ptr(), gx.ld, gg.ptr(), gm.ptr(), gr.ptr(),
                           gres.ptr() if gres else None, dx.ptr(), dx.ld, dxb.ptr() if dxb else None, part.ptr(), max_parts,
                           ctypes.byref(nparts), rows, dim, int(colsum), S()))
    assert nparts.value == max_parts
    xr = x.double().requires_grad_(True)
    gr_ = gam.double().requires_grad_(True)
    br_ = bet.double().requires_grad_(True)
    y = F.layer_norm(xr, (dim,), gr_, br_, 1e-6)
    y.backward(dy.double())
    ref_dx = xr.grad + (dres.double() if dres is not None else 0.0)
    assert relerr(r["dx"], ref_dx) < 1e-5, (c.name, relerr(r["dx"], ref_dx))
    assert_close(r["dx"], ref_dx, c.name + " dx", rtol=1e-4, atol_rel=1e-5)
    if want_bf16:
        assert_equal(r["dx_bf16"], r["dx"].to(torch.bfloat16), c.name + " dx_bf16 == bf16(dx)")
    sums = r["dgb_part"].double().sum(0)
    assert relerr(sums[:dim], gr_.grad) < 1e-5 and relerr(sums[dim:2 * dim], br_.grad) < 1e-5, c.name
    if colsum:
        assert_close(sums[2 * dim:], r["dx_bf16"].double().sum(0), c.name + " dx colsum", rtol=1e-5, atol_rel=1e-5)


@covers("b200_layernorm_bf16_fwd", "b200_layernorm_bf16_bwd")
@pytest.mark.gpu
@pytest.mark.parametrize("with_dres", [False, True])
@pytest.mark.parametrize("dim", [8, 2048])
@pytest.mark.parametrize("rows", [1, 333])
def test_layernorm_bf16_footprint(rows, dim, with_dres):
    x = rand((rows, dim), 91, 1.5)
    gam, bet = rand((dim,), 92, dtype=torch.float32), rand((dim,), 93, dtype=torch.float32)
    c = Case(f"layernorm_bf16_fwd {rows}x{dim}")
    gx, gg, gb = c.input("x", x), c.input("gamma", gam), c.input("beta", bet)
    y = c.output("y", rows, dim, dtype=torch.bfloat16)
    mean, rstd = c.output("mean", 1, rows), c.output("rstd", 1, rows)
    r = c.run(lambda: call("b200_layernorm_bf16_fwd", gx.ptr(), gg.ptr(), gb.ptr(), y.ptr(), mean.ptr(), rstd.ptr(), rows, dim, 1e-5, S()))
    ref, m, rs, _ = layernorm(x, gam, bet, 1e-5)
    assert_ulp(r["y"], ref, c.name + " y", floor=1e-5)
    assert_close(r["mean"].view(-1), m, c.name + " mean", rtol=1e-5, atol_rel=1e-6)
    assert_close(r["rstd"].view(-1), rs, c.name + " rstd", rtol=1e-5)

    dy = rand((rows, dim), 94)
    dres = rand((rows, dim), 95) if with_dres else None
    natural = _ln_natural_parts(rows)
    max_parts = max(1, min(5, natural - 1)) if natural > 1 else 1
    c = Case(f"layernorm_bf16_bwd {rows}x{dim} dres {with_dres}")
    gdy, gx, gg = c.input("dy", dy), c.input("x", x), c.input("gamma", gam)
    gm, gr = c.input("mean", m.float()), c.input("rstd", rs.float())
    gres = c.input("dres", dres) if with_dres else None
    dx = c.output("dx", rows, dim, dtype=torch.bfloat16)
    part = c.output("dgb_part", max_parts, 2 * dim)
    nparts = ctypes.c_int(-1)
    r = c.run(lambda: call("b200_layernorm_bf16_bwd", gdy.ptr(), gx.ptr(), gg.ptr(), gm.ptr(), gr.ptr(), gres.ptr() if gres else None,
                           dx.ptr(), part.ptr(), max_parts, ctypes.byref(nparts), rows, dim, S()))
    assert nparts.value == max_parts
    xr = x.double().requires_grad_(True)
    gr_, br_ = gam.double().requires_grad_(True), bet.double().requires_grad_(True)
    F.layer_norm(xr, (dim,), gr_, br_, 1e-5).backward(dy.double())
    ref_dx = bf16(xr.grad).double() + (dres.double() if with_dres else 0.0)
    assert_ulp(r["dx"], ref_dx, c.name + " dx", ulps=2.01, floor=1e-3)
    sums = r["dgb_part"].double().sum(0)
    assert relerr(sums[:dim], gr_.grad) < 1e-5 and relerr(sums[dim:], br_.grad) < 1e-5, c.name


# ------------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------------
def _packed_attention(entry, B, T, H, causal, with_dbias=True):
    """attention_fwd / _bwd (T <= 256) or attention_long_fwd / _bwd on packed qkv [B, T, 3 H 64]."""
    long_ = entry == "long"
    D = H * 64
    qkv = rand((B * T, 3 * D), 101)
    dout = rand((B * T, D), 102)
    fwd = "b200_attention_long_fwd" if long_ else "b200_attention_fwd"
    bwd = "b200_attention_long_bwd" if long_ else "b200_attention_bwd"
    c = Case(f"{fwd} B {B} T {T} H {H} causal {causal}")
    gq = c.input("qkv", qkv)
    out = c.output("out", B * T, D, dtype=torch.bfloat16, back_rows=64)
    lse = c.output("lse", B * H, T)
    r = c.run(lambda: call(fwd, gq.ptr(), out.ptr(), lse.ptr(), B, T, H, 64, 0.125, causal, S()))
    (o, l), (ref,) = with_grads(packed_attention, (qkv,), dout, B, T, H, 0.125, causal)
    assert relerr(r["out"], o) < 5e-3, (c.name, relerr(r["out"], o))
    assert_close(r["lse"].view(B, H, T), l, c.name + " lse", rtol=1e-4, atol_rel=1e-5)

    c2 = Case(f"{bwd} B {B} T {T} H {H} causal {causal}")
    gq = c2.input("qkv", qkv)
    go = c2.input("out", r["out"])
    gd = c2.input("dout", dout)
    gl = c2.input("lse", r["lse"])
    dqkv = c2.output("dqkv", B * T, 3 * D, dtype=torch.bfloat16, back_rows=64)
    dbp = c2.output("dbias_part", B, 3 * D) if with_dbias else None
    ws = c2.scratch("workspace", int(_cabi.lib().b200_attention_long_bwd_workspace_floats(B, T, H))) if long_ else None
    args = [gq.ptr(), go.ptr(), gd.ptr(), gl.ptr(), dqkv.ptr(), B, T, H, 64, 0.125, causal, dbp.ptr() if dbp else None]
    if long_:
        args.append(ws.ptr())
    r2 = c2.run(lambda: call(bwd, *args, S()))
    for name, sl in (("dq", slice(0, D)), ("dk", slice(D, 2 * D)), ("dv", slice(2 * D, 3 * D))):
        e = grad_err(r2["dqkv"][:, sl], ref[:, sl], ref)
        assert e < 1e-2, f"{c2.name}: {name} relative error {e}"
    if with_dbias:
        want = r2["dqkv"].double().view(B, T, 3 * D).sum(1)
        absw = r2["dqkv"].double().abs().view(B, T, 3 * D).sum(1)
        bad = (r2["dbias_part"].double() - want).abs() > 1e-5 * absw + 1e-30
        assert first_bad(bad) is None, f"{c2.name}: dbias_part element {first_bad(bad)}"


@covers("b200_attention_fwd", "b200_attention_bwd")
@pytest.mark.gpu
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("T", [1, 63, 64, 65, 129, 255, 256])
def test_attention_footprint(T, causal):
    _packed_attention("resident", 2, T, 2, causal)


@pytest.mark.gpu
def test_attention_footprint_more_items_than_sms():
    _packed_attention("resident", 12, 65, 12, 0)  # B * H = 144 > 132 items


@covers("b200_attention_long_fwd", "b200_attention_long_bwd")
@pytest.mark.gpu
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("T", [1, 65, 257, 1025])
def test_attention_long_footprint(T, causal):
    _packed_attention("long", 1 if T > 512 else 2, T, 2, causal)


def _cross_case(B, Tq, Tk, H, Dh, causal, packed=False):
    L = H * Dh
    scale = Dh ** -0.5
    q = rand((B * Tq, L), 111)
    k = rand((B * Tk, L), 112)
    v = rand((B * Tk, L), 113)
    dout = rand((B * Tq, L), 114)
    c = Case(f"cross_attention_fwd B {B} Tq {Tq} Tk {Tk} Dh {Dh} causal {causal}" + (" packed" if packed else ""))
    if packed:  # q / k / v and dq / dk / dv: column slices of one [B, T, 3 L + 8] buffer
        ld = 3 * L + 8
        gqkv = c.input("qkv", torch.cat([q, k, v], 1), ld=ld)
        pq, pk, pv, ldq, ldkv = gqkv.ptr(), gqkv.ptr() + 2 * L, gqkv.ptr() + 4 * L, ld, ld
    else:
        gq = c.input("q", q, ld=L + 8)
        gk = c.input("k", k, ld=L + 8)
        gv = c.input("v", v, ld=L + 8)
        pq, pk, pv, ldq, ldkv = gq.ptr(), gk.ptr(), gv.ptr(), L + 8, L + 8
    out = c.output("out", B * Tq, L, ld=L + 8, dtype=torch.bfloat16, back_rows=64)
    lse = c.output("lse", B * H, Tq)
    r = c.run(lambda: call("b200_cross_attention_fwd", pq, ldq, pk, pv, ldkv, out.ptr(), out.ld, lse.ptr(), B, Tq, Tk, H, Dh, scale,
                           causal, S()))
    (o, l), (dq64, dk64, dv64) = with_grads(attention_rows, (q, k, v), dout, B, H, scale, causal)
    assert relerr(r["out"], o) < 5e-3, (c.name, relerr(r["out"], o))
    assert_close(r["lse"].view(B, H, Tq), l, c.name + " lse", rtol=1e-4, atol_rel=1e-5)

    c2 = Case(c.name.replace("fwd", "bwd"))
    go = c2.input("out", r["out"], ld=L + 8)
    gd = c2.input("dout", dout, ld=L + 8)
    gl = c2.input("lse", r["lse"])
    ws = c2.scratch("workspace", int(_cabi.lib().b200_cross_attention_bwd_workspace_floats(B, Tq, Tk, H, Dh)))
    if packed:
        gqkv = c2.input("qkv", torch.cat([q, k, v], 1), ld=ld)
        pq, pk, pv = gqkv.ptr(), gqkv.ptr() + 2 * L, gqkv.ptr() + 4 * L
        dqkv = c2.output("dqkv", B * Tq, 3 * L, ld=ld, dtype=torch.bfloat16, back_rows=64)
        pdq, pdk, pdv = dqkv.ptr(), dqkv.ptr() + 2 * L, dqkv.ptr() + 4 * L
    else:
        gq, gk, gv = c2.input("q", q, ld=L + 8), c2.input("k", k, ld=L + 8), c2.input("v", v, ld=L + 8)
        pq, pk, pv = gq.ptr(), gk.ptr(), gv.ptr()
        dq = c2.output("dq", B * Tq, L, ld=L + 8, dtype=torch.bfloat16, back_rows=64)
        dk = c2.output("dk", B * Tk, L, ld=L + 8, dtype=torch.bfloat16, back_rows=64)
        dv = c2.output("dv", B * Tk, L, ld=L + 8, dtype=torch.bfloat16, back_rows=64)
        pdq, pdk, pdv = dq.ptr(), dk.ptr(), dv.ptr()
    r2 = c2.run(lambda: call("b200_cross_attention_bwd", pq, ldq, pk, pv, ldkv, go.ptr(), go.ld, gd.ptr(), gl.ptr(), pdq, pdk, pdv, B,
                             Tq, Tk, H, Dh, scale, causal, ws.ptr(), S()))
    if packed:
        got = {"dq": r2["dqkv"][:, :L], "dk": r2["dqkv"][:, L:2 * L], "dv": r2["dqkv"][:, 2 * L:]}
    else:
        got = r2
    whole = torch.cat([dq64.flatten(), dk64.flatten(), dv64.flatten()])
    for name, ref in (("dq", dq64), ("dk", dk64), ("dv", dv64)):
        e = grad_err(got[name], ref, whole)
        assert e < 1e-2, f"{c2.name}: {name} relative error {e}"


@covers("b200_cross_attention_fwd", "b200_cross_attention_bwd")
@pytest.mark.gpu
@pytest.mark.parametrize("Tq,Tk,causal", [(65, 1, 0), (300, 77, 0), (129, 129, 1)])
@pytest.mark.parametrize("Dh", [8, 40, 72, 160])
def test_cross_attention_footprint(Dh, Tq, Tk, causal):
    _cross_case(2, Tq, Tk, 2, Dh, causal)


@pytest.mark.gpu
def test_cross_attention_packed_slices_footprint():
    _cross_case(2, 129, 129, 2, 40, 1, packed=True)


# ------------------------------------------------------------------------------------------------------------------------
# FCNN step
# ------------------------------------------------------------------------------------------------------------------------
FC_DIMS = [10, 32, 32, 1]
FC_WOFF = [0, 360, 1384]
FC_BOFF = [324, -1, 1416]  # gaps at 320..323, 356..359 and 1417..1419; layer 1 has no bias
FC_P = 1420


@covers("b200_fcnn_step")
@pytest.mark.gpu
@pytest.mark.parametrize("with_pred", [False, True])
@pytest.mark.parametrize("loss_mode", [0, 1])
@pytest.mark.parametrize("M", [1, 129])
def test_fcnn_step_footprint(M, loss_mode, with_pred):
    params = rand((FC_P,), 121, 0.3, torch.float32)
    gaps = torch.ones(FC_P, dtype=torch.bool)
    for l in range(3):
        gaps[FC_WOFF[l]:FC_WOFF[l] + FC_DIMS[l] * FC_DIMS[l + 1]] = False
        if FC_BOFF[l] >= 0:
            gaps[FC_BOFF[l]:FC_BOFF[l] + FC_DIMS[l + 1]] = False
    params.view(torch.int32)[gaps] = POISON[torch.float32]  # the arena's alignment gaps are never read
    x = rand((M, 10), 122, dtype=torch.float32)
    y = rand((M, 1), 123, dtype=torch.float32)
    dpred = rand((M, 1), 124, dtype=torch.float32)
    nblk = (M + 127) // 128
    c = Case(f"fcnn_step M {M} loss_mode {loss_mode} pred {with_pred}")
    gx, gy, gdp, gp = c.input("x", x), c.input("y", y), c.input("dpred", dpred), c.input("params", params)
    pred = c.output("pred", M, 1) if with_pred else None
    part = c.output("part", nblk, FC_P + 1)
    dims = (ctypes.c_int * 4)(*FC_DIMS)
    wo = (ctypes.c_int * 3)(*FC_WOFF)
    bo = (ctypes.c_int * 3)(*FC_BOFF)
    nb = ctypes.c_int(-1)
    r = c.run(lambda: call("b200_fcnn_step", gx.ptr(), gy.ptr() if loss_mode else None, gdp.ptr() if not loss_mode else None, gp.ptr(),
                           pred.ptr() if pred else None, part.ptr(), M, 3, dims, wo, bo, FC_P, loss_mode, 0.5, 0.7, ctypes.byref(nb), S()))
    assert nb.value == nblk
    inv = 1.0 / M
    for blk in range(nblk):
        p = params.double().clone()
        p[gaps] = 0.0
        p.requires_grad_(True)
        rows = slice(blk * 128, min(M, blk * 128 + 128))
        a = x.double()[rows]
        for l in range(3):
            W = p[FC_WOFF[l]:FC_WOFF[l] + FC_DIMS[l] * FC_DIMS[l + 1]].view(FC_DIMS[l + 1], FC_DIMS[l])
            a = a @ W.t() + (p[FC_BOFF[l]:FC_BOFF[l] + FC_DIMS[l + 1]] if FC_BOFF[l] >= 0 else 0.0)
            if l < 2:
                a = torch.relu(a)
        if with_pred:
            assert_close(r["pred"][rows], a.detach(), c.name + " pred", rtol=1e-5, atol_rel=1e-5)
        if loss_mode:
            d = a - y.double()[rows]
            loss = (0.5 * d.abs() + 0.7 * d * d).sum() * inv
        else:
            loss = (a * dpred.double()[rows]).sum()
        loss.backward()
        ref = torch.cat([p.grad, torch.tensor([loss.item() if loss_mode else 0.0], dtype=torch.float64)])
        assert_close(r["part"][blk], ref, f"{c.name} part row {blk}", rtol=1e-4, atol_rel=1e-5)
        assert (r["part"][blk, :FC_P][gaps] == 0).all(), f"{c.name}: arena gaps of part row {blk} are not zero"


# ------------------------------------------------------------------------------------------------------------------------
# patch embedding glue
# ------------------------------------------------------------------------------------------------------------------------
@covers("b200_patch_im2col")
@pytest.mark.gpu
@pytest.mark.parametrize("B,C,img,P", [(1, 3, 32, 16), (2, 1, 64, 32)])
def test_patch_im2col_footprint(B, C, img, P):
    x = rand((B, C, img, img), 131, dtype=torch.float32)
    side = img // P
    c = Case(f"patch_im2col {B}x{C}x{img} P {P}")
    gx = c.input("x", x.reshape(1, -1))
    cols = c.output("cols", B * side * side, C * P * P, dtype=torch.bfloat16)
    r = c.run(lambda: call("b200_patch_im2col", gx.ptr(), cols.ptr(), B, C, img, P, S()))
    ref = F.unfold(x, kernel_size=P, stride=P).transpose(1, 2).reshape(B * side * side, C * P * P)
    assert_equal(r["cols"], ref.to(torch.bfloat16), c.name)


@covers("b200_patch_im2col_u8")
@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 3, 4])
def test_patch_im2col_u8_footprint(C):
    B, img, P = 2, 32, 16
    x = torch.randint(0, 256, (B, img, img, C), dtype=torch.uint8, generator=torch.Generator().manual_seed(C))
    mean = [0.485, 0.456, 0.406, 0.5][:C]
    std = [0.229, 0.224, 0.225, 0.25][:C]
    side = img // P
    c = Case(f"patch_im2col_u8 C {C}")
    gx = c.input("x", x.reshape(1, -1))
    cols = c.output("cols", B * side * side, C * P * P, dtype=torch.bfloat16)
    dbl = ctypes.c_double * C
    r = c.run(lambda: call("b200_patch_im2col_u8", gx.ptr(), cols.ptr(), B, C, img, P, 255.0, dbl(*mean), dbl(*std), S()))
    norm = ((x.double() / 255.0 - torch.tensor(mean, dtype=torch.float64)) / torch.tensor(std, dtype=torch.float64)).float()
    chw = norm.permute(0, 3, 1, 2).contiguous()
    ref = F.unfold(chw, kernel_size=P, stride=P).transpose(1, 2).reshape(B * side * side, C * P * P)
    assert_equal(r["cols"], ref.to(torch.bfloat16), c.name)


@covers("b200_assemble_tokens", "b200_assemble_tokens_bwd")
@pytest.mark.gpu
@pytest.mark.parametrize("flag", [0, 1])  # conv bias (forward) / accumulate (backward)
@pytest.mark.parametrize("B,C,img,P", [(1, 3, 32, 16), (2, 1, 64, 32)])
def test_assemble_tokens_footprint(B, C, img, P, flag):
    np_ = (img // P) ** 2
    D = 40
    patch = rand((B * np_, D), 141)
    cls = rand((D,), 142, dtype=torch.float32)
    pos = rand((np_ + 1, D), 143, dtype=torch.float32)
    cb = rand((D,), 144)
    c = Case(f"assemble_tokens B {B} np {np_} bias {flag}")
    gp, gc, gpos = c.input("patch", patch), c.input("cls", cls), c.input("pos", pos)
    gcb = c.input("conv_bias", cb) if flag else None
    net = c.output("net", B * (np_ + 1), D)
    r = c.run(lambda: call("b200_assemble_tokens", gp.ptr(), gc.ptr(), gpos.ptr(), net.ptr(), B, np_, D, gcb.ptr() if gcb else None, S()))
    pf = patch.float()
    if flag:
        pf = bf16(pf + cb.float()).float()
    ref = torch.cat([cls.view(1, 1, D).expand(B, 1, D), pf.view(B, np_, D)], 1) + pos
    assert_equal(r["net"].view(B, np_ + 1, D), ref, c.name)

    dnet = rand((B, np_ + 1, D), 145, dtype=torch.float32)
    prior_pos, prior_cls = rand((np_ + 1, D), 146, dtype=torch.float32), rand((D,), 147, dtype=torch.float32)
    c = Case(f"assemble_tokens_bwd B {B} np {np_} accumulate {flag}")
    gd = c.input("dnet", dnet.reshape(B * (np_ + 1), D))
    dpatch = c.output("dpatch", B * np_, D, dtype=torch.bfloat16)
    dpos = c.inout("dpos", prior_pos) if flag else c.output("dpos", np_ + 1, D)
    dcls = c.inout("dcls", prior_cls) if flag else c.output("dcls", 1, D)
    r = c.run(lambda: call("b200_assemble_tokens_bwd", gd.ptr(), dpatch.ptr(), dpos.ptr(), dcls.ptr(), B, np_, D, flag, S()))
    s = torch.zeros(np_ + 1, D)
    for b in range(B):
        s = s + dnet[b]  # fp32 in the kernel's order
    assert_equal(r["dpatch"], dnet[:, 1:].reshape(B * np_, D).to(torch.bfloat16), c.name + " dpatch")
    assert_equal(r["dpos"], prior_pos + s if flag else s, c.name + " dpos")
    assert_equal(r["dcls"].view(-1), prior_cls + s[0] if flag else s[0], c.name + " dcls")


@covers("b200_add_pos", "b200_add_pos_bwd")
@pytest.mark.gpu
@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("B,T,D", [(1, 5, 12), (3, 77, 40)])
def test_add_pos_footprint(B, T, D, accumulate):
    x = rand((B * T, D), 151, dtype=torch.float32)
    pos = rand((T, D), 152, dtype=torch.float32)
    c = Case(f"add_pos {B}x{T}x{D}")
    gx, gp = c.input("x", x), c.input("pos", pos)
    net = c.output("net", B * T, D)
    r = c.run(lambda: call("b200_add_pos", gx.ptr(), gp.ptr(), net.ptr(), B, T, D, S()))
    assert_equal(r["net"], (x.view(B, T, D) + pos).view(B * T, D), c.name)
    prior = rand((T, D), 153, dtype=torch.float32)
    c = Case(f"add_pos_bwd {B}x{T}x{D} accumulate {accumulate}")
    gd = c.input("dnet", x)
    dpos = c.inout("dpos", prior) if accumulate else c.output("dpos", T, D)
    r = c.run(lambda: call("b200_add_pos_bwd", gd.ptr(), dpos.ptr(), B, T, D, accumulate, S()))
    s = torch.zeros(T, D)
    for b in range(B):
        s = s + x.view(B, T, D)[b]
    assert_equal(r["dpos"], prior + s if accumulate else s, c.name)


# ------------------------------------------------------------------------------------------------------------------------
# CLIP text glue: integer-indexed row moves
# ------------------------------------------------------------------------------------------------------------------------
@covers("b200_embedding_fwd", "b200_embedding_bwd")
@pytest.mark.gpu
def test_embedding_footprint():
    V, D = 10, 12
    ids = torch.tensor([3, 1, 3, 9, 0, 3, 12, 5, 1, 3, -1, 7, 7], dtype=torch.int64)  # repeats; 12 and -1 are out of range
    n = ids.numel()
    weight = rand((V, D), 161, dtype=torch.float32)
    c = Case("embedding_fwd")
    gi, gw = c.input("ids", ids), c.input("weight", weight)
    out = c.output("out", n, D)
    flag = c.inout("bad_index_flag", torch.zeros(1, dtype=torch.int32))
    r = c.run(lambda: call("b200_embedding_fwd", gi.ptr(), gw.ptr(), out.ptr(), n, D, V, flag.ptr(), S()))
    assert r["bad_index_flag"].item() == 1
    assert_equal(r["out"], weight[torch.where((ids >= 0) & (ids < V), ids, 0)], "embedding_fwd")

    dnet = rand((n, D), 162, dtype=torch.float32)
    prior = rand((V, D), 163, dtype=torch.float32)  # the caller's values: the kernel only adds
    pad = 3
    c = Case("embedding_bwd")
    gi, gd = c.input("ids", ids), c.input("dnet", dnet)
    dw = c.inout("dweight", prior)
    r = c.run(lambda: call("b200_embedding_bwd", gi.ptr(), gd.ptr(), dw.ptr(), n, D, V, pad, S()), by_value=("dweight",))
    keep = (ids >= 0) & (ids < V) & (ids != pad)
    ref = prior.double().index_add(0, ids[keep], dnet.double()[keep])
    assert_close(r["dweight"], ref, "embedding_bwd", rtol=1e-6, atol_rel=1e-6)
    untouched = torch.ones(V, dtype=torch.bool)
    untouched[ids[keep]] = False
    assert_equal(r["dweight"][untouched], prior[untouched], "embedding_bwd rows no id owns")


@covers("b200_argmax_gather_rows", "b200_scatter_rows")
@pytest.mark.gpu
def test_argmax_gather_scatter_footprint():
    B, T, D = 4, 7, 132
    ids = torch.tensor([[1, 5, 2, 5, 0, 0, 0],      # tie: the first maximum
                        [9, 9, 9, 9, 9, 9, 9],      # all equal: position 0
                        [0, 1, 2, 3, 4, 5, 6],      # the last position
                        [-3, -1, -2, -1, -7, -9, -1]], dtype=torch.int64)
    want_pos = torch.tensor([1, 0, 6, 1], dtype=torch.int32)
    x = rand((B * T, D), 171, dtype=torch.float32)
    c = Case("argmax_gather_rows")
    gi, gx = c.input("ids", ids), c.input("x", x)
    out = c.output("out", B, D)
    pos = c.output("pos", 1, B, dtype=torch.int32)
    r = c.run(lambda: call("b200_argmax_gather_rows", gi.ptr(), gx.ptr(), out.ptr(), pos.ptr(), B, T, D, S()))
    assert_equal(r["pos"].view(-1), want_pos, "argmax_gather_rows pos")
    assert_equal(r["out"], x.view(B, T, D)[torch.arange(B), want_pos.long()], "argmax_gather_rows out")

    dout = rand((B, D), 172, dtype=torch.float32)
    prior = rand((B * T, D), 173, dtype=torch.float32)  # the caller's zeros, as values that must survive
    c = Case("scatter_rows")
    gd, gp = c.input("dout", dout), c.input("pos", want_pos)
    dx = c.inout("dx", prior)
    r = c.run(lambda: call("b200_scatter_rows", gd.ptr(), gp.ptr(), dx.ptr(), B, T, D, S()))
    ref = prior.clone().view(B, T, D)
    ref[torch.arange(B), want_pos.long()] = dout
    assert_equal(r["dx"], ref.view(B * T, D), "scatter_rows")


# ------------------------------------------------------------------------------------------------------------------------
# losses
# ------------------------------------------------------------------------------------------------------------------------
@covers("b200_softmax_xent_fwd_bwd")
@pytest.mark.gpu
@pytest.mark.parametrize("with_mean", [False, True])
@pytest.mark.parametrize("Bn", [1, 5, 300])
@pytest.mark.parametrize("C", [13, 1000])
def test_softmax_xent_footprint(C, Bn, with_mean):
    logits = rand((Bn, C), 181, 3.0)
    labels = torch.randint(0, C, (Bn,), generator=torch.Generator().manual_seed(182))
    gs = torch.tensor([0.75], dtype=torch.float32)
    ldl = rup(C) + 8
    c = Case(f"softmax_xent B {Bn} C {C} mean {with_mean}")
    gl, glab, ggs = c.input("logits", logits, ld=ldl), c.input("labels", labels), c.input("grad_scale_dev", gs)
    rows = c.output("loss_rows", 1, Bn)
    mean = c.output("loss_mean", 1, 1) if with_mean else None
    dl = c.output("dlogits", Bn, C, ld=ldl, dtype=torch.bfloat16)
    flag = c.inout("bad_label_flag", torch.zeros(1, dtype=torch.int32))
    r = c.run(lambda: call("b200_softmax_xent_fwd_bwd", gl.ptr(), ldl, glab.ptr(), rows.ptr(), mean.ptr() if mean else None, dl.ptr(),
                           flag.ptr(), Bn, C, 2.0, ggs.ptr(), S()))
    assert r["bad_label_flag"].item() == 0
    lf = logits.double().requires_grad_(True)
    ref_rows = -F.log_softmax(lf, 1).gather(1, labels[:, None])[:, 0]
    (ref_rows.mean() * 2.0 * 0.75).backward()
    assert_close(r["loss_rows"].view(-1), ref_rows.detach(), c.name + " loss_rows", rtol=1e-5, atol_rel=1e-5)
    if with_mean:
        assert abs(r["loss_mean"].item() - ref_rows.mean().item()) < 1e-5 * max(1.0, abs(ref_rows.mean().item()))
    assert_ulp(r["dlogits"], lf.grad, c.name + " dlogits", ulps=1.01, floor=1e-3)


@covers("b200_symmetric_xent_fwd_bwd")
@pytest.mark.gpu
@pytest.mark.parametrize("Bn", [1, 5, 300])
def test_symmetric_xent_footprint(Bn):
    logits = rand((Bn, Bn), 191, 4.0)
    gs = torch.tensor([0.5], dtype=torch.float32)
    ldl = rup(Bn) + 8
    c = Case(f"symmetric_xent B {Bn}")
    gl, ggs = c.input("logits", logits, ld=ldl), c.input("grad_scale_dev", gs)
    loss = c.output("loss", 1, 1)
    dl = c.output("dlogits", Bn, Bn, ld=ldl, dtype=torch.bfloat16)
    ws = c.scratch("lse_ws", 2 * Bn)
    r = c.run(lambda: call("b200_symmetric_xent_fwd_bwd", gl.ptr(), ldl, loss.ptr(), dl.ptr(), ws.ptr(), Bn, 3.0, ggs.ptr(), S()))
    lf = logits.double().requires_grad_(True)
    tgt = torch.arange(Bn)
    ref = 0.5 * (F.cross_entropy(lf, tgt) + F.cross_entropy(lf.t(), tgt))
    (ref * 3.0 * 0.5).backward()
    assert abs(r["loss"].item() - ref.item()) < 1e-5 * max(1.0, abs(ref.item()))
    assert_ulp(r["dlogits"], lf.grad, c.name + " dlogits", ulps=1.01, floor=1e-3)


# ------------------------------------------------------------------------------------------------------------------------
# optimizer and element-wise helpers
# ------------------------------------------------------------------------------------------------------------------------
ADAM_HYPER = (1e-2, 0.8, 0.99, 1e-6, 0.05, 0.5)  # lr, beta1, beta2, eps, weight_decay, grad_scale (hyper_dev only)
ADAM_VARIANTS = ["host_step", "step_dev", "hyper_dev"]
ADAM_SIZES = [(4, "randn"), (1028, "randn"), (1028, "sweep")]
ADAM_TOL = {"params": 1e-6, "exp_avg": 1e-5, "exp_avg_sq": 1e-5}  # rtol; atol 1e-6 max |ref| for all three


def _adam_inputs(n, grads):
    """(params, grads, exp_avg, exp_avg_sq, scale) of an Adam case.  "sweep": element i's gradient and first moment times
    scale_i = 2^e_i, e_i from -40 to 40, its second moment times scale_i^2, every 7th gradient exactly 0 and every 14th element's
    moments too.  Below about 2^-20, eps dominates the denominator."""
    p0, g = rand((n,), 201, dtype=torch.float32), rand((n,), 202, dtype=torch.float32)
    m0 = rand((n,), 203, 0.1, dtype=torch.float32)
    v0 = rand((n,), 204, 0.1, dtype=torch.float32).abs()
    scale = torch.ones(n, dtype=torch.float64)
    if grads == "sweep":
        scale = torch.exp2(torch.linspace(-40, 40, n, dtype=torch.float64).round())
        g, m0, v0 = (g * scale).float(), (m0 * scale).float(), (v0 * scale * scale).float()  # exact: powers of 2
        g[::7] = 0.0
        m0[::14] = 0.0
        v0[::14] = 0.0
    return p0, g, m0, v0, scale


def _adam_steps(variant):
    """The step numbers the case's five calls run with (hyper_dev's last call does not increment: step 6 twice)."""
    return [3, 4, 5, 6, 7] if variant != "hyper_dev" else [3, 4, 5, 6, 6]


def _adam_case(n, grads, variant, decoupled):
    lr, b1, b2, eps, wd, gs = ADAM_HYPER
    p0, g, m0, v0, scale = _adam_inputs(n, grads)
    entry = "b200_adamw_step" if decoupled else "b200_adam_step"
    c = Case(f"{entry[5:]} {variant} n {n} {grads}")
    gg = c.input("grads", g)
    p, m, v = c.inout("params", p0), c.inout("exp_avg", m0), c.inout("exp_avg_sq", v0)
    step = c.inout("step_dev", torch.tensor([2], dtype=torch.int32))
    hyper = c.input("hyper", torch.tensor([lr, b1, b2, eps, wd, gs], dtype=torch.float32))

    def launch():
        for k in range(5):
            if variant == "host_step":
                call(entry, p.ptr(), gg.ptr(), m.ptr(), v.ptr(), n, lr, b1, b2, eps, wd, 3 + k, None, S())
            elif variant == "step_dev":
                call(entry, p.ptr(), gg.ptr(), m.ptr(), v.ptr(), n, lr, b1, b2, eps, wd, 0, step.ptr(), S())
            else:
                call(entry + "_dev", p.ptr(), gg.ptr(), m.ptr(), v.ptr(), n, hyper.ptr(), step.ptr(), int(k < 4), S())

    r = c.run(launch)
    want_step = {"host_step": 2, "step_dev": 7, "hyper_dev": 6}[variant]
    assert r["step_dev"].item() == want_step
    rp, rm, rv = adam(p0, g, m0, v0, _adam_steps(variant), lr, b1, b2, eps, wd, gs if variant == "hyper_dev" else 1.0,
                      decoupled=decoupled)
    assert_close(r["params"].view(-1), rp, c.name + " params", ADAM_TOL["params"], 1e-6)
    # the moments in units of their element's scale (exact), so that the sweep's small elements are held as tightly as its large ones
    assert_close(r["exp_avg"].view(-1) / scale, rm / scale, c.name + " exp_avg", ADAM_TOL["exp_avg"], 1e-6)
    assert_close(r["exp_avg_sq"].view(-1) / scale ** 2, rv / scale ** 2, c.name + " exp_avg_sq", ADAM_TOL["exp_avg_sq"], 1e-6)


@covers("b200_adam_step", "b200_adam_step_dev")
@pytest.mark.gpu
@pytest.mark.parametrize("variant", ADAM_VARIANTS)
@pytest.mark.parametrize("n,grads", ADAM_SIZES, ids=["4", "1028", "1028-sweep"])
def test_adam_footprint(n, grads, variant):
    _adam_case(n, grads, variant, decoupled=False)


@covers("b200_adamw_step", "b200_adamw_step_dev")
@pytest.mark.gpu
@pytest.mark.parametrize("variant", ADAM_VARIANTS)
@pytest.mark.parametrize("n,grads", ADAM_SIZES, ids=["4", "1028", "1028-sweep"])
def test_adamw_footprint(n, grads, variant):
    _adam_case(n, grads, variant, decoupled=True)


ADAMW_MISTAKES = ["L2 decay", "decay after the update", "no decay", "decay scaled by grad_scale", "decay using lr / bc1"]


def _adamw_mistake(p, g, m, v, steps, lr, b1, b2, eps, wd, gs, mistake):
    """AdamW in float64 with one plausible implementation mistake: the params the kernel would return."""
    if mistake == "L2 decay":
        return adam(p, g, m, v, steps, lr, b1, b2, eps, wd, gs)[0]
    p, m, v = p.double(), m.double(), v.double()
    for t in steps:
        bc1 = 1 - b1 ** t
        keep = {"decay after the update": 1.0, "no decay": 1.0, "decay scaled by grad_scale": 1 - lr * wd * gs,
                "decay using lr / bc1": 1 - lr / bc1 * wd}[mistake]
        p = p * keep
        gg = g.double() * gs
        m = b1 * m + (1 - b1) * gg
        v = b2 * v + (1 - b2) * gg * gg
        p = p - lr / bc1 * m / (v.sqrt() / math.sqrt(1 - b2 ** t) + eps)
        if mistake == "decay after the update":
            p = p * (1 - lr * wd)
    return p


@pytest.mark.parametrize("variant", ADAM_VARIANTS)
@pytest.mark.parametrize("n,grads", ADAM_SIZES[1:], ids=["1028", "1028-sweep"])
def test_adamw_footprint_tolerance_rejects_plausible_mistakes(n, grads, variant):
    """CPU: on test_adamw_footprint's own inputs, steps and tolerance, each mistake moves many params out of the bound (the decay
    scaled by grad_scale differs only where grad_scale is not 1: hyper_dev), so loosening the tolerance fails here first."""
    lr, b1, b2, eps, wd, gs = ADAM_HYPER
    gs = gs if variant == "hyper_dev" else 1.0
    p0, g, m0, v0, _ = _adam_inputs(n, grads)
    steps = _adam_steps(variant)
    ref = adam(p0, g, m0, v0, steps, lr, b1, b2, eps, wd, gs, decoupled=True)[0]
    for mistake in ADAMW_MISTAKES:
        if mistake == "decay scaled by grad_scale" and gs == 1.0:
            continue
        got = _adamw_mistake(p0, g, m0, v0, steps, lr, b1, b2, eps, wd, gs, mistake)
        caught = int((~within(got, ref, ADAM_TOL["params"], 1e-6)).sum())
        assert caught >= n // 4, f"{mistake} ({variant}, {grads}): only {caught} of {n} params outside the tolerance"


@covers("b200_cast_f32_to_bf16", "b200_fill_f32")
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3, 7, 9, 1000003])
def test_cast_fill_footprint(n):
    src = rand((n,), 211, 100.0, torch.float32)
    c = Case(f"cast_f32_to_bf16 n {n}")
    gs = c.input("src", src)
    dst = c.output("dst", 1, n, dtype=torch.bfloat16)
    r = c.run(lambda: call("b200_cast_f32_to_bf16", gs.ptr(), dst.ptr(), n, S()))
    assert_equal(r["dst"].view(-1), src.to(torch.bfloat16), c.name)
    c = Case(f"fill_f32 n {n}")
    out = c.output("dst", 1, n)
    r = c.run(lambda: call("b200_fill_f32", out.ptr(), -2.5, n, S()))
    assert_equal(r["dst"].view(-1), torch.full((n,), -2.5), c.name)


# ------------------------------------------------------------------------------------------------------------------------
# GroupNorm(32) + SiLU
# ------------------------------------------------------------------------------------------------------------------------
@covers("b200_groupnorm_silu_fwd", "b200_groupnorm_silu_bwd")
@pytest.mark.gpu
@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("silu", [0, 1])
@pytest.mark.parametrize("B,HW,C", [(3, 72, 32), (2, 4225, 320)])
def test_groupnorm_footprint(B, HW, C, silu, accumulate):
    eps = 1e-5
    x = (rand((B * HW, C), 221, 1.5, torch.float64) + 0.3).to(torch.bfloat16)
    gamma = 1.0 + 0.1 * rand((C,), 222, dtype=torch.float32)
    beta = 0.05 * rand((C,), 223, dtype=torch.float32)
    ws_n = int(_cabi.lib().b200_groupnorm_workspace_floats(B, HW, C))
    c = Case(f"groupnorm_silu_fwd {B}x{HW}x{C} silu {silu}")
    gx, gg, gb = c.input("x", x), c.input("gamma", gamma), c.input("beta", beta)
    y = c.output("y", B * HW, C, dtype=torch.bfloat16)
    mean, rstd = c.output("mean", B, 32), c.output("rstd", B, 32)
    ws = c.scratch("workspace", ws_n)
    r = c.run(lambda: call("b200_groupnorm_silu_fwd", gx.ptr(), gg.ptr(), gb.ptr(), y.ptr(), mean.ptr(), rstd.ptr(), ws.ptr(), B, HW, C,
                           eps, silu, S()))
    dy = rand((B * HW, C), 224)
    (ref, m, rs, _), (dx64, dg64, db64) = with_grads(groupnorm, (x.view(B, HW, C), gamma, beta), dy.view(B, HW, C), eps, silu)
    assert_ulp(r["y"], ref.reshape(B * HW, C), c.name + " y", ulps=1.01, floor=1e-3)
    assert_close(r["mean"], m, c.name + " mean", rtol=1e-4, atol_rel=1e-5)
    assert_close(r["rstd"], rs, c.name + " rstd", rtol=1e-4)

    pg, pb = rand((C,), 225, dtype=torch.float32), rand((C,), 226, dtype=torch.float32)
    c = Case(f"groupnorm_silu_bwd {B}x{HW}x{C} silu {silu} accumulate {accumulate}")
    gx, gdy, gg, gb = c.input("x", x), c.input("dy", dy), c.input("gamma", gamma), c.input("beta", beta)
    gm, gr = c.input("mean", r["mean"]), c.input("rstd", r["rstd"])
    dx = c.output("dx", B * HW, C, dtype=torch.bfloat16)
    dg = c.inout("dgamma", pg) if accumulate else c.output("dgamma", 1, C)
    db = c.inout("dbeta", pb) if accumulate else c.output("dbeta", 1, C)
    ws = c.scratch("workspace", ws_n)
    r = c.run(lambda: call("b200_groupnorm_silu_bwd", gx.ptr(), gdy.ptr(), gg.ptr(), gb.ptr(), gm.ptr(), gr.ptr(), dx.ptr(), dg.ptr(),
                           db.ptr(), ws.ptr(), B, HW, C, silu, accumulate, S()))
    assert_ulp(r["dx"], dx64.reshape(B * HW, C), c.name + " dx", ulps=1.01, floor=1e-3)
    prior_g = pg.double() if accumulate else 0.0
    prior_b = pb.double() if accumulate else 0.0
    assert relerr(r["dgamma"].view(-1).double() - prior_g, dg64) < 1e-4, c.name
    assert relerr(r["dbeta"].view(-1).double() - prior_b, db64) < 1e-4, c.name


# ------------------------------------------------------------------------------------------------------------------------
# CPU checks: the table covers every entry point, and the guard bookkeeping reports what it should
# ------------------------------------------------------------------------------------------------------------------------
# the modules that hold the footprint cases of the companion header's entry points (include/b200_cflearn_ext.h); importing one
# registers its @covers
EXT_CASE_MODULES = ("test_resample_gpu", "test_unet_gpu", "test_autoencoder_gpu", "test_ddpm_gpu", "test_ddim_gpu")


def test_every_compute_entry_point_has_a_footprint_case():
    for name in EXT_CASE_MODULES:
        importlib.import_module(name)
    abi = set(_cabi.SIGNATURES) | set(_cabi.EXT_SIGNATURES)
    missing = sorted(abi - NOT_FOOTPRINT - COVERED)
    assert not missing, f"C-ABI entry points without a footprint case: {missing}"
    stale = sorted(COVERED - abi) + sorted(NOT_FOOTPRINT - abi)
    assert not stale, f"names that are not C-ABI entry points: {stale}"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_guarded_view_is_16_mod_256(dtype):
    for rows, width, ld in ((1, 1, 1), (3, 13, 24), (129, 1003, 1016)):
        g = Guarded(rows, width, ld, dtype, device="cpu")
        assert g.ptr() % 256 == 16
        assert g.view.shape == (rows, width) and g.view.stride() == (ld, 1)
        es = g.flat.element_size()
        assert g.front * es >= GUARD_BYTES and (g.flat.numel() - g.front - rows * ld) * es >= GUARD_BYTES


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_guarded_reports_pokes_outside_the_view(dtype):
    rows, width, ld = 5, 13, 24
    g = Guarded(rows, width, ld, dtype, device="cpu")
    g.bits.fill_(_as_signed(SENTINEL[dtype], g.bits.dtype))
    before = g.bits.clone()
    for flat, where in ((g.front - 1, (-1, ld - 1)),                 # front guard, right before the view
                        (0, divmod(-g.front, ld)),                    # the first element of the allocation
                        (g.front + 2 * ld + width, (2, width)),       # a padding column
                        (g.front + rows * ld - 1, (rows - 1, ld - 1)),  # the tail of the last row
                        (g.front + rows * ld, (rows, 0)),             # the back guard
                        (g.flat.numel() - 1, divmod(g.flat.numel() - 1 - g.front, ld))):
        g.bits.copy_(before)
        g.bits[flat] = 0
        assert g.outside_changed(before) == where, (flat, where)
    g.bits.copy_(before)
    for r, col in ((0, 0), (rows - 1, width - 1), (2, 7)):  # inside the view: not an outside write
        g.view[r, col] = 1.0
        assert g.outside_changed(before) is None
    assert g.unwritten(SENTINEL[dtype]) == (0, 1)
    g.view.fill_(0.0)
    assert g.unwritten(SENTINEL[dtype]) is None
