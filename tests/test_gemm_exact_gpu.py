"""The GEMM and the implicit-GEMM 3x3 convolution bit for bit, on operands whose every product and partial sum is exact in fp32.

The operands (``_refs.exact_operands``) are small integers times a power of two per row of A and per column of B (per image and
output channel for the convolution), so the accumulator holds the float64 value exactly and t = bf16(acc + bias) is fixed to the
bit: an accumulator narrower than fp32, a bf16 rounding between k-blocks or split planes, a missed or repeated k-block, a wrong
row, column, tap, image or bias, or ties rounded away from zero all change some bit.  Exponents of 2^+-20 per row, column, image
and channel make a value that leaks across a boundary differ by orders of magnitude.  Cancellation cases add products of +-2^20
units that cancel inside one k16 step, across two k-blocks or across two splits, next to the small terms.  Outputs that are
transcendental functions of t are checked within the GELU tests' ulp bounds of float64 of the exact t.  An exact zero sum is +0
in the kernels (the accumulator starts from +0), so the references add +0 to theirs, which turns float64's -0 into +0.

Every operand row is padded with NaN past K or N (and NaN rows follow the last one), so a read past an edge reaches an output.
Every case runs on all SMs, on one CTA and on three, and the three results must be bit-identical.  ``test_gemm_exact.py`` checks,
on the CPU, that this sweep's shapes cross every tile edge: an emulation of the kernels' index maps with one local mistake each
fails somewhere in it.  Run on an H100: pytest -m gpu."""
import math

import pytest
import torch

import cflearn_b200  # noqa: F401  (registers the package)
from cflearn_b200 import _cabi, ops
from _refs import (bf16, conv3x3, conv3x3_dgrad, conv3x3_wgrad, exact_conv_operands, exact_operands, exact_wgrad_operands, exponents,
                   cancel_pairs, gemm_epilogue, gemm_t, relerr, splitk_ranges)

DEV = "cuda"
GRIDS = (0, 1, 3)  # all SMs, one CTA, three CTAs
_BITS = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}

# ---- the sweep -------------------------------------------------------------------------------------------------------------------------
MS = (1, 63, 64, 65, 127, 128, 129, 257)
NS = (1, 7, 8, 9, 255, 256, 257, 264, 513)
KS = (1, 8, 63, 64, 65, 136, 4104)
FS = (8, 120, 128, 136, 264)
GEMM_EPIS = [(0, 0, 0), (0, 0, 1), (0, 1, 0), (0, 1, 1), (1, 0, 0), (2, 0, 0), (3, 0, 1), (4, 1, 1), (5, 0, 0), (6, 0, 1), (7, 0, 0),
             (8, 0, 1), (9, 0, 0)]
LINEAR = (0, 2, 4, 9)  # epilogues whose outputs are linear in acc: exponents of 2^+-20; the GELU family keeps t near 1


def gemm_cases(epi):
    """(M, N, K, splits, cancel) of one epilogue.  N is the C-ABI's N (2F for GEGLU).  Every M, N (F) and K of the lists above, each
    epilogue pairing them differently; K = 9 x 2560 with cancellation; one shape of more 128 x 256 tiles than the 132 SMs."""
    geglu = epi in (7, 8)
    ns = [2 * f for f in FS] * 2 if geglu else NS
    split_list = (1, 2, 3, "pick")
    cases = []
    for i, n in enumerate(ns[:9]):
        M, K = MS[(i + epi) % len(MS)], KS[(i + 2 * epi) % len(KS)]
        cases.append((M, n, K, split_list[i % 4] if epi == 4 else 1, None))
    big_k = 9 * 2560
    cases.append((MS[epi % 8], 2 * FS[epi % 5] if geglu else NS[(epi + 3) % 9], big_k, 2 if epi == 4 else 1, "k16"))
    cases.append((MS[(epi + 5) % 8], 2 * FS[(epi + 2) % 5] if geglu else NS[(epi + 6) % 9], 4104, 3 if epi == 4 else 1, "kblock"))
    cases.append((65, 2 * 136 if geglu else 257, 4104, "pick" if epi == 4 else 1, "split"))
    cases.append((2176, 4096 if epi == 8 else 2048, 64, 3 if epi == 4 else 1, None))  # 17 x 8 = 136 tiles
    return cases


# conv forward (B, H, W, Cin, Cout, epilogue): every admitted W at H = 1 and at two tiles per image, H W in {16, 32, 64} with B not a
# multiple of the images per tile, W < H rectangles, Cin in {64, 320, 2560}, Cout in {8, 72, 256, 264, 1280}
CONV_CASES = [
    (3, 1, 1, 64, 72, 0), (2, 256, 1, 64, 8, 2), (5, 1, 2, 320, 264, 10), (1, 128, 2, 64, 256, 11), (3, 1, 4, 2560, 8, 0),
    (2, 64, 4, 64, 72, 10), (3, 1, 8, 64, 1280, 2), (1, 32, 8, 320, 72, 0), (2, 1, 16, 64, 264, 11), (2, 16, 16, 64, 8, 2),
    (3, 1, 32, 320, 8, 10), (1, 8, 32, 64, 256, 0), (2, 1, 64, 64, 72, 2), (1, 4, 64, 2560, 72, 11), (3, 1, 128, 64, 8, 10),
    (2, 2, 128, 64, 264, 0), (3, 4, 4, 64, 1280, 11), (5, 4, 8, 320, 72, 2), (3, 8, 8, 64, 264, 10), (3, 8, 4, 64, 72, 0),
    (1, 4, 4, 2560, 256, 2),
]
# input gradient through pack_conv3x3_weight_dgrad (B, H, W, Cin, Cout): the call's input channels are Cout, a multiple of 64
DGRAD_CASES = [(2, 16, 8, 72, 64), (3, 4, 4, 8, 256), (1, 8, 32, 264, 1280), (2, 1, 128, 320, 64), (3, 1, 2, 72, 128)]
# weight gradient (B, H, W, Cin, Cout, splits): every W dividing 64 with H W % 64 == 0, Cout across the 128-row tile edge
WGRAD_CASES = [(1, 64, 1, 64, 8, 1), (2, 32, 2, 64, 72, 2), (1, 16, 4, 320, 128, 3), (3, 8, 8, 64, 136, "pick"), (2, 4, 16, 64, 264, 2),
               (1, 2, 32, 320, 8, 3), (2, 1, 64, 64, 72, "pick"), (2, 16, 8, 64, 264, 1)]


def gemm_exponents(epi, M, N, K, seed):
    """Row exponents of A and of B: 2^+-20 for the linear epilogues; otherwise +-1 around the scale that makes t of order 1."""
    if epi in LINEAR:
        return exponents(M, -20, 20, seed), exponents(N, -20, 20, seed + 1)
    q = max(q for q in (1, 3, 7, 15) if K * q * q <= 2 ** 20)
    base = -round(math.log2(max(1.0, math.sqrt(K) * q * q / 3)))
    return exponents(M, base // 2 - 1, base // 2 + 1, seed), exponents(N, base - base // 2 - 1, base - base // 2 + 1, seed + 1)


def gemm_inputs(epi, M, N, K, cancel, seed, with_bias=True):
    """The operands of one case (CPU): A [M, K], B [cols, K] (cols = F for dGEGLU), bias (required by GEGLU, else with_bias) or None,
    aux or None."""
    cols = N // 2 if epi == 8 else N
    ea, eb = gemm_exponents(epi, M, cols, K, seed)
    A, B = exact_operands(M, cols, K, ea, eb, cancel_pairs(K, cancel), seed)
    g = torch.Generator().manual_seed(seed + 2)
    bias = None
    if epi == 7 or (epi in (0, 1, 2, 5, 9) and with_bias):
        q = 127 if epi in LINEAR else 15
        bias = (torch.randint(-q, q + 1, (N,), generator=g).to(torch.float64) * torch.exp2(eb)).to(torch.bfloat16)
    aux = None
    if epi in (2, 9):
        scale = torch.exp2(ea[:, None] + eb[None, :] + round(math.log2(max(1.0, math.sqrt(K)))))
        aux = (torch.randn(M, N, generator=g, dtype=torch.float64) * scale).to(torch.float32 if epi == 2 else torch.bfloat16)
    elif epi in (3, 6, 8):
        aux = torch.randn(M, N, generator=g, dtype=torch.float64).mul(1.5).to(torch.bfloat16)
    return A, B, bias, aux


# ---- buffers with NaN around every operand -------------------------------------------------------------------------------------
def _nan_rows(t, ld, extra_rows=64):
    """``t`` [rows, cols] on the device inside a NaN-filled [rows + extra_rows, ld] buffer: the view [rows, cols]."""
    buf = torch.full((t.shape[0] + extra_rows, ld), float("nan"), dtype=t.dtype, device=DEV)
    buf[: t.shape[0], : t.shape[1]] = t.to(DEV)
    return buf[: t.shape[0], : t.shape[1]]


def _nan_flat(t, pad=4096):
    """``t`` contiguous on the device with NaN in the ``pad`` elements before and after it (16-byte aligned)."""
    buf = torch.full((t.numel() + 2 * pad,), float("nan"), dtype=t.dtype, device=DEV)
    buf[pad:pad + t.numel()] = t.reshape(-1).to(DEV)
    return buf[pad:pad + t.numel()].view(t.shape)


def _rup(n, m=8):
    return (n + m - 1) // m * m


SENT = {torch.bfloat16: 0x7FA5, torch.float32: 0x7FA5A5A5}


def _sentinel_rows(rows, cols, ld, dtype):
    """[rows, cols] view of a [rows + 8, ld] buffer whose every element holds a NaN payload no kernel writes."""
    buf = torch.empty((rows + 8, ld), dtype=dtype, device=DEV)
    buf.view(_BITS[dtype]).fill_(SENT[dtype])
    return buf[:rows, :cols]


def _untouched(view, what):
    """The buffer behind ``view`` (a _sentinel_rows view) still holds the sentinel outside the view."""
    base = view._base
    bits = base.view(_BITS[base.dtype])
    inside = torch.zeros_like(bits, dtype=torch.bool)
    inside[: view.shape[0], : view.shape[1]] = True
    bad = (bits != SENT[base.dtype]) & ~inside
    assert not bad.any(), f"{what}: written outside the output at (row, col) {tuple(torch.nonzero(bad)[0].tolist())}"


# ---- comparisons ----------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.view(_BITS[t.dtype]).long() & ((1 << (8 * t.element_size())) - 1)


def _locate_gemm(r, c):
    return f"(tile ({r // 128}, {c // 256}), row {r % 128}, col {c % 256})"


def _locate_conv(H, W):
    def where(r, c):
        b, p = divmod(r, H * W)
        return f"(image {b}, y {p // W}, x {p % W}, channel {c})"
    return where


def assert_exact(got, want, what, where=_locate_gemm):
    """Bit for bit; the message names the first bad element and both bit patterns."""
    got = got.reshape(want.shape[0], -1)
    want = want.reshape(got.shape).to(got.device)
    bad = _bits(got) != _bits(want.to(got.dtype))
    if bad.any():
        r, c = torch.nonzero(bad)[0].tolist()
        n = int(bad.sum())
        raise AssertionError(f"{what}: {n} elements differ, first at {where(r, c)}: got {got[r, c].item()!r} "
                             f"(0x{_bits(got)[r, c].item():x}), expected {want[r, c].item()!r} (0x{_bits(want.to(got.dtype))[r, c].item():x})")


def assert_within(got, want, tol, what, where=_locate_gemm):
    got = got.reshape(want.shape[0], -1).to(torch.float64)
    want, tol = want.to(got.device), tol.to(got.device)
    bad = ~((got - want).abs() <= tol)
    if bad.any():
        r, c = torch.nonzero(bad)[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} elements outside the bound, first at {where(r, c)}: got {got[r, c].item()!r}, "
                             f"expected {want[r, c].item()!r} +- {tol[r, c].item():.3g}")


def check_outputs(outs, expected, what, where=_locate_gemm):
    for name, (want, tol) in expected.items():
        if tol is None:
            assert_exact(outs[name], want, f"{what} {name}", where)
        else:
            assert_within(outs[name], want, tol, f"{what} {name}", where)


def same_bits(runs, what):
    """Every run's outputs are bit-identical to the first's."""
    for grid, outs in runs[1:]:
        for name, t in outs.items():
            assert torch.equal(_bits(t), _bits(runs[0][1][name])), f"{what}: {name} at grid {grid} differs from grid {runs[0][0]}"


# ---- GEMM ---------------------------------------------------------------------------------------------------------------------------
def run_gemm(epi, a_mn, b_mn, A, B, bias, aux, splits, max_ctas):
    """One C-ABI call with every operand in NaN-padded rows; the outputs' [M, N] views (planes for EPI 4)."""
    M, K = A.shape
    cols = B.shape[0]
    N = 2 * cols if epi == 8 else cols
    a = _nan_rows(A.t() if a_mn else A, _rup(M if a_mn else K) + 8)
    b = _nan_rows(B.t() if b_mn else B, _rup(cols if b_mn else K) + 8)
    ldo = _rup(N) + 8
    f32 = epi in (2, 4)
    dtype = torch.float32 if f32 else torch.bfloat16
    s = len(splitk_ranges(K, splits)) if epi == 4 else 1
    out0 = _sentinel_rows(s * M, N, ldo, dtype)
    out1 = None
    if epi in (1, 5):
        out1 = _sentinel_rows(M, N, ldo, torch.bfloat16)
    if epi == 7:  # dense [M, F]
        out1 = _sentinel_rows(M, N // 2, N // 2, torch.bfloat16)
    bias_d = None
    if bias is not None:
        bias_d = torch.full((_rup(N) + 8,), float("nan"), dtype=torch.bfloat16, device=DEV)
        bias_d[:N] = bias.to(DEV)
    aux_d = _nan_rows(aux, ldo) if aux is not None else None
    _cabi.call("b200_gemm_bf16", a.data_ptr(), a.stride(0), a_mn, b.data_ptr(), b.stride(0), b_mn, M, N, K, epi,
               bias_d.data_ptr() if bias_d is not None else None, out0.data_ptr(), out1.data_ptr() if out1 is not None else None,
               aux_d.data_ptr() if aux_d is not None else None, ldo, splits, max_ctas, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    outs = {"out0": out0}
    if out1 is not None:
        outs["out1"] = out1
    for name, t in outs.items():
        _untouched(t, f"epilogue {epi} {name}")
    return outs


def gemm_expected(epi, A, B, bias, aux, splits, device=DEV):
    """The float64 reference of every output of one case, computed on ``device``."""
    Ad, Bd = A.to(device, torch.float64), B.to(device, torch.float64)
    if epi == 4:
        planes = torch.cat([Ad[:, k0:k1] @ Bd[:, k0:k1].t() for k0, k1 in splitk_ranges(A.shape[1], splits)]) + 0.0
        return {"out0": (planes.float(), None)}
    acc = Ad @ Bd.t() + 0.0
    t = gemm_t(acc, None if bias is None else bias.to(device)) if epi not in (3, 6, 8) else bf16(acc)
    return gemm_epilogue(epi, t, None if aux is None else aux.to(device))


@pytest.mark.gpu
@pytest.mark.parametrize("epi,a_mn,b_mn", GEMM_EPIS, ids=lambda v: str(v))
def test_gemm_exact(epi, a_mn, b_mn):
    for i, (M, N, K, splits, cancel) in enumerate(gemm_cases(epi)):
        if splits == "pick":
            splits = ops.pick_splits(M, N, K)
        what = f"epilogue {epi} majors ({a_mn}, {b_mn}) M {M} N {N} K {K} splits {splits} cancel {cancel}"
        A, B, bias, aux = gemm_inputs(epi, M, N, K, cancel, seed=1000 * epi + 10 * i, with_bias=i % 2 == 0)
        expected = gemm_expected(epi, A, B, bias, aux, splits)
        runs = [(g, run_gemm(epi, a_mn, b_mn, A, B, bias, aux, splits, g)) for g in GRIDS]
        check_outputs(runs[0][1], expected, what)
        same_bits(runs, what)


@pytest.mark.gpu
@pytest.mark.parametrize("round_bf16,accumulate", [(False, False), (True, False), (True, True)])
def test_wgrad_and_splitk_reduce_exact(round_bf16, accumulate):
    """ops.wgrad (split-K partials, then b200_splitk_reduce) over 4104 tokens: the planes' fp32 sum is exact, so is its bf16 rounding
    and the fp32 add to a prior gradient."""
    M, n_out, k_in = 4104, 264, 520
    ea, eb = exponents(n_out, -20, 20, 7), exponents(k_in, -20, 20, 8)
    dyt, xt = exact_operands(n_out, k_in, M, ea, eb, cancel_pairs(M, "split"), seed=9)
    dy, x = _nan_rows(dyt.t(), _rup(n_out) + 8), _nan_rows(xt.t(), _rup(k_in) + 8)
    exact = dyt.to(DEV, torch.float64) @ xt.to(DEV, torch.float64).t() + 0.0
    want = exact.float()
    if round_bf16:
        want = want.to(torch.bfloat16).float()
    prior = (torch.randn(n_out, k_in, generator=torch.Generator().manual_seed(10)) * 2.0 ** 10).to(DEV)
    out = prior.clone()
    ops.wgrad(dy, x, out, round_bf16=round_bf16, accumulate=accumulate)
    torch.cuda.synchronize()
    assert_exact(out, want + prior if accumulate else want, f"wgrad round_bf16={round_bf16} accumulate={accumulate}")


# ---- convolution --------------------------------------------------------------------------------------------------------------------
def _with_ctas(n, fn):
    """``fn()`` with the persistent grid bounded to n CTAs (0: all SMs) for its one launch."""
    lib = _cabi.lib()
    old = lib.b200_set_persistent_ctas(n, 1 if n else 0)
    try:
        return fn()
    finally:
        lib.b200_set_persistent_ctas(old, 0)


def run_conv(x, wp, bias, aux, epi, Cout, ctas):
    B, H, W, Cin = x.shape
    M = B * H * W
    xd, wd = _nan_flat(x), _nan_rows(wp, wp.shape[1])
    ldo = _rup(Cout) + 8
    out = _sentinel_rows(M, Cout, ldo, torch.float32 if epi == 2 else torch.bfloat16)
    bias_d = None
    if bias is not None:
        bias_d = torch.full((_rup(Cout) + 8,), float("nan"), dtype=torch.bfloat16, device=DEV)
        bias_d[:Cout] = bias.to(DEV)
    aux_d = _nan_rows(aux, ldo) if aux is not None else None
    _with_ctas(ctas, lambda: _cabi.call("b200_conv3x3_nhwc_bf16", xd.data_ptr(), wd.data_ptr(), bias_d.data_ptr() if bias_d is not None else None,
                                        out.data_ptr(), aux_d.data_ptr() if aux_d is not None else None, ldo, B, H, W, Cin, Cout, epi,
                                        torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    _untouched(out, f"conv3x3 epilogue {epi} out0")
    return {"out0": out}


def conv_inputs(B, H, W, Cin, Cout, epi, seed):
    ex, ew = exponents(B, -20, 20, seed), exponents(Cout, -20, 20, seed + 1)
    x, w = exact_conv_operands(B, H, W, Cin, Cout, ex, ew, seed)
    g = torch.Generator().manual_seed(seed + 2)
    bias = (torch.randint(-127, 128, (Cout,), generator=g).to(torch.float64) * torch.exp2(ew)).to(torch.bfloat16)
    scale = torch.exp2(ex.repeat_interleave(H * W)[:, None] + ew[None, :] + round(math.log2(math.sqrt(9 * Cin))))
    aux = None
    if epi == 2:
        aux = (torch.randn(B * H * W, Cout, generator=g, dtype=torch.float64) * scale).float()
    elif epi == 10:
        aux = (torch.randn(B, Cout, generator=g, dtype=torch.float64) * scale[:: H * W]).to(torch.bfloat16)
    elif epi == 11:
        aux = (torch.randn(B * H * W, Cout, generator=g, dtype=torch.float64) * scale).to(torch.bfloat16)
        # the sums of pixel 0, channel 0 and of the last pixel, last channel overflow: clamped to +-bf16 max
        bias[0], bias[Cout - 1] = 2e38, -2e38
        aux[0, 0], aux[-1, -1] = 3e38, -3e38
    return x, w, bias, aux


def conv_expected(epi, x, w, bias, aux, device=DEV):
    """The float64 reference of the forward convolution's output, computed on ``device``."""
    HW = x.shape[1] * x.shape[2]
    t = gemm_t(conv3x3(x.to(device), w.to(device)) + 0.0, bias.to(device))
    aux_rows = None if aux is None else aux.to(device).repeat_interleave(HW, 0) if epi == 10 else aux.to(device)
    return gemm_epilogue(epi, t, aux_rows)


def dgrad_inputs(B, H, W, Cin, Cout):
    """(dy [B, H, W, Cout], w [Cout, Cin, 3, 3]): dy scaled per image, w per input channel (the dgrad call's output channel)."""
    seed = 7 * B * H * W + Cin + Cout
    ey, ew = exponents(B, -20, 20, seed), exponents(Cin, -20, 20, seed + 1)
    dy, wt = exact_conv_operands(B, H, W, Cout, Cin, ey, ew, seed)  # wt [Cin, Cout, 3, 3]: the weights the dgrad call applies
    return dy, wt.flip(2, 3).transpose(0, 1).contiguous()


def wgrad_inputs(B, H, W, Cin, Cout):
    """(x [B, H, W, Cin], dy [B H W, Cout]): x scaled per input channel, dy per output channel."""
    seed = 3 * B * H * W + Cin + Cout
    return exact_wgrad_operands(B, H, W, Cin, Cout, exponents(Cin, -20, 20, seed), exponents(Cout, -20, 20, seed + 1)[None, :], seed)


def wgrad_planes(x, dy, splits):
    """float64 split-K planes [s Cout, 9 Cin] of the convolution's weight gradient, on x's device."""
    planes = []
    for k0, k1 in splitk_ranges(dy.shape[0], splits):
        part = torch.zeros_like(dy, dtype=torch.float64)
        part[k0:k1] = dy[k0:k1].double()
        planes.append(conv3x3_wgrad(part, x))
    return torch.cat(planes) + 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,Cin,Cout,epi", CONV_CASES, ids=lambda v: str(v))
def test_conv3x3_exact(B, H, W, Cin, Cout, epi):
    what = f"conv3x3 epilogue {epi} B {B} H {H} W {W} Cin {Cin} Cout {Cout}"
    x, w, bias, aux = conv_inputs(B, H, W, Cin, Cout, epi, seed=B * H * W + Cin + Cout + epi)
    expected = conv_expected(epi, x, w, bias, aux)
    wp = ops.pack_conv3x3_weight(w)
    runs = [(c, run_conv(x, wp, bias, aux, epi, Cout, c)) for c in GRIDS]
    check_outputs(runs[0][1], expected, what, _locate_conv(H, W))
    same_bits(runs, what)


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,Cin,Cout", DGRAD_CASES, ids=lambda v: str(v))
def test_conv3x3_dgrad_exact(B, H, W, Cin, Cout):
    """dx = the forward call on dy with pack_conv3x3_weight_dgrad(w), against float64 conv_transpose2d.  dy is scaled per image and w
    per input channel (the dgrad call's output channel)."""
    what = f"conv3x3 dgrad B {B} H {H} W {W} Cin {Cin} Cout {Cout}"
    dy, w = dgrad_inputs(B, H, W, Cin, Cout)
    expected = {"out0": (bf16(conv3x3_dgrad(dy.to(DEV), w.to(DEV)) + 0.0), None)}
    wp = ops.pack_conv3x3_weight_dgrad(w)
    runs = [(c, run_conv(dy, wp, None, None, 0, Cin, c)) for c in GRIDS]
    check_outputs(runs[0][1], expected, what, _locate_conv(H, W))
    same_bits(runs, what)


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,Cin,Cout,splits", WGRAD_CASES, ids=lambda v: str(v))
def test_conv3x3_wgrad_exact(B, H, W, Cin, Cout, splits):
    """The split-K planes of b200_conv3x3_wgrad_nhwc_bf16, and ops.conv3x3_wgrad with and without round_bf16, bit for bit."""
    M = B * H * W
    if splits == "pick":
        splits = ops.pick_splits(Cout, 9 * Cin, M)
    what = f"conv3x3 wgrad B {B} H {H} W {W} Cin {Cin} Cout {Cout} splits {splits}"
    x, dy = wgrad_inputs(B, H, W, Cin, Cout)
    xd, dyd = x.to(DEV), dy.to(DEV)
    want = wgrad_planes(xd, dyd, splits).float()
    nplanes = want.shape[0] // Cout
    tap = lambda r, c: f"(plane {r // Cout}, out channel {r % Cout}, tap {c // Cin}, in channel {c % Cin})"  # noqa: E731
    runs = []
    for c in GRIDS:
        xn, dyn = _nan_flat(x), _nan_rows(dy, _rup(Cout) + 8)
        part = _sentinel_rows(nplanes * Cout, 9 * Cin, 9 * Cin, torch.float32)
        _with_ctas(c, lambda: _cabi.call("b200_conv3x3_wgrad_nhwc_bf16", dyn.data_ptr(), dyn.stride(0), xn.data_ptr(), part.data_ptr(),
                                         B, H, W, Cin, Cout, splits, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        _untouched(part, what)
        runs.append((c, {"planes": part}))
    assert_exact(runs[0][1]["planes"], want, what, tap)
    same_bits(runs, what)
    exact = conv3x3_wgrad(dyd, xd) + 0.0
    for rnd in (False, True):
        got = ops.conv3x3_wgrad(dyd.view(B, H, W, Cout), xd, round_bf16=rnd)
        torch.cuda.synchronize()
        assert_exact(got, exact.float().to(torch.bfloat16).float() if rnd else exact.float(), f"{what} ops.conv3x3_wgrad round_bf16={rnd}", tap)


# ---- precision on random operands ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["K16384", "vit_b16_wgrad"])
def test_precision_on_random_operands(shape):
    """Random bf16 operands: relative L2 error against float64 within 1.5x that of torch's fp32 GEMM (TF32 off) rounded to bf16 once."""
    g = torch.Generator().manual_seed(11)
    if shape == "K16384":
        a = torch.randn(512, 16384, generator=g).to(torch.bfloat16).to(DEV)
        b = torch.randn(768, 16384, generator=g).to(torch.bfloat16).to(DEV)
        got = ops.gemm(a, b).float()
        ref = a.double() @ b.double().t()
        x32, y32 = a.float(), b.float().t()
    else:  # the ViT-B/16 weight gradient of a 768 -> 768 projection over 256 images of 197 tokens
        dy = torch.randn(50432, 768, generator=g).to(torch.bfloat16).to(DEV)
        x = torch.randn(50432, 768, generator=g).to(torch.bfloat16).to(DEV)
        got = ops.wgrad(dy, x, torch.empty(768, 768, device=DEV), round_bf16=True)
        ref = dy.double().t() @ x.double()
        x32, y32 = dy.float().t(), x.float()
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        eager = (x32 @ y32).to(torch.bfloat16)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    torch.cuda.synchronize()
    e_ours, e_eager = relerr(got, ref), relerr(eager, ref)
    print(f"precision {shape}: relative L2 {e_ours:.4e}, eager floor {e_eager:.4e}, ratio {e_ours / e_eager:.4f}")
    assert e_ours <= 1.5 * e_eager, f"{shape}: relative L2 {e_ours:.3e}, fp32 GEMM rounded once {e_eager:.3e}"
