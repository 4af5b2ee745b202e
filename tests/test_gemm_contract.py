"""The argument contract of b200_gemm_bf16 and b200_conv3x3_nhwc_bf16 (include/b200_cflearn.h), checked without a GPU.

Every refusal happens before a tensor map is encoded, so it is the same with or without a device.  The pointers are fake and
never dereferenced: refused calls stop at the argument checks.  A call that passes them reaches B200_ERR_DRIVER on a machine
without a GPU; the matrices that make such calls run only there, so no kernel ever sees a fake pointer."""
import itertools
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import _cabi, ops  # noqa: E402

ARG, ALIGN, DRIVER = -1, -2, -3
FAKE = 1 << 20
ODD = FAKE + 8        # not 16-byte aligned
ODD_BIAS = FAKE + 2   # not 4-byte aligned
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="accepted calls would launch kernels on fake pointers")

GEMM, CONV = "gemm", "conv3x3"
ALL_MAJORS = {(0, 0), (0, 1), (1, 0), (1, 1)}
# Per public epilogue, from the header: entry points, (a_mn_major, b_mn_major) pairs, bias rule ("optional", "ignored",
# "none" = must be NULL, "pair" = required and 4-byte aligned), aux required, out1 required, N = 2F with F % 8 == 0,
# out0 fp32, split-K.
CONTRACT = {
    0: ({GEMM, CONV}, ALL_MAJORS, "optional", False, False, False, False, False),
    1: ({GEMM}, {(0, 0)}, "optional", False, True, False, False, False),
    2: ({GEMM, CONV}, {(0, 0)}, "optional", True, False, False, True, False),
    3: ({GEMM}, {(0, 1)}, "ignored", True, False, False, False, False),
    4: ({GEMM}, {(1, 1)}, "ignored", False, False, False, True, True),
    5: ({GEMM}, {(0, 0)}, "optional", False, True, False, False, False),
    6: ({GEMM}, {(0, 1)}, "ignored", True, False, False, False, False),
    7: ({GEMM}, {(0, 0)}, "pair", False, True, True, False, False),
    8: ({GEMM}, {(0, 1)}, "none", True, False, True, False, False),
    9: ({GEMM}, {(0, 0)}, "optional", True, False, False, False, False),
    10: ({CONV}, {(0, 0)}, "optional", True, False, False, False, False),
    11: ({CONV}, {(0, 0)}, "optional", True, False, False, False, False),
}


def expected(entry, epi, majors, bias, out0, out1, aux, N, ldo, splits):
    """The statuses the contract allows for one call: the codes of every rule it breaks, or DRIVER if it breaks none."""
    if epi not in CONTRACT:
        return {ARG}
    entries, ok_majors, bias_rule, need_aux, need_out1, n2f, f32, splitk = CONTRACT[epi]
    arg = [
        entry not in entries,
        majors not in ok_majors,
        splits != 1 and not splitk,
        n2f and N % 16 != 0,
        ldo < N,
        need_out1 and out1 is None,
        need_aux and aux is None,
        bias_rule == "none" and bias is not None,
        bias_rule == "pair" and (bias is None or bias % 4 != 0),
    ]
    align = [(ldo * (4 if f32 else 2)) % 16 != 0, any(p is not None and p % 16 != 0 for p in (out0, out1, aux))]
    return ({ARG} if any(arg) else set()) | ({ALIGN} if any(align) else set()) or {DRIVER}


def gemm(epi, majors=(0, 0), bias=FAKE, out0=FAKE, out1=FAKE, aux=FAKE, N=2560, ldo=2560, splits=1):
    return _cabi.lib().b200_gemm_bf16(FAKE, 320, majors[0], FAKE, 320, majors[1], 4096, N, 320, epi, bias, out0, out1, aux, ldo,
                                      splits, 0, None)


def conv(epi, bias=FAKE, out0=FAKE, aux=FAKE, Cout=320, ldo=320, B=2, H=16, W=16, Cin=320):
    return _cabi.lib().b200_conv3x3_nhwc_bf16(FAKE, FAKE, bias, out0, aux, ldo, B, H, W, Cin, Cout, epi, None)


POINTERS = (FAKE, None, ODD)
# (N, ldo): valid; ldo < N; ldo rows not 16-byte aligned in bf16 (and F % 8 != 0); F % 8 != 0 with aligned rows
WIDTHS = ((2560, 2560), (2560, 2552), (2556, 2556), (2568, 2568))


@no_device
def test_gemm_statuses_follow_the_header():
    for epi, majors, bias, out0, out1, aux, (N, ldo), splits in itertools.product(
            range(-1, 13), sorted(ALL_MAJORS), (FAKE, None, ODD_BIAS), (FAKE, ODD), POINTERS, POINTERS, WIDTHS, (1, 2)):
        got = gemm(epi, majors, bias, out0, out1, aux, N, ldo, splits)
        want = expected(GEMM, epi, majors, bias, out0, out1, aux, N, ldo, splits)
        assert got in want, (epi, majors, bias, out0, out1, aux, N, ldo, splits, got, _cabi.last_error())


@no_device
def test_conv3x3_statuses_follow_the_header():
    for epi, bias, out0, aux, (Cout, ldo) in itertools.product(
            range(-1, 13), (FAKE, None, ODD_BIAS), (FAKE, ODD), POINTERS, ((320, 320), (320, 312), (316, 324))):
        got = conv(epi, bias, out0, aux, Cout, ldo)
        want = expected(CONV, epi, (0, 0), bias, out0, None, aux, Cout, ldo, 1)
        assert got in want, (epi, bias, out0, aux, Cout, ldo, got, _cabi.last_error())


@no_device
def test_ops_table_agrees_with_the_c_side():
    """ops.EPILOGUES and the library agree on which epilogues take aux / out1 and on out0's element size."""
    assert sorted(ops.EPILOGUES) == sorted(CONTRACT)
    for epi, (dtype, aux_kind, out1_kind) in ops.EPILOGUES.items():
        majors = sorted(CONTRACT[epi][1])[0]
        if CONTRACT[epi][0] == {CONV}:
            assert aux_kind is not None and out1_kind is None
            assert conv(epi) == DRIVER
            assert conv(epi, aux=None) == ARG
            continue
        assert gemm(epi, majors, bias=None if epi == ops.EPI_DGEGLU_BF16 else FAKE) == DRIVER, epi
        call = lambda **kw: gemm(epi, majors, bias=None if epi == ops.EPI_DGEGLU_BF16 else FAKE, **kw)  # noqa: E731
        assert (call(aux=None) == ARG) == (aux_kind is not None), epi
        assert (call(out1=None) == ARG) == (out1_kind is not None), epi
        # rows of 20 elements are 80 bytes in fp32 (16-byte aligned) and 40 in bf16 (not)
        assert (call(N=16, ldo=20) == DRIVER) == (dtype == torch.float32), epi
        assert (aux_kind == "image") == (epi == ops.EPI_BIAS_ADD_PER_IMAGE_BF16)
        assert (out1_kind == "dense") == (epi == ops.EPI_BIAS_GEGLU_BF16)


def test_geglu_and_bf16_residual_refusals():
    G, DG, R = ops.EPI_BIAS_GEGLU_BF16, ops.EPI_DGEGLU_BF16, ops.EPI_BIAS_RESID_BF16
    assert gemm(G, out1=None) == -1 and "out1" in _cabi.last_error()
    assert gemm(G, bias=None) == -1 and "bias" in _cabi.last_error()
    assert gemm(G, N=2568) == -1 and gemm(DG, N=2568, majors=(0, 1), bias=None) == -1  # F = 1284 is not a multiple of 8
    assert gemm(DG, aux=None, majors=(0, 1), bias=None) == -1 and gemm(R, aux=None) == -1
    assert gemm(DG, bias=None) == -1 and gemm(G, majors=(0, 1)) == -1 and gemm(R, majors=(1, 0)) == -1  # majors
    assert gemm(DG, majors=(0, 1)) == -1  # no bias in the backward
    assert gemm(G, ldo=2552) == -1 and gemm(R, N=2556, ldo=2556) == -2
    assert gemm(G, out1=ODD) == -2 and gemm(DG, aux=ODD, majors=(0, 1), bias=None) == -2 and gemm(R, out0=ODD) == -2
    assert "aligned" in _cabi.last_error()


def test_resblock_conv_epilogue_refusals():
    for epi in (ops.EPI_BIAS_ADD_PER_IMAGE_BF16, ops.EPI_BIAS_RESID_CLAMP_BF16):
        assert conv(epi, aux=None) == -1 and "aux" in _cabi.last_error()
        assert conv(epi, aux=ODD) == -2 and conv(epi, out0=ODD) == -2 and "aligned" in _cabi.last_error()
        assert conv(epi, ldo=312) == -1 and conv(epi, ldo=324, Cout=316) == -2
        assert conv(epi, Cin=96) == -1 and conv(epi, W=48) == -1 and conv(epi, B=0) == -1  # sizes
        # the plain GEMM entry refuses both
        assert _cabi.lib().b200_gemm_bf16(FAKE, 320, 0, FAKE, 320, 0, 4096, 320, 320, epi, FAKE, FAKE, None, FAKE, 320, 1, 0, None) == -1
        assert "conv3x3" in _cabi.last_error()
    assert conv(12) == -1 and "epilogue" in _cabi.last_error()
