"""The argument contract of the six attention entry points (include/b200_cflearn.h), checked without a GPU, and the tensor checks
of ops.attention_* / ops.cross_attention_* on one.

Every refusal of the C-ABI happens before a tensor map is encoded, so it is the same with or without a device.  The pointers are
fake and never dereferenced: refused calls stop at the argument checks.  A call that passes them reaches B200_ERR_DRIVER on a
machine without a GPU; the matrices that make such calls run only there, so no kernel ever sees a fake pointer."""
import ctypes
import itertools
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import B200Error, _cabi, ops  # noqa: E402

ARG, ALIGN, DRIVER = -1, -2, -3
FAKE = 1 << 20
ODD = FAKE + 8  # not 16-byte aligned
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="accepted calls would launch kernels on fake pointers")

# Per entry point, from the header: the longest sequence, separate Q / K / V (any Dh that is a multiple of 8 in [8, 160], given
# leading dims) or packed qkv (Dh = 64), and the pointers in signature order, each required or optional.
ENTRIES = {
    "b200_attention_fwd": (256, False, {"qkv": True, "out": True, "lse": True}),
    "b200_attention_bwd": (256, False, {"qkv": True, "out": True, "dout": True, "lse": True, "dqkv": True, "dbias_part": False}),
    "b200_attention_long_fwd": (16384, False, {"qkv": True, "out": True, "lse": True}),
    "b200_attention_long_bwd": (16384, False, {"qkv": True, "out": True, "dout": True, "lse": True, "dqkv": True, "dbias_part": False,
                                               "workspace": True}),
    "b200_cross_attention_fwd": (16384, True, {"q": True, "k": True, "v": True, "out": True, "lse": True}),
    "b200_cross_attention_bwd": (16384, True, {"q": True, "k": True, "v": True, "out": True, "dout": True, "lse": True, "dq": True, "dk": True,
                                               "dv": True, "workspace": True}),
}


def attn(entry, B=2, Tq=77, Tk=77, H=4, Dh=64, causal=0, ldq=None, ldkv=None, ldo=None, **ptrs):
    """Calls `entry` with fake pointers (FAKE unless given); leading dims default to H * Dh.  The packed entries take T = Tq."""
    _, cross, names = ENTRIES[entry]
    p = [ptrs.get(n, FAKE) for n in names]
    fn = getattr(_cabi.lib(), entry)
    if not cross:
        fwd = len(p) == 3
        return fn(*p[:3], B, Tq, H, Dh, 0.125, causal, None) if fwd else fn(*p[:5], B, Tq, H, Dh, 0.125, causal, *p[5:], None)
    w = H * Dh
    ldq, ldkv, ldo = (w if x is None else x for x in (ldq, ldkv, ldo))
    if len(p) == 5:
        q, k, v, out, lse = p
        return fn(q, ldq, k, v, ldkv, out, ldo, lse, B, Tq, Tk, H, Dh, 0.125, causal, None)
    q, k, v, out, dout, lse, dq, dk, dv, ws = p
    return fn(q, ldq, k, v, ldkv, out, ldo, dout, lse, dq, dk, dv, B, Tq, Tk, H, Dh, 0.125, causal, ws, None)


def expected(entry, B=2, Tq=77, Tk=77, H=4, Dh=64, causal=0, ldq=None, ldkv=None, ldo=None, **ptrs):
    """The statuses the contract allows for one call: the codes of every rule it breaks, or DRIVER if it breaks none."""
    max_t, cross, names = ENTRIES[entry]
    if not cross:
        Tk = Tq
    lds = [H * Dh if x is None else x for x in (ldq, ldkv, ldo)] if cross else [3 * H * 64, 3 * H * 64, H * 64]
    p = {n: ptrs.get(n, FAKE) for n in names}
    arg = [
        B < 1 or H < 1,
        not (1 <= Tq <= max_t and 1 <= Tk <= max_t),
        (Dh % 8 != 0 or not 8 <= Dh <= 160) if cross else Dh != 64,
        causal and Tq != Tk,
        any(ld < H * Dh for ld in lds),
        any(required and p[n] is None for n, required in names.items()),
    ]
    align = [any(ld % 8 != 0 for ld in lds), any(x is not None and x % 16 != 0 for x in p.values())]
    return ({ARG} if any(arg) else set()) | ({ALIGN} if any(align) else set()) or {DRIVER}


def check_all(entry, calls):
    """Makes every call and asserts that each one's status is one the contract allows."""
    bad = []
    for call in calls:
        got = attn(entry, **call)
        if got not in expected(entry, **call):
            bad.append((call, got, _cabi.last_error()))
    assert not bad, f"{entry}: {len(bad)} of {len(calls)} calls disagree with the header, e.g. {bad[:3]}"


@no_device
@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_sizes_follow_the_header(entry):
    max_t, cross, _ = ENTRIES[entry]
    lengths = (0, 1, 77, max_t, max_t + 1)
    check_all(entry, [dict(B=B, H=H, Tq=Tq, Tk=Tq if Tk is None else Tk, Dh=Dh, causal=causal)
                      for B, H, Tq, Tk, Dh, causal in itertools.product((0, 1, 2), (0, 1, 3), lengths, lengths if cross else (None,),
                                                                        (0, 8, 40, 64, 80, 160, 168), (0, 1))])


@no_device
@pytest.mark.parametrize("entry", ["b200_cross_attention_fwd", "b200_cross_attention_bwd"])
def test_leading_dims_follow_the_header(entry):
    H, Dh = 8, 40
    lds = (H * Dh, H * Dh - 8, H * Dh + 4, H * Dh + 8, 3 * H * Dh)
    check_all(entry, [dict(H=H, Dh=Dh, Tq=300, Tk=77, ldq=ldq, ldkv=ldkv, ldo=ldo) for ldq, ldkv, ldo in itertools.product(lds, lds, lds)])


@no_device
@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_pointers_follow_the_header(entry):
    names = list(ENTRIES[entry][2])
    Dh = 40 if ENTRIES[entry][1] else 64
    check_all(entry, [dict(Dh=Dh, **dict(zip(names, ptrs))) for ptrs in itertools.product((FAKE, None, ODD), repeat=len(names))])


def test_refusals_name_the_rule():
    for entry in ENTRIES:
        assert attn(entry, out=None) == ARG and "null" in _cabi.last_error(), entry
        assert attn(entry, out=ODD) == ALIGN and "aligned" in _cabi.last_error(), entry
        assert attn(entry, lse=ODD) == ALIGN, entry
    for entry in ("b200_attention_long_bwd", "b200_cross_attention_bwd"):
        assert attn(entry, workspace=None) == ARG and "workspace" in _cabi.last_error(), entry
    for entry in ("b200_attention_bwd", "b200_attention_long_bwd"):
        assert attn(entry, dqkv=None) == ARG and attn(entry, dout=ODD) == ALIGN and attn(entry, dbias_part=ODD) == ALIGN, entry


# ---- moved unchanged from the long- and cross-attention test files --------------------------------------------------------
def test_long_entry_points_reject_bad_arguments():
    lib = _cabi.lib()
    null = ctypes.c_void_p(0)
    assert lib.b200_attention_long_fwd(null, null, null, 1, 16385, 1, 64, 0.125, 0, null) == -1
    assert lib.b200_attention_long_fwd(null, null, null, 1, 0, 1, 64, 0.125, 0, null) == -1
    assert lib.b200_attention_long_fwd(null, null, null, 1, 300, 1, 80, 0.125, 0, null) == -1
    assert lib.b200_attention_long_bwd(null, null, null, null, null, 1, 16385, 1, 64, 0.125, 0, null, null, null) == -1
    assert lib.b200_attention_long_bwd(null, null, null, null, null, 1, 300, 1, 64, 0.125, 0, null, null, null) == -1  # no workspace
    assert lib.b200_attention_fwd(null, null, null, 1, 257, 1, 64, 0.125, 0, null) == -1  # the resident kernels keep T <= 256
    # delta [B, H, T] + column-sum partials [B, H, ceil(T / 64), 3, 64]
    assert lib.b200_attention_long_bwd_workspace_floats(2, 577, 12) == 2 * 12 * (577 + 10 * 192)


def test_cross_entry_points_reject_bad_arguments():
    lib = _cabi.lib()
    null = ctypes.c_void_p(0)
    fake = ctypes.c_void_p(1 << 20)  # never dereferenced: every case fails its checks before any launch
    odd = ctypes.c_void_p((1 << 20) + 8)

    def fwd(q=fake, ldq=512, k=fake, v=fake, ldkv=512, out=fake, ldo=512, lse=fake, B=1, Tq=4096, Tk=77, H=8, Dh=40, causal=0):
        return lib.b200_cross_attention_fwd(q, ldq, k, v, ldkv, out, ldo, lse, B, Tq, Tk, H, Dh, 0.125, causal, null)

    def bwd(ws=fake, dq=fake, Dh=40, Tq=4096, Tk=77, causal=0, ldq=512):
        return lib.b200_cross_attention_bwd(fake, ldq, fake, fake, 512, fake, 512, fake, fake, dq, fake, fake, 1, Tq, Tk, 8, Dh, 0.125, causal,
                                            ws, null)

    for Dh in (0, 4, 12, 168, 192):
        assert fwd(Dh=Dh) == -1 and bwd(Dh=Dh) == -1, Dh
    for Tq, Tk in ((0, 77), (77, 0), (16385, 77), (77, 16385)):
        assert fwd(Tq=Tq, Tk=Tk) == -1 and bwd(Tq=Tq, Tk=Tk) == -1
    assert fwd(causal=1) == -1 and bwd(causal=1) == -1           # causal needs Tq == Tk
    assert fwd(ldq=312) == -1 and fwd(ldkv=312) == -1 and fwd(ldo=312) == -1  # < H * Dh = 320
    assert fwd(ldq=324) == -2 and fwd(ldkv=324) == -2 and bwd(ldq=324) == -2  # not a multiple of 8
    assert fwd(q=null) == -1 and fwd(lse=null) == -1 and bwd(dq=null) == -1
    assert "null" in _cabi.last_error()
    assert bwd(ws=null) == -1 and "workspace" in _cabi.last_error()
    assert fwd(k=odd) == -2 and bwd(dq=odd) == -2 and bwd(ws=odd) == -2
    assert "aligned" in _cabi.last_error()


def _chunks(B, Tq, Tk, H, Dh):
    rows = 128 if Dh <= 64 else 64
    ctas = B * H * -(-Tk // rows)
    nqb = -(-Tq // 64)
    want = min(nqb, 1 if ctas >= 132 else 132 // ctas)
    per = -(-nqb // want)
    return -(-nqb // per)


@pytest.mark.parametrize("B,Tq,Tk,H,Dh", [(8, 4096, 77, 8, 40), (1, 4096, 77, 2, 40), (8, 1024, 77, 8, 80), (8, 256, 77, 8, 160),
                                          (8, 64, 64, 8, 160), (2, 577, 577, 12, 64), (1, 1, 1, 1, 8)])
def test_cross_workspace_formula(B, Tq, Tk, H, Dh):
    n = _chunks(B, Tq, Tk, H, Dh)
    delta = -(-(B * H * Tq) // 4) * 4
    want = delta + (2 * n * B * H * Tk * Dh if n > 1 else 0)
    assert _cabi.lib().b200_cross_attention_bwd_workspace_floats(B, Tq, Tk, H, Dh) == want
    if (B, Tq, Tk, H) == (1, 4096, 77, 2):
        assert n == 64  # the determinism test's split case really is split
    if (B, Tq, Tk, H) == (8, 4096, 77, 8):
        assert n == 2


# ---- ops: every tensor handed to the library is checked against the header's layout ------------------------------------------
def _bf16(*shape):
    return torch.randn(*shape, device="cuda").to(torch.bfloat16)


def _refused(fn, *args, **kw):
    with pytest.raises(B200Error):
        fn(*args, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [77, 300])
def test_ops_attention_refuses_bad_tensors(T):
    B, H = 2, 3
    D = H * 64
    qkv, dout = _bf16(B * T, 3 * D), _bf16(B * T, D)
    out, lse = ops.attention_fwd(qkv, B, T, H)
    _refused(ops.attention_fwd, qkv.half(), B, T, H)                                    # dtype
    _refused(ops.attention_fwd, qkv[:, :D], B, T, H)                                    # shape (and not contiguous)
    _refused(ops.attention_fwd, qkv.reshape(B * T * 3, D), B, T, H)                     # rows of the wrong width
    _refused(ops.attention_fwd, _bf16(3 * D, B * T).t(), B, T, H)                       # strided

    def bwd(qkv=qkv, out=out, dout=dout, lse=lse, **kw):
        return ops.attention_bwd(qkv, out, dout, lse, B, T, H, **kw)

    _refused(bwd, qkv=qkv[:-1])
    _refused(bwd, out=_bf16(D, B * T).t())
    _refused(bwd, out=out[:-1])
    _refused(bwd, dout=dout.float())
    _refused(bwd, dout=_bf16(B * T, 2 * D)[:, :D])
    _refused(bwd, lse=lse.half())
    _refused(bwd, lse=lse.transpose(1, 2).contiguous())
    _refused(bwd, lse=lse[:, :, :-1])
    _refused(bwd, dqkv=torch.empty(B * T - 1, 3 * D, dtype=torch.bfloat16, device="cuda"))
    _refused(bwd, dqkv=torch.empty(B * T, 4 * D, dtype=torch.bfloat16, device="cuda")[:, :3 * D])
    _refused(bwd, dqkv=torch.empty(B * T, 3 * D, dtype=torch.float32, device="cuda"))
    _refused(bwd, dbias=torch.zeros(3 * D, dtype=torch.bfloat16, device="cuda"))
    _refused(bwd, dbias=torch.zeros(2 * D, device="cuda"))
    _refused(bwd, dbias=torch.zeros(3 * D, 2, device="cuda")[:, 0])
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_ops_cross_attention_refuses_bad_tensors():
    B, H, Dh, Tq, Tk = 2, 4, 40, 300, 77
    L = H * Dh
    q, kv = _bf16(B * Tq, L), _bf16(B * Tk, 2 * L)
    k, v = kv[:, :L], kv[:, L:]
    out, lse = ops.cross_attention_fwd(q, k, v, B, H)
    dout = _bf16(B * Tq, L)
    _refused(ops.cross_attention_fwd, q.float(), k, v, B, H)
    _refused(ops.cross_attention_fwd, q, _bf16(L, B * Tk).t(), v, B, H)
    _refused(ops.cross_attention_fwd, q, k, v[:-1], B, H)

    def bwd(q=q, k=k, v=v, out=out, dout=dout, lse=lse, **kw):
        return ops.cross_attention_bwd(q, k, v, out, dout, lse, B, H, **kw)

    grads = dict(dq=torch.empty_like(q), dk=torch.empty_like(kv)[:, :L], dv=torch.empty_like(kv)[:, L:])
    _refused(bwd, v=_bf16(B * Tk, L).half(), **grads)
    _refused(bwd, out=out[:-B], dout=dout[:-B], **grads)
    _refused(bwd, out=_bf16(B * Tq, 2 * L)[:, :L], **grads)
    _refused(bwd, dout=_bf16(L, B * Tq).t(), **grads)
    _refused(bwd, lse=lse.half(), **grads)
    _refused(bwd, lse=lse[:, :, :-1], **grads)
    _refused(bwd, lse=lse.transpose(1, 2), **grads)
    _refused(bwd, **dict(grads, dq=torch.empty_like(q)[:-1]))
    _refused(bwd, **dict(grads, dk=torch.empty_like(kv)[:-1, :L]))
    _refused(bwd, **dict(grads, dv=torch.empty_like(kv)[:, L:].float()))
    torch.cuda.synchronize()
