"""Every attention entry point, element by element: out, dq, dk and dv against the per-element bound of _refs.attention_bounds,
lse against float64 to 1e-4 relative.  The backward reads the forward's own bf16 out, as in training.

A relative L2 error over the whole tensor hides a mistake confined to one key tile, one query row, one head or the causal
diagonal; the per-element bound, derived from the kernels' rounding points, does not (test_attention_bounds.py shows it on an
emulation of the kernels and on broken variants of it).  The shapes sit on either side of every tile edge: 64-key blocks,
the resident kernels' 128-query tiles, the streamed dK / dV kernel's 128-key tile (Dh <= 64), the 64-column boxes of the
padded head dim and each k16-step instance of the streamed kernels, both dK / dV grid regimes (queries split into chunks
and reduced, or one chunk), more (batch, head) items than SMs, and scores that peak at 100..200.  Needs an H100
(pytest -m gpu)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import _cabi, ops  # noqa: E402
from _refs import F64, attention_bounds_rows, peaked_qkv, rand_bf16  # noqa: E402

DEV = "cuda"


# ---- the check ---------------------------------------------------------------------------------------------------------------------
def _check(tag, q, k, v, dout, B, H, scale, causal, out, lse, dq, dk, dv):
    """All tensors in the kernels' row layout (q / out / dout / dq [B Tq, H Dh], k / v / dk / dv [B Tk, H Dh]), lse [B, H, Tq].
    Fails on the first element past its bound, reported as (b, h, row, col), with the case's worst err / tol per output."""
    torch.cuda.synchronize()
    (o64, lse64, dq64, dk64, dv64), tols = attention_bounds_rows(q, k, v, dout, B, H, scale, causal, out)
    Dh = q.shape[1] // H
    worst, first = {}, None
    for name, got, ref, tol in zip(("out", "dq", "dk", "dv"), (out, dq, dk, dv), (o64, dq64, dk64, dv64), tols):
        err = (got.to(F64) - ref).abs()
        worst[name] = torch.nan_to_num(err / tol.clamp_min(1e-300), nan=float("inf")).max().item()
        bad = torch.nonzero(~(err <= tol))
        if first is None and bad.numel():
            r, c = bad[0].tolist()
            T = got.shape[0] // B
            first = (f"{name} at (b, h, row, col) = ({r // T}, {c // Dh}, {r % T}, {c % Dh}): {got[r, c].item():.6g} vs float64 "
                     f"{ref[r, c].item():.6g}, |err| {err[r, c].item():.3e} > tol {tol[r, c].item():.3e}; {bad.shape[0]} elements over")
    le = (lse.to(F64) - lse64).abs() / (1 + lse64.abs())
    worst["lse"] = le.max().item() / 1e-4
    summary = ", ".join(f"{n} {w:.3f}" for n, w in worst.items())
    print(f"{tag}: worst err / tol {summary}")
    assert first is None, f"{tag}: {first}; worst err / tol {summary}"
    bad = torch.nonzero(~(le <= 1e-4))
    assert not bad.numel(), f"{tag}: lse at (b, h, row) = {tuple(bad[0].tolist())} off by {le.max().item():.3e} relative"


def _qkv(B, Tq, Tk, H, Dh, scale, causal, seed, peaked):
    """bf16 rows q [B Tq, H Dh], k / v [B Tk, H Dh] and dout: N(0, 1), or peaked_qkv's near-one-hot scores."""
    if peaked:
        rows = lambda t: t.to(torch.bfloat16).permute(0, 2, 1, 3).reshape(-1, H * Dh).to(DEV)  # noqa: E731
        q, k, v = (rows(t) for t in peaked_qkv(B, H, Tq, Tk, Dh, scale, causal, seed))
    else:
        q, k, v = rand_bf16(B * Tq, H * Dh, seed=seed), rand_bf16(B * Tk, H * Dh, seed=seed + 1), rand_bf16(B * Tk, H * Dh, seed=seed + 2)
    return q, k, v, rand_bf16(B * Tq, H * Dh, seed=seed + 3)


# ---- packed qkv: the resident (T <= 256) and the streamed kernels ------------------------------------------------------------------
def _long_entry(qkv, dout, B, T, H, scale, causal):
    """The streamed kernels on packed qkv: through ops past 256 tokens, where it dispatches to them; below, from the C-ABI."""
    if T > ops.ATTENTION_RESIDENT_MAX_T:
        out, lse = ops.attention_fwd(qkv, B, T, H, scale=scale, causal=causal)
        return out, lse, ops.attention_bwd(qkv, out, dout, lse, B, T, H, scale=scale, causal=causal)
    stream = torch.cuda.current_stream().cuda_stream
    out = torch.empty((B * T, H * 64), dtype=torch.bfloat16, device=DEV)
    lse = torch.empty((B, H, T), dtype=torch.float32, device=DEV)
    _cabi.call("b200_attention_long_fwd", qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, T, H, 64, scale, int(causal), stream)
    dqkv = torch.empty_like(qkv)
    ws = torch.empty(int(_cabi.lib().b200_attention_long_bwd_workspace_floats(B, T, H)), device=DEV)
    _cabi.call("b200_attention_long_bwd", qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), B, T, H, 64,
               scale, int(causal), None, ws.data_ptr(), stream)
    return out, lse, dqkv


def _packed_case(entry, B, T, H, causal, scale=0.125, peaked=False):
    q, k, v, dout = _qkv(B, T, T, H, 64, scale, causal, seed=T * 4 + int(causal), peaked=peaked)
    qkv = torch.cat([q, k, v], 1).contiguous()
    if entry == "resident":
        out, lse = ops.attention_fwd(qkv, B, T, H, scale=scale, causal=causal)
        dqkv = ops.attention_bwd(qkv, out, dout, lse, B, T, H, scale=scale, causal=causal)
    else:
        out, lse, dqkv = _long_entry(qkv, dout, B, T, H, scale, causal)
    D = H * 64
    _check(f"{entry} B{B} T{T} H{H} causal={causal} scale={scale:g}{' peaked' if peaked else ''}", q, k, v, dout, B, H, scale, causal,
           out, lse, dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:])


RESIDENT_T = [1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 197, 255, 256]


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("T", RESIDENT_T)
def test_resident(T, causal):
    _packed_case("resident", 2, T, 2, causal)


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,H,causal,scale,peaked", [
    (12, 65, 12, False, 0.125, False), (12, 197, 12, True, 0.125, False),  # 144 (batch, head) items: more than the 132 SMs
    (2, 197, 2, False, 0.1, False), (2, 129, 3, True, 0.1, False),        # a scale that is not a power of two
    (2, 197, 2, False, 0.125, True), (2, 197, 2, True, 0.125, True), (2, 77, 4, True, 0.125, True)])
def test_resident_more(B, T, H, causal, scale, peaked):
    _packed_case("resident", B, T, H, causal, scale, peaked)


LONG_T = [1, 64, 65, 127, 128, 129, 257, 385, 1025]


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("T", LONG_T)
def test_streamed(T, causal):
    _packed_case("streamed", 2, T, 2, causal)


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,H,causal,scale,peaked", [
    (1, 4096, 2, True, 0.125, False), (2, 257, 3, True, 0.1, False),
    (1, 385, 2, True, 0.125, True), (1, 1025, 2, False, 0.125, True)])
def test_streamed_more(B, T, H, causal, scale, peaked):
    _packed_case("streamed", B, T, H, causal, scale, peaked)


# ---- separate Q / K / V: cross_attention_fwd / _bwd ---------------------------------------------------------------------------------
def _cross_case(B, Tq, Tk, H, Dh, causal, scale=None, peaked=False, ld=None):
    """``ld``: q, k, v (and dq, dk, dv) are column slices of one packed [B T, ld] buffer, as a fused qkv projection leaves them."""
    scale = Dh ** -0.5 if scale is None else scale
    q, k, v, dout = _qkv(B, Tq, Tk, H, Dh, scale, causal, seed=Tq * 7 + Tk * 3 + Dh + int(causal), peaked=peaked)
    grads = {}
    if ld is not None:
        L = H * Dh
        buf = torch.zeros(B * Tq, ld, dtype=torch.bfloat16, device=DEV)
        buf[:, :L], buf[:, L:2 * L], buf[:, 2 * L:3 * L] = q, k, v
        q, k, v = buf[:, :L], buf[:, L:2 * L], buf[:, 2 * L:3 * L]
        dbuf = torch.empty_like(buf)
        grads = dict(dq=dbuf[:, :L], dk=dbuf[:, L:2 * L], dv=dbuf[:, 2 * L:3 * L])
    out, lse = ops.cross_attention_fwd(q, k, v, B, H, scale=scale, causal=causal)
    dq, dk, dv = ops.cross_attention_bwd(q, k, v, out, dout, lse, B, H, scale=scale, causal=causal, **grads)
    tag = f"cross B{B} Tq{Tq} Tk{Tk} H{H} Dh{Dh} causal={causal}{' peaked' if peaked else ''}{f' ld={ld}' if ld else ''}"
    _check(tag, q, k, v, dout, B, H, scale, causal, out, lse, dq, dk, dv)


# 2, 2, 3, 3, 4, 5, 5, 8, 8, 10, 10 k16 steps (attn_long_ksteps); 8 ... 64 in one 64-column box, 72 ... 128 in two, 136 / 160 in three
CROSS_DH = [8, 32, 40, 48, 64, 72, 80, 96, 128, 136, 160]
CROSS_TT = [(1, 1, False), (1, 77, False), (77, 1, False), (64, 65, False), (65, 64, False), (300, 77, False), (129, 129, True),
            (193, 193, True)]
# every (Tq, Tk) at the model head dims (SD-UNet 40 / 80 / 160, ViT 64), the key and query tile edges and a causal case at the rest
CROSS_CASES = [(Dh, *tt) for Dh in CROSS_DH for tt in (CROSS_TT if Dh in (40, 64, 80, 160) else [CROSS_TT[i] for i in (3, 4, 5, 7)])]


@pytest.mark.gpu
@pytest.mark.parametrize("Dh,Tq,Tk,causal", CROSS_CASES)
def test_cross(Dh, Tq, Tk, causal):
    # B H = 6 with at most 4 key tiles: the dK / dV grid is split over query chunks and reduced whenever Tq > 64
    _cross_case(2, Tq, Tk, 3, Dh, causal)


@pytest.mark.gpu
@pytest.mark.parametrize("B,Tq,Tk,H,Dh,causal", [
    (1, 4096, 77, 1, 40, False), (1, 4096, 77, 1, 64, False), (1, 4096, 77, 1, 160, False),  # one key tile: 64 query chunks
    (1, 1025, 1025, 1, 64, True), (1, 1025, 1025, 1, 80, True),                                # causal over chunks
    (12, 300, 77, 12, 40, False), (12, 300, 77, 12, 64, False), (12, 300, 77, 12, 160, False),  # >= 132 CTAs: one chunk
    (4, 300, 300, 8, 128, True)])
def test_cross_dkdv_regimes(B, Tq, Tk, H, Dh, causal):
    _cross_case(B, Tq, Tk, H, Dh, causal)


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,H,Dh,causal", [(2, 300, 8, 40, False), (2, 193, 2, 160, True)])
def test_cross_packed_slices(B, T, H, Dh, causal):
    _cross_case(B, T, T, H, Dh, causal, ld=3 * H * Dh + 64)


@pytest.mark.gpu
@pytest.mark.parametrize("Tq,Tk,Dh,causal,scale", [(300, 77, 40, False, None), (193, 193, 160, True, None), (65, 64, 72, False, 0.1)])
def test_cross_peaked(Tq, Tk, Dh, causal, scale):
    _cross_case(2, Tq, Tk, 3, Dh, causal, scale=scale, peaked=True)
