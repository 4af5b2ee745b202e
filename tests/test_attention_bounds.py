"""CPU: _refs.attention_bounds against an emulation of the attention kernels' rounding chain, and against broken variants of it.

``emulate`` restates in fp32 / bf16 what the kernels in attention_sm90.cu compute: fp32 scores, the softmax in the exp2 domain
with the scale folded in and probabilities below 2^-126 flushed to zero, P rounded to bf16 for P V, the fp32 row sum, bf16 out,
lse = m scale + ln(l); in the backward P recomputed from the fp32 lse, delta from the bf16 out, dS rounded to bf16,
dV = bf16(P)^T dO, dQ / dK scaled in fp32 at the end.
The emulation must stay within half of the bound at every element, and every mutant -- each a local mistake of the kind a kernel
change makes: one key, one row, one head, the causal diagonal, a query tile, a missing factor -- must break it somewhere."""
import math

import pytest
import torch

from _refs import attention_bounds, peaked_qkv

F64 = torch.float64
LOG2E = math.log2(math.e)

# (B, H, Tq, Tk, D, scale): partial 64-key tiles, the 128-row dK / dV tile edge and a Tq != Tk case; no scale is a power of two
SHAPES = [(2, 2, 65, 65, 64, 0.1), (1, 2, 129, 129, 64, 0.1), (1, 2, 197, 197, 64, 0.1), (2, 2, 77, 100, 40, 40 ** -0.5),
          (1, 2, 200, 77, 80, 80 ** -0.5)]
CAUSAL_ONLY = {"causal_plus_one", "causal_minus_one", "last_row_previous_mask"}
MUTANTS = ["causal_plus_one", "causal_minus_one", "last_key_dropped", "last_row_previous_mask", "heads_swapped", "dq_unscaled",
           "dk_unscaled", "delta_wrong_row", "dkdv_without_last_query_tile", "lse_log2"]


def _inputs(B, H, Tq, Tk, D, seed):
    g = torch.Generator().manual_seed(seed)
    q, dout = (torch.randn(B, H, Tq, D, generator=g).to(torch.bfloat16) for _ in range(2))
    k, v = (torch.randn(B, H, Tk, D, generator=g).to(torch.bfloat16) for _ in range(2))
    return q, k, v, dout


def _bf(x):
    return x.to(torch.bfloat16).float()


def _ex2_ftz(x):
    """exp2 as ex2.approx.ftz.f32 rounds it: results below the smallest normal fp32 are 0."""
    y = torch.exp2(x)
    return torch.where(y < 2.0 ** -126, 0.0, y)


def emulate(q, k, v, dout, scale, causal, mutant=None):
    """The kernels' forward and backward on bf16 [B, H, T, D] inputs: (out, lse, dq, dk, dv), out and the gradients bf16 values."""
    qf, kf, vf, df = (t.float() for t in (q, k, v, dout))
    Tq, Tk = qf.shape[-2], kf.shape[-2]
    i, j = torch.arange(Tq)[:, None], torch.arange(Tk)[None, :]
    seen = j <= i + (1 if mutant == "causal_plus_one" else 0) if causal else torch.ones(Tq, Tk, dtype=torch.bool)
    if mutant == "causal_minus_one":
        seen = (j < i) | (j == 0)
    if mutant == "last_key_dropped":  # key Tk - 1: the last key of a partial 64-key tile
        seen = seen & (j != Tk - 1)
    if mutant == "last_row_previous_mask":
        seen[-1] = seen[-2]
    sl2 = torch.tensor(scale * LOG2E, dtype=torch.float32)
    s = (qf @ kf.transpose(-1, -2)).masked_fill(~seen, float("-inf"))
    # forward
    m = s.amax(-1)
    p = _ex2_ftz(s * sl2 - (m * sl2)[..., None])
    l = p.sum(-1)  # noqa: E741
    out = _bf((_bf(p) @ vf) / l[..., None])
    lse = m * scale + (torch.log2(l) if mutant == "lse_log2" else torch.log(l))
    # backward
    delta = (df * out).sum(-1)
    if mutant == "delta_wrong_row":
        delta[..., -1] = delta[..., -2]
    p = _ex2_ftz(s * sl2 - (lse * LOG2E)[..., None])
    ds = _bf(p * (df @ vf.transpose(-1, -2) - delta[..., None]))
    pb = _bf(p)
    if mutant == "dkdv_without_last_query_tile":  # the last 64-query block: a query-chunk boundary of the streamed dK / dV
        keep = (torch.arange(Tq) < (Tq - 1) // 64 * 64)[:, None].float()
        ds_kv, pb = ds * keep, pb * keep
    else:
        ds_kv = ds
    dq = (ds @ kf) * (1.0 if mutant == "dq_unscaled" else scale)
    dk = (ds_kv.transpose(-1, -2) @ qf) * (1.0 if mutant == "dk_unscaled" else scale)
    dv = pb.transpose(-1, -2) @ df
    res = [out, lse, _bf(dq), _bf(dk), _bf(dv)]
    if mutant == "heads_swapped":  # heads 0 and 1 of the last query row (and of the last key row) trade places
        for t in res[:1] + res[2:]:
            t[:, [0, 1], -1] = t[:, [1, 0], -1]
    return tuple(res)


def _ratios(got, refs, tols):
    """max |got - ref| / tol per output (out, dq, dk, dv); inf where an element breaks a zero tolerance or is not finite."""
    out = []
    for x, r, t in zip((got[0],) + got[2:], (refs[0],) + refs[2:], tols):
        err = (x.to(F64) - r).abs()
        ratio = torch.where(t > 0, err / t.clamp_min(1e-300), torch.where(err == 0, 0.0, float("inf")))
        out.append(torch.where(torch.isfinite(err), ratio, float("inf")).max().item())
    return out


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "B{}H{}Tq{}Tk{}D{}".format(*s[:5]))
def test_emulated_kernels_stay_within_half_the_bound(shape, causal):
    B, H, Tq, Tk, D, scale = shape
    if causal and Tq != Tk:
        pytest.skip("causal attention needs Tq == Tk")
    q, k, v, dout = _inputs(B, H, Tq, Tk, D, seed=Tq + Tk + int(causal))
    got = emulate(q, k, v, dout, scale, causal)
    refs, tols = attention_bounds(q, k, v, dout, scale, causal, got[0])
    ratios = _ratios(got, refs, tols)
    assert max(ratios) <= 0.5, f"err / tol of out, dq, dk, dv: {ratios}"
    assert ((got[1].to(F64) - refs[1]).abs() <= 1e-4 * (1 + refs[1].abs())).all()


@pytest.mark.parametrize("causal", [False, True])
def test_emulated_kernels_stay_within_half_the_bound_on_peaked_scores(causal):
    """Scores 100..200 above the rest of the row: most probabilities underflow fp32, and the bound's 2^-126 terms carry them."""
    B, H, T, D, scale = 2, 2, 129, 64, 0.125
    q, k, v = (t.to(torch.bfloat16) for t in peaked_qkv(B, H, T, T, D, scale, causal, seed=5))
    dout = _inputs(B, H, T, T, D, seed=6)[3]
    got = emulate(q, k, v, dout, scale, causal)
    refs, tols = attention_bounds(q, k, v, dout, scale, causal, got[0])
    ratios = _ratios(got, refs, tols)
    assert max(ratios) <= 0.5, f"err / tol of out, dq, dk, dv: {ratios}"


@pytest.mark.parametrize("mutant", MUTANTS)
def test_the_bound_rejects_every_mutant(mutant):
    cases = 0
    for B, H, Tq, Tk, D, scale in SHAPES:
        for causal in (False, True):
            if (causal and Tq != Tk) or (mutant in CAUSAL_ONLY and not causal):
                continue
            q, k, v, dout = _inputs(B, H, Tq, Tk, D, seed=Tq + Tk + int(causal))
            got = emulate(q, k, v, dout, scale, causal, mutant)
            refs, tols = attention_bounds(q, k, v, dout, scale, causal, got[0])
            ratios = _ratios(got, refs, tols)
            assert max(ratios) > 1.0, f"{mutant} passes at B{B} H{H} Tq{Tq} Tk{Tk} D{D} causal={causal}: err / tol {ratios}"
            cases += 1
    assert cases >= 2
