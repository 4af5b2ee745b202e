"""The kernels that reduce a row or a group to statistics, on ill-conditioned inputs, against float64 references.

GroupNorm(+SiLU), both LayerNorms, both cross-entropies and the three attention families are compared with the same operation
computed in torch.float64 from the kernel's own bf16 / fp32 inputs, at inputs where a cancelling formula or a mishandled running
max shows: groups and rows whose mean is hundreds of standard deviations, constant and near-constant groups, outliers, logits up to
+-3e4 and -inf, and attention rows whose softmax is close to one-hot with the peak in the first, the last or a partial key block.

Each comparison is against the "eager floor": the error, against the same float64 reference, of the PyTorch op that eager bf16
autocast runs on the same inputs.  The per-element check counts elements more than one bf16 ulp from bf16(float64 reference) and
allows no more of them than eager has; the relative L2 error must stay within 1.5x eager's + 1e-6.  Statistics (mean, rstd) must
be within 4x eager's relative error or 1e-5.  The references are in _refs.py.  The CPU cases check the input generators against
the conditioning they claim; the others need an H100 (pytest -m gpu)."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import _cabi, ops  # noqa: E402
from _refs import (F64, GROUPS, attention, bf16_ulps_off, groupnorm, layernorm, peaked_qkv, relerr, softmax_xent,  # noqa: E402
                   symmetric_xent, with_grads)

DEV = "cuda"


# ---- checks ------------------------------------------------------------------------------------------------------------------------
def _assert_like_eager(what, got, eager, ref, per_element=True, l2_factor=1.5):
    """``per_element=False`` keeps only the L2 bound (and still counts NaN / inf as failures)."""
    ours_bad, eager_bad = bf16_ulps_off(got, ref), bf16_ulps_off(eager, ref)
    e_ours, e_eager = relerr(got, ref), relerr(eager, ref)
    msg = (f"{what}: {ours_bad} elements more than 1 bf16 ulp from float64 (eager: {eager_bad}), relative L2 {e_ours:.3e} "
           f"(eager: {e_eager:.3e}) of {got.numel()} elements")
    assert bool(torch.isfinite(got).all()) and e_ours <= l2_factor * e_eager + 1e-6, msg
    assert not per_element or ours_bad <= eager_bad, msg


def _assert_stats(what, got, eager, ref, scale):
    """max over rows / groups of |got - ref| / scale  <=  max(4 x eager's, 1e-5)."""
    e_ours = ((got.to(F64).flatten() - ref.flatten()).abs() / scale.flatten()).max().item()
    e_eager = ((eager.to(F64).flatten() - ref.flatten()).abs() / scale.flatten()).max().item()
    assert e_ours <= max(4.0 * e_eager, 1e-5), f"{what}: max relative error {e_ours:.3e} (eager: {e_eager:.3e})"


# ---- GroupNorm inputs --------------------------------------------------------------------------------------------------------------
OFFSETS = {"offset_0.2": (0.3, 1.5), "offset_30": (30.0, 1.0), "offset_100": (100.0, 1.0), "offset_400": (400.0, 1.0)}
KINDS = list(OFFSETS) + ["near_constant", "constant", "outlier"]
GN_CONDS = KINDS + ["mixed"]
NEAR_CONST = 4.0  # a few percent of the pixels one bf16 ulp (2^-5) above it
OUTLIER = 1000.0  # the first pixel of every channel of the group; the rest ~ N(0.5, 1)


def gn_kinds(B, cond):
    """Kind of every (image, group); "mixed" varies it with both the image and the group."""
    return [[KINDS[(5 * b + g) % len(KINDS)] if cond == "mixed" else cond for g in range(GROUPS)] for b in range(B)]


def gn_input(B, HW, C, cond, seed):
    """bf16 [B, HW, C] with every (image, group) drawn from its kind (gn_kinds)."""
    g = torch.Generator().manual_seed(seed)
    cpg = C // GROUPS
    z = torch.randn(B, HW, GROUPS, cpg, generator=g, dtype=F64)
    u = torch.rand(B, HW, GROUPS, cpg, generator=g, dtype=F64)
    x = torch.empty_like(z)
    for b, row in enumerate(gn_kinds(B, cond)):
        for gi, kind in enumerate(row):
            if kind in OFFSETS:
                mu, sd = OFFSETS[kind]
                x[b, :, gi] = mu + sd * z[b, :, gi]
            elif kind == "near_constant":
                x[b, :, gi] = NEAR_CONST + 2.0 ** -5 * (u[b, :, gi] < 0.03).to(F64)
            elif kind == "constant":
                x[b, :, gi] = -2.5
            else:
                x[b, :, gi] = 0.5 + z[b, :, gi]
                x[b, 0, gi] = OUTLIER
    return x.reshape(B, HW, C).to(torch.bfloat16)


def gn_slabs(B, HW):
    """csrc/groupnorm.cu gn_slabs: pixel slabs per image (4 x 132 blocks over the batch, at least 64 pixels per slab)."""
    return max(1, min((4 * 132 + B - 1) // B, (HW + 63) // 64))


# ---- CPU: the references and the generators ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("cond", GN_CONDS)
def test_groupnorm_inputs_have_the_conditioning_they_claim(cond):
    B, HW, C = 3, 256, 320
    x = gn_input(B, HW, C, cond, seed=7)
    xg = x.to(F64).view(B, HW, GROUPS, C // GROUPS)
    mean, sd = xg.mean(dim=(1, 3)), xg.std(dim=(1, 3), unbiased=False)
    for b, row in enumerate(gn_kinds(B, cond)):
        for gi, kind in enumerate(row):
            m, s = mean[b, gi].item(), sd[b, gi].item()
            if kind in OFFSETS:  # bf16 quantisation widens the spread a little at mean / std = 400 (ulp 2 at 400); the sample
                want = OFFSETS[kind][0] / OFFSETS[kind][1]  # mean of n values moves the ratio by ~1 / sqrt(n)
                assert abs(m / s - want) <= 0.25 * want + 5 / math.sqrt(xg[b, :, gi].numel()), (b, gi, kind, m / s)
            elif kind == "near_constant":
                assert s > 0 and m / s > 300, (b, gi, m, s)
            elif kind == "constant":
                assert s == 0, (b, gi, s)
            else:
                grp = xg[b, :, gi]
                assert (grp[0] == OUTLIER).all() and grp[1:].abs().max() < 10 and (OUTLIER - m) / s > 10, (b, gi)
    if cond == "mixed":
        assert len({k for row in gn_kinds(B, cond) for k in row}) == len(KINDS)
        assert all(gn_kinds(B, cond)[b][0] != gn_kinds(B, cond)[b + 1][0] for b in range(B - 1))


def test_the_last_slab_at_65x65_batch_8_is_empty():
    B, HW = 8, 65 * 65
    nslab = gn_slabs(B, HW)
    pps = (HW + nslab - 1) // nslab
    assert (nslab, pps) == (66, 65) and (nslab - 1) * pps >= HW  # the launch covers 66 x 65 = 4290 pixel slots for 4225 pixels
    assert gn_slabs(8, 49) == 1 and gn_slabs(1, 4096) == 64 and gn_slabs(16, 4096) == 33


# ---- GroupNorm(+SiLU) --------------------------------------------------------------------------------------------------------------
GN_SHAPES = [(b, s, s, c) for s, c in ((64, 320), (32, 640), (16, 960), (8, 1280), (16, 2560)) for b in (1, 16)] + [(8, 7, 7, 320), (8, 65, 65, 320)]


def _groupnorm_case(B, H, W, C, cond, silu, seed):
    HW = H * W
    eps = 1e-5 if silu else 1e-6
    x = gn_input(B, HW, C, cond, seed).to(DEV)
    g = torch.Generator().manual_seed(seed + 1)
    gamma = (1.0 + 0.1 * torch.randn(C, generator=g)).to(DEV)
    beta = (0.05 * torch.randn(C, generator=g)).to(DEV)
    dy = torch.randn(B, HW, C, generator=g).to(torch.bfloat16).to(DEV)

    # float64 reference, forward and backward
    (y64, mean64, rstd64, var64), (dx64, dg64, db64) = with_grads(groupnorm, (x, gamma, beta), dy, eps, silu)
    # eager under bf16 autocast: GroupNorm in fp32 on the upcast input (ATen's kernel, which returns its mean / rstd), SiLU in fp32,
    # one bf16 rounding; the input gradient reaches the bf16 input as bf16
    xe = x.float().permute(0, 2, 1).contiguous().requires_grad_(True)
    ge, be = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    ze, mean_e, rstd_e = torch.native_group_norm(xe, ge, be, B, C, HW, GROUPS, eps)
    ye = (F.silu(ze) if silu else ze).to(torch.bfloat16)
    ye.backward(dy.permute(0, 2, 1))
    ye = ye.permute(0, 2, 1)
    dx_e = xe.grad.permute(0, 2, 1).to(torch.bfloat16)

    y, mean, rstd = ops.groupnorm_silu_fwd(x, gamma, beta, eps, silu=silu)
    dx, dgamma, dbeta = ops.groupnorm_silu_bwd(x, dy, gamma, beta, mean, rstd, silu=silu)
    torch.cuda.synchronize()

    tag = f"B{B} {H}x{W} C{C} {cond} silu={silu}"
    sd64 = var64.sqrt()
    _assert_stats(f"{tag}: mean", mean, mean_e, mean64, torch.maximum(mean64.abs(), sd64).clamp_min(1e-30))
    _assert_stats(f"{tag}: rstd", rstd, rstd_e, rstd64, rstd64)
    const = var64 == 0
    if const.any():  # a constant group: rstd = rsqrt(eps), exactly as eager computes it
        assert torch.allclose(rstd[const], rstd_e[const], rtol=1e-6, atol=0), f"{tag}: rstd of constant groups {rstd[const]} vs {rstd_e[const]}"
    # Per element, only the L2 bound: the kernel's fp32 mean can sit a few fp32 ulps from eager's correctly rounded one, and at
    # mean / std ~ 1e3 that moves outputs near zero by more than their own bf16 ulp (the floor eps * mean / std both share).  The
    # SiLU derivative's fast exp2 / reciprocal leave dgamma / dbeta up to ~2x eager's (small) error.
    _assert_like_eager(f"{tag}: y", y, ye, y64, per_element=False)
    _assert_like_eager(f"{tag}: dx", dx, dx_e, dx64, per_element=False)
    _assert_like_eager(f"{tag}: dgamma", dgamma, ge.grad, dg64, per_element=False, l2_factor=4.0)
    _assert_like_eager(f"{tag}: dbeta", dbeta, be.grad, db64, per_element=False, l2_factor=4.0)
    # deterministic: a second run is bit-identical
    y2, m2, r2 = ops.groupnorm_silu_fwd(x, gamma, beta, eps, silu=silu)
    dx2, dg2, db2 = ops.groupnorm_silu_bwd(x, dy, gamma, beta, m2, r2, silu=silu)
    assert torch.equal(y, y2) and torch.equal(mean, m2) and torch.equal(rstd, r2)
    assert torch.equal(dx, dx2) and torch.equal(dgamma, dg2) and torch.equal(dbeta, db2)


@pytest.mark.gpu
@pytest.mark.parametrize("cond", GN_CONDS)
@pytest.mark.parametrize("B,H,W,C", GN_SHAPES)
def test_groupnorm_silu(B, H, W, C, cond):
    _groupnorm_case(B, H, W, C, cond, True, seed=B * 1000 + H * 10 + C + GN_CONDS.index(cond))


@pytest.mark.gpu
@pytest.mark.parametrize("cond", GN_CONDS)
@pytest.mark.parametrize("B,H,W,C", [(2, 32, 32, 640), (8, 65, 65, 320)])
def test_groupnorm_plain(B, H, W, C, cond):
    _groupnorm_case(B, H, W, C, cond, False, seed=7 + B + GN_CONDS.index(cond))


# ---- LayerNorm ---------------------------------------------------------------------------------------------------------------------
def ln_input(rows, dim, seed, dtype):
    """Rows cycle through mean / std = 0.2, 30 and 1e3, a constant row and a row with one outlier (200 at column dim // 2)."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(rows, dim, generator=g, dtype=F64)
    kind = torch.arange(rows) % 5
    mu = torch.tensor([0.3, 30.0, 1000.0, 5.0, 0.5], dtype=F64)[kind]
    sd = torch.tensor([1.5, 1.0, 1.0, 0.0, 1.0], dtype=F64)[kind]
    x = mu[:, None] + sd[:, None] * z
    x[kind == 4, dim // 2] = 200.0
    return x.to(dtype)


def _ln_eager(x32, gamma, beta, eps, dy, out_dtype):
    xe = x32.clone().requires_grad_(True)
    ge, be = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    ye, mean_e, rstd_e = torch.native_layer_norm(xe, (x32.shape[1],), ge, be, eps)
    ye = ye.to(out_dtype)
    ye.backward(dy.to(out_dtype))
    return ye, mean_e.flatten(), rstd_e.flatten(), xe.grad, ge.grad, be.grad


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [8, 40, 768, 1024])
def test_layernorm_fp32(dim):
    """b200_layernorm_fwd/_bwd: fp32 rows read with a row stride > dim, bf16 dy, fp32 dres, dx in fp32 and bf16, dx_colsum."""
    rows, eps, ld = 300, 1e-6, dim + 8
    g = torch.Generator().manual_seed(dim)
    xbuf = torch.zeros(rows, ld, dtype=torch.float32)
    xbuf[:, :dim] = ln_input(rows, dim, dim, torch.float32)
    xbuf = xbuf.to(DEV)
    x = xbuf[:, :dim]
    gamma, beta = torch.randn(dim, generator=g).to(DEV), torch.randn(dim, generator=g).to(DEV)
    dy = torch.randn(rows, dim, generator=g).to(torch.bfloat16).to(DEV)
    dres = torch.randn(rows, dim, generator=g).to(DEV)
    (y64, mean64, rstd64, var64), (dx64, dg64, db64) = with_grads(layernorm, (x, gamma, beta), dy, eps)
    ye, mean_e, rstd_e, dx_e, dg_e, db_e = _ln_eager(x.contiguous(), gamma, beta, eps, dy, torch.bfloat16)

    y, mean, rstd = ops.layernorm_fwd(xbuf, gamma, beta, eps, rows=rows, dim=dim, ld_x=ld)
    dx = torch.empty(rows, dim, device=DEV)
    dxb = torch.empty(rows, dim, device=DEV, dtype=torch.bfloat16)
    dg, db = torch.empty(dim, device=DEV), torch.empty(dim, device=DEV)
    dxs = torch.empty(dim, device=DEV)
    ops.layernorm_bwd(dy, xbuf, gamma, mean, rstd, rows=rows, dim=dim, ld_x=ld, dres=dres, dx_out=dx, ld_dx=dim, dx_bf16=dxb,
                      dgamma=dg, dbeta=db, dx_colsum=dxs)
    torch.cuda.synchronize()
    tag = f"layernorm fp32 dim {dim}"
    _assert_stats(f"{tag}: mean", mean, mean_e, mean64, torch.maximum(mean64.abs(), var64.sqrt()).clamp_min(1e-30))
    _assert_stats(f"{tag}: rstd", rstd, rstd_e, rstd64, rstd64)
    _assert_like_eager(f"{tag}: y", y, ye, y64, per_element=False)  # one element of 230400 at dim 768 is 2 ulp off (eager: 0)
    _assert_like_eager(f"{tag}: dx", dx, dx_e + dres, dx64 + dres.to(F64))
    assert torch.equal(dxb, dx.to(torch.bfloat16)), f"{tag}: dx_bf16 is not bf16(dx)"
    _assert_like_eager(f"{tag}: dgamma", dg, dg_e, dg64)
    _assert_like_eager(f"{tag}: dbeta", db, db_e, db64)
    ref = dxb.to(F64).sum(0)
    assert (dxs.to(F64) - ref).abs().max().item() <= 2.0 ** -8 * ref.abs().max().item() + 1e-6, f"{tag}: dx_colsum"
    assert torch.isfinite(dx[3::5]).all() and torch.equal(y[3::5], beta.to(torch.bfloat16).expand(rows // 5, dim)), f"{tag}: constant rows"


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [8, 40, 768, 1280, 2048])
def test_layernorm_bf16(dim):
    """b200_layernorm_bf16_fwd/_bwd: bf16 rows, dx = bf16(dres + bf16(LN'(dy)))."""
    rows, eps = 300, 1e-5
    g = torch.Generator().manual_seed(dim + 1)
    x = ln_input(rows, dim, dim + 1, torch.bfloat16).to(DEV)
    gamma, beta = torch.randn(dim, generator=g).to(DEV), torch.randn(dim, generator=g).to(DEV)
    dy = torch.randn(rows, dim, generator=g).to(torch.bfloat16).to(DEV)
    dres = torch.randn(rows, dim, generator=g).to(torch.bfloat16).to(DEV)
    (y64, mean64, rstd64, var64), (dx64, dg64, db64) = with_grads(layernorm, (x, gamma, beta), dy, eps)
    ye, mean_e, rstd_e, dx_e, dg_e, db_e = _ln_eager(x.float(), gamma, beta, eps, dy, torch.bfloat16)
    dx_e = dres + dx_e.to(torch.bfloat16)  # eager: the cast back to the bf16 input, then the bf16 residual add

    y, mean, rstd = ops.layernorm_bf16_fwd(x, gamma, beta, eps)
    dx, dg, db = ops.layernorm_bf16_bwd(dy, x, gamma, mean, rstd, dres=dres)
    torch.cuda.synchronize()
    tag = f"layernorm bf16 dim {dim}"
    _assert_stats(f"{tag}: mean", mean, mean_e, mean64, torch.maximum(mean64.abs(), var64.sqrt()).clamp_min(1e-30))
    _assert_stats(f"{tag}: rstd", rstd, rstd_e, rstd64, rstd64)
    _assert_like_eager(f"{tag}: y", y, ye, y64)
    _assert_like_eager(f"{tag}: dx", dx, dx_e, dx64 + dres.to(F64))
    _assert_like_eager(f"{tag}: dgamma", dg, dg_e, dg64)
    _assert_like_eager(f"{tag}: dbeta", db, db_e, db64)
    assert torch.isfinite(dx[3::5].float()).all() and torch.equal(y[3::5], beta.to(torch.bfloat16).expand(rows // 5, dim))


# ---- cross-entropies ---------------------------------------------------------------------------------------------------------------
XENT_CASES = ["large", "dominant_label", "dominant_other", "neg_inf", "C1", "C2", "scale_dev"]


def _padded(vals, ld):
    """bf16 [B, C] view with row stride ld > C (the padding holds a value the kernel must never read: NaN)."""
    buf = torch.full((vals.shape[0], ld), float("nan"), dtype=torch.bfloat16, device=DEV)
    buf[:, :vals.shape[1]] = vals.to(torch.bfloat16).to(DEV)
    return buf[:, :vals.shape[1]]


def xent_input(case, seed):
    """(logits [B, C] float64 before the bf16 cast, labels [B]).  Large logits reach +-3e4; a dominant logit leads by 80."""
    g = torch.Generator().manual_seed(seed)
    B, C = {"C1": (1, 1), "C2": (1, 2)}.get(case, (64, 1000))
    x = torch.randn(B, C, generator=g, dtype=F64) * 3
    lab = torch.randint(0, C, (B,), generator=g)
    rows = torch.arange(B)
    if case == "large":
        x = (x * 1e4).clamp(-3e4, 3e4)
    elif case == "dominant_label":
        x[rows, lab] += 80
    elif case == "dominant_other":
        x[rows, (lab + 1) % C] += 80
    elif case == "neg_inf":
        mask = torch.rand(B, C, generator=g) < 0.3
        mask[rows, lab] = False
        x[mask] = float("-inf")
    return x, lab


@pytest.mark.gpu
@pytest.mark.parametrize("case", XENT_CASES)
def test_softmax_xent(case):
    x, lab = xent_input(case, seed=XENT_CASES.index(case))
    B, C = x.shape
    logits = _padded(x, (C + 15) // 8 * 8)
    labels = lab.to(DEV)
    gs, gsd = (0.5, torch.tensor([3.0], device=DEV)) if case == "scale_dev" else (1.0, None)
    loss_mean, loss_rows, dl, bad = ops.softmax_xent(logits, labels, grad_scale=gs, grad_scale_dev=gsd)
    torch.cuda.synchronize()
    sc = gs * (gsd.item() if gsd is not None else 1.0)
    ref_rows, dl64 = softmax_xent(logits, labels)
    dl64 = dl64 * sc
    lf = logits.float().requires_grad_(True)
    rows_e = F.cross_entropy(lf, labels, reduction="none")
    rows_e.mean().backward()
    dl_e = (lf.grad * sc).to(torch.bfloat16)
    assert bad.item() == 0
    # an fp32 log-sum-exp is worth half an ulp of the largest logit: allow that on top of 4x eager's error
    mag = max(1.0, logits.float()[torch.isfinite(logits.float())].abs().max().item())
    e_ours, e_eager = (loss_rows.to(F64) - ref_rows).abs().max().item(), (rows_e.to(F64) - ref_rows).abs().max().item()
    assert e_ours <= 4 * e_eager + 2.0 ** -23 * mag, f"{case}: loss rows max abs error {e_ours:.3e} (eager {e_eager:.3e}, |logit| {mag:.0f})"
    e_mean = abs(loss_mean.item() - ref_rows.mean().item())
    assert e_mean <= 4 * abs(rows_e.mean().item() - ref_rows.mean().item()) + 2.0 ** -23 * mag + 1e-6 * abs(ref_rows.mean().item()), (case, e_mean)
    _assert_like_eager(f"softmax_xent {case}: dlogits", dl, dl_e, dl64)


@pytest.mark.gpu
@pytest.mark.parametrize("case", XENT_CASES)
def test_symmetric_xent(case):
    x, _ = xent_input(case, seed=10 + XENT_CASES.index(case))
    B = min(x.shape)
    x = x[:B, :B].clone()
    if case == "C2":  # B = 2: a 2 x 2 logit matrix
        x = torch.randn(2, 2, generator=torch.Generator().manual_seed(2), dtype=F64) * 3
        B = 2
    elif case.startswith("dominant"):  # the dominant logit of each row on (or off) the diagonal
        x = torch.randn(B, B, generator=torch.Generator().manual_seed(3), dtype=F64) * 3
        x[torch.arange(B), torch.arange(B) if case == "dominant_label" else (torch.arange(B) + 1) % B] += 80
    elif case == "neg_inf":
        x.fill_diagonal_(0.0)
    ld = (B + 15) // 8 * 8
    logits = _padded(x, ld)
    gs, gsd = (0.5, torch.tensor([3.0], device=DEV)) if case == "scale_dev" else (1.0, None)
    dl = torch.zeros(B, ld, dtype=torch.bfloat16, device=DEV)[:, :B]
    loss = ops.symmetric_xent(logits, dlogits=dl, grad_scale=gs, grad_scale_dev=gsd)
    torch.cuda.synchronize()
    sc = gs * (gsd.item() if gsd is not None else 1.0)
    ref, dl64 = symmetric_xent(logits)
    idx = torch.arange(B, device=DEV)
    lf = logits.float().requires_grad_(True)
    loss_e = 0.5 * (F.cross_entropy(lf, idx) + F.cross_entropy(lf.t(), idx))
    loss_e.backward()
    mag = max(1.0, logits.float()[torch.isfinite(logits.float())].abs().max().item())
    e_ours, e_eager = abs(loss.item() - ref.item()), abs(loss_e.item() - ref.item())
    assert e_ours <= 4 * e_eager + 2.0 ** -23 * mag + 1e-6 * abs(ref.item()), f"{case}: loss error {e_ours:.3e} (eager {e_eager:.3e})"
    _assert_like_eager(f"symmetric_xent {case}: dlogits", dl, (lf.grad * sc).to(torch.bfloat16), dl64 * sc)


# ---- attention with peaked scores --------------------------------------------------------------------------------------------------
def _row_errors(x, ref):
    """Per-row L2 error of [..., T, D] tensors, relative to the row's own norm."""
    return (x.to(F64) - ref).norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-300)


def _check_attention(tag, q, k, v, dout, scale, causal, out, lse, dq, dk, dv):
    """q, k, v, dout: bf16 [B, H, T, D] on the device; the kernel's results in the same layout (lse [B, H, Tq])."""
    (o64, lse64), (dq64, dk64, dv64) = with_grads(attention, (q, k, v), dout, scale, causal)
    qe, ke, ve = (t.clone().requires_grad_(True) for t in (q, k, v))
    oe = F.scaled_dot_product_attention(qe, ke, ve, is_causal=causal, scale=scale)
    oe.backward(dout)
    # out: every row against float64, no further than 2x eager's row error + one bf16 ulp
    ro, re = _row_errors(out, o64), _row_errors(oe, o64)
    bad = ro > 2 * re + 2.0 ** -7
    w = ro.argmax().item()
    assert not bad.any(), (f"{tag}: {int(bad.sum())} of {ro.numel()} output rows off (worst row {w}: {ro.flatten()[w]:.3e}, eager "
                           f"{re.flatten()[w]:.3e})")
    le = (lse.to(F64) - lse64).abs() / lse64.abs().clamp_min(1.0)
    assert le.max().item() <= 1e-3, f"{tag}: lse error {le.max().item():.3e} at flat index {le.argmax().item()}"
    for name, ours, eager, ref in (("dq", dq, qe.grad, dq64), ("dk", dk, ke.grad, dk64), ("dv", dv, ve.grad, dv64)):
        if ref.norm().item() == 0.0:  # one key: P = 1 and dS = 0 exactly, so dq / dk are 0 and only rounding noise may remain
            assert ours.to(F64).norm().item() <= 1e-3 * dv64.norm().item(), (tag, name, ours.float().norm().item())
            continue
        e_ours, e_eager = relerr(ours, ref), relerr(eager, ref)
        assert e_ours <= 2 * e_eager + 1e-3, f"{tag}: {name} relative L2 {e_ours:.3e} (eager {e_eager:.3e})"
        rms = ref.norm(dim=-1).pow(2).mean().sqrt().item()  # a wrong row stands out against the typical row norm
        r_ours = ((ours.to(F64) - ref).norm(dim=-1) / rms).max().item()
        r_eager = ((eager.to(F64) - ref).norm(dim=-1) / rms).max().item()
        assert r_ours <= 2 * r_eager + 1e-2, f"{tag}: {name} worst row error {r_ours:.3e} of the rms row norm (eager {r_eager:.3e})"


def _packed_case(B, T, H, causal, seed):
    q, k, v = (t.to(torch.bfloat16).to(DEV) for t in peaked_qkv(B, H, T, T, 64, 0.125, causal, seed))
    qkv = torch.stack([t.permute(0, 2, 1, 3) for t in (q, k, v)], 2).reshape(B * T, 3 * H * 64).contiguous()
    dout = torch.randn(B, H, T, 64, generator=torch.Generator().manual_seed(seed + 1)).to(torch.bfloat16).to(DEV)
    out, lse = ops.attention_fwd(qkv, B, T, H, scale=0.125, causal=causal)
    dqkv = ops.attention_bwd(qkv, out, dout.permute(0, 2, 1, 3).reshape(B * T, H * 64).contiguous(), lse, B, T, H, scale=0.125, causal=causal)
    torch.cuda.synchronize()
    heads = lambda t: t.reshape(B, T, H, 64).permute(0, 2, 1, 3)  # noqa: E731
    d = dqkv.view(B, T, 3, H * 64)
    _check_attention(f"attention B{B} T{T} H{H} causal={causal}", q, k, v, dout, 0.125, causal, heads(out), lse,
                     heads(d[:, :, 0]), heads(d[:, :, 1]), heads(d[:, :, 2]))


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("B,T,H", [(2, 77, 4), (2, 197, 4), (2, 256, 2)])
def test_attention_peaked(B, T, H, causal):
    _packed_case(B, T, H, causal, seed=T + int(causal))


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("B,T,H", [(2, 300, 4), (1, 1025, 4), (1, 4096, 2)])
def test_long_attention_peaked(B, T, H, causal):
    _packed_case(B, T, H, causal, seed=T + int(causal))


def _cross_case(B, Tq, Tk, H, Dh, causal, seed):
    scale = Dh ** -0.5
    q, k, v = (t.to(torch.bfloat16).to(DEV) for t in peaked_qkv(B, H, Tq, Tk, Dh, scale, causal, seed))
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(-1, H * Dh).contiguous()  # noqa: E731
    dout = torch.randn(B, H, Tq, Dh, generator=torch.Generator().manual_seed(seed + 1)).to(torch.bfloat16).to(DEV)
    out, lse = ops.cross_attention_fwd(rows(q), rows(k), rows(v), B, H, scale=scale, causal=causal)
    dq, dk, dv = ops.cross_attention_bwd(rows(q), rows(k), rows(v), out, rows(dout), lse, B, H, scale=scale, causal=causal)
    torch.cuda.synchronize()
    heads = lambda t: t.view(B, -1, H, Dh).permute(0, 2, 1, 3)  # noqa: E731
    _check_attention(f"cross_attention B{B} Tq{Tq} Tk{Tk} H{H} Dh{Dh} causal={causal}", q, k, v, dout, scale, causal, heads(out), lse,
                     heads(dq), heads(dk), heads(dv))


@pytest.mark.gpu
@pytest.mark.parametrize("Tk", [1, 77, 200])
@pytest.mark.parametrize("Dh", [40, 80, 160])
def test_cross_attention_peaked(Dh, Tk):
    _cross_case(2, 300, Tk, 8, Dh, False, seed=Dh + Tk)


@pytest.mark.gpu
@pytest.mark.parametrize("Dh", [40, 80, 160])
def test_cross_attention_peaked_causal(Dh):
    _cross_case(2, 200, 200, 8, Dh, True, seed=Dh)


# ---- modules on inputs whose channel groups share an offset -------------------------------------------------------------------------
def _check_modules(ours, eager, fp32):
    for k in ours:
        floor = relerr(eager[k], fp32[k].to(F64))
        e_f, e_e = relerr(ours[k], fp32[k]), relerr(ours[k], eager[k])
        assert e_f <= 1.5 * floor + 1e-6, f"{k}: vs fp32 {e_f:.3e}, eager vs fp32 {floor:.3e}"
        assert e_e <= 2.0 * floor + 1e-6, f"{k}: vs eager {e_e:.3e}, eager vs fp32 {floor:.3e}"


def _offset_input(B, C, side, seed):
    g = torch.Generator().manual_seed(seed)
    net = (4.0 + 0.02 * torch.randn(B, C, side, side, generator=g)).to(torch.bfloat16)
    return net.to(DEV).contiguous(memory_format=torch.channels_last), g


@pytest.mark.gpu
def test_res_block_on_offset_input():
    import unet_oracle as uo
    from cflearn_b200.unet_blocks import ResidualBlockWithTimeEmbeddingB200 as ResBlock

    B, C, side, tdim = 2, 320, 32, 1280
    m = ResBlock(C, C, norm_eps=1e-5, time_embedding_channels=tdim)
    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=3)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV)
    net, g = _offset_input(B, C, side, seed=4)
    tn = torch.randn(B, tdim, generator=g).to(DEV).to(torch.bfloat16)
    up = torch.randn(B, C, side, side, generator=g).to(DEV)
    x, t = net.detach().clone().requires_grad_(True), tn.detach().clone().requires_grad_(True)
    y = m(x, t)
    (y.float() * up).sum().backward()
    ours = {"out": y, "net": x.grad, "time_net": t.grad, **{k: p.grad for k, p in m.named_parameters()}}
    refs = []
    for autocast in (True, False):
        sdg = {k: v.detach().clone().to(DEV).requires_grad_(True) for k, v in sd.items()}
        xr = (net if autocast else net.float()).detach().clone().requires_grad_(True)
        tr = (tn if autocast else tn.float()).detach().clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            yr = uo.res_block(sdg, "", xr, tr)
        (yr.float() * up).sum().backward()
        refs.append({"out": yr, "net": xr.grad, "time_net": tr.grad, **{k: v.grad for k, v in sdg.items()}})
    _check_modules(ours, *refs)


@pytest.mark.gpu
def test_spatial_transformer_on_offset_input():
    import unet_oracle as uo
    from cflearn_b200.spatial_transformer import SpatialTransformerB200

    B, C, side, heads = 2, 320, 32, 8
    m = SpatialTransformerB200(C, heads, C // heads, context_dim=768)
    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=5)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV)
    net, g = _offset_input(B, C, side, seed=6)
    context = torch.randn(B, 77, 768, generator=g).to(DEV)
    up = torch.randn(B, C, side, side, generator=g).to(DEV)
    x, c = net.detach().clone().requires_grad_(True), context.detach().clone().requires_grad_(True)
    y = m(x, c)
    (y.float() * up).sum().backward()
    ours = {"out": y, "net": x.grad, "context": c.grad, **{k: p.grad for k, p in m.named_parameters()}}
    refs = []
    for autocast in (True, False):
        sdg = {k: v.detach().clone().to(DEV).requires_grad_(True) for k, v in sd.items()}
        xr = (net if autocast else net.float()).detach().clone().requires_grad_(True)
        cr = context.detach().clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            yr = uo.spatial_transformer(sdg, "", xr, cr, heads)
        (yr.float() * up).sum().backward()
        refs.append({"out": yr, "net": xr.grad, "context": cr.grad, **{k: v.grad for k, v in sdg.items()}})
    _check_modules(ours, *refs)
