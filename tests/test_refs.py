"""CPU: every float64 reference in _refs.py against torch's own op on small inputs."""
import torch
import torch.nn.functional as F

import _refs as refs
from test_ill_conditioned_gpu import gn_input

F64 = torch.float64


def test_float64_references_match_torch():
    g = torch.Generator().manual_seed(0)
    g2 = torch.Generator().manual_seed(1)  # the draws the backward checks add
    # GroupNorm(32) (+ SiLU) on channels-last rows with every kind of ill-conditioned group, its statistics and its backward
    x = gn_input(2, 49, 64, "mixed", seed=1)
    gamma, beta = torch.randn(64, generator=g, dtype=F64), torch.randn(64, generator=g, dtype=F64)
    dy = torch.randn(2, 49, 64, generator=g2, dtype=F64)
    for silu in (False, True):
        (y, mean, rstd, _), grads = refs.with_grads(refs.groupnorm, (x, gamma, beta), dy, 1e-5, silu)
        xt = x.to(F64).permute(0, 2, 1).requires_grad_(True)
        gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        want = F.group_norm(xt, refs.GROUPS, gt, bt, 1e-5)
        want = (F.silu(want) if silu else want).permute(0, 2, 1)
        want.backward(dy)
        assert torch.allclose(y, want.detach(), rtol=1e-12, atol=1e-12)
        for ours, theirs in zip(grads, (xt.grad.permute(0, 2, 1), gt.grad, bt.grad)):
            assert torch.allclose(ours, theirs, rtol=1e-9, atol=1e-9)
        _, m2, r2 = torch.native_group_norm(x.to(F64).permute(0, 2, 1).contiguous(), gamma, beta, 2, 64, 49, refs.GROUPS, 1e-5)
        assert torch.allclose(mean, m2, rtol=1e-12, atol=1e-12) and torch.allclose(rstd, r2, rtol=1e-9)
    # LayerNorm on float64, fp32 and bf16 rows, its statistics and its backward
    xl = torch.randn(37, 40, generator=g, dtype=F64) * 3 + 1e3
    dyl = torch.randn(37, 40, generator=g2, dtype=F64)
    for dtype in (F64, torch.float32, torch.bfloat16):
        xs = xl.to(dtype)
        (y, mean, rstd, var), grads = refs.with_grads(refs.layernorm, (xs, gamma[:40], beta[:40]), dyl, 1e-6)
        xt, gt, bt = (t.to(F64).clone().requires_grad_(True) for t in (xs, gamma[:40], beta[:40]))
        want = F.layer_norm(xt, (40,), gt, bt, 1e-6)
        want.backward(dyl)
        assert torch.allclose(y, want.detach(), rtol=1e-10, atol=1e-10)
        for ours, theirs in zip(grads, (xt.grad, gt.grad, bt.grad)):
            assert torch.allclose(ours, theirs, rtol=1e-9, atol=1e-9)
        _, m2, r2 = torch.native_layer_norm(xs.to(F64), (40,), None, None, 1e-6)
        assert torch.allclose(mean, m2.flatten(), rtol=1e-12) and torch.allclose(rstd, r2.flatten(), rtol=1e-9)
        assert torch.allclose(var, xs.to(F64).var(-1, unbiased=False), rtol=1e-9)
    # log-softmax with a -inf logit, softmax cross-entropy and the symmetric cross-entropy
    logits = torch.randn(9, 31, generator=g, dtype=F64) * 300
    logits[0, 3] = float("-inf")
    lsm = refs.log_softmax(logits)
    assert torch.equal(torch.isinf(lsm), torch.isinf(logits))
    assert torch.allclose(lsm[torch.isfinite(logits)], F.log_softmax(logits, -1)[torch.isfinite(logits)], rtol=1e-12)
    labels = torch.randint(0, 31, (9,), generator=g2)
    labels[0] = 2
    rows, dl = refs.softmax_xent(logits, labels)
    lt = logits.clone().requires_grad_(True)
    want = F.cross_entropy(lt, labels, reduction="none")
    want.mean().backward()
    assert torch.allclose(rows, want.detach(), rtol=1e-12) and torch.allclose(dl, lt.grad, rtol=1e-10, atol=1e-14)
    sq = torch.randn(7, 7, generator=g2, dtype=F64) * 4
    sq[2, 5] = float("-inf")
    loss, dsq = refs.symmetric_xent(sq)
    st = sq.clone().requires_grad_(True)
    want = 0.5 * (F.cross_entropy(st, torch.arange(7)) + F.cross_entropy(st.t(), torch.arange(7)))
    want.backward()
    assert torch.allclose(loss, want.detach(), rtol=1e-12) and torch.allclose(dsq, st.grad, rtol=1e-10, atol=1e-14)
    # attention on [B, H, T, D] with scale and causal; on rows with Tq != Tk, backward included; on packed qkv rows
    q, k, v = (torch.randn(2, 3, 50, 40, generator=g, dtype=F64) for _ in range(3))
    for causal in (False, True):
        o, lse = refs.attention(q * 10, k, v, 40 ** -0.5, causal)
        assert torch.allclose(o, F.scaled_dot_product_attention(q * 10, k, v, is_causal=causal), rtol=1e-10, atol=1e-10)
        s = (q * 10) @ k.transpose(-1, -2) * 40 ** -0.5
        if causal:
            s = s.masked_fill(torch.ones(50, 50, dtype=torch.bool).triu(1), float("-inf"))
        assert torch.allclose(lse, torch.logsumexp(s, -1), rtol=1e-12)
    B, Tq, Tk, H, Dh = 2, 5, 9, 3, 8
    qr, kr, vr = (torch.randn(B * T, H * Dh, generator=g2, dtype=F64) for T in (Tq, Tk, Tk))
    dout = torch.randn(B * Tq, H * Dh, generator=g2, dtype=F64)
    (o, lse), grads = refs.with_grads(refs.attention_rows, (qr, kr, vr), dout, B, H, 0.3, False)
    heads = lambda t: t.view(B, -1, H, Dh).permute(0, 2, 1, 3)  # noqa: E731
    qt, kt, vt = (t.clone().requires_grad_(True) for t in (qr, kr, vr))
    want = F.scaled_dot_product_attention(heads(qt), heads(kt), heads(vt), scale=0.3).permute(0, 2, 1, 3).reshape(B * Tq, H * Dh)
    want.backward(dout)
    assert torch.allclose(o, want.detach(), rtol=1e-10, atol=1e-10) and lse.shape == (B, H, Tq)
    for ours, theirs in zip(grads, (qt.grad, kt.grad, vt.grad)):
        assert torch.allclose(ours, theirs, rtol=1e-9, atol=1e-10)
    qkv = torch.randn(2 * 20, 3 * 2 * 64, generator=g2, dtype=F64)
    o, lse = refs.packed_attention(qkv, 2, 20, 2, causal=True)
    pq, pk, pv = qkv.view(2, 20, 3, 2, 64).permute(2, 0, 3, 1, 4)
    want = F.scaled_dot_product_attention(pq, pk, pv, is_causal=True, scale=0.125).permute(0, 2, 1, 3).reshape(40, 128)
    assert torch.allclose(o, want, rtol=1e-10, atol=1e-10) and lse.shape == (2, 2, 20)
    # the 3x3 convolution and its weight gradient (packed order: tap, then channel)
    xc = torch.randn(2, 5, 6, 8, generator=g2, dtype=F64)
    w = torch.randn(4, 8, 3, 3, generator=g2, dtype=F64, requires_grad=True)
    y = F.conv2d(xc.permute(0, 3, 1, 2), w, padding=1)
    dyc = torch.randn(y.shape, generator=g2, dtype=F64)
    y.backward(dyc)
    assert torch.allclose(refs.conv3x3(xc, w.detach()), y.detach().permute(0, 2, 3, 1).reshape(60, 4), rtol=1e-12, atol=1e-12)
    dw = refs.conv3x3_wgrad(dyc.permute(0, 2, 3, 1).reshape(60, 4), xc)
    assert torch.allclose(dw, w.grad.permute(0, 2, 3, 1).reshape(4, 72), rtol=1e-10, atol=1e-12)
    # Adam with L2 weight decay against torch.optim.Adam
    p0, grad = torch.randn(50, generator=g2, dtype=F64), torch.randn(50, generator=g2, dtype=F64)
    pt = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([pt], lr=1e-2, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.05)
    for _ in range(4):
        pt.grad = grad.clone()
        opt.step()
    zeros = torch.zeros(50, dtype=F64)
    p, m, v = refs.adam(p0, grad, zeros, zeros, [1, 2, 3, 4], 1e-2, 0.8, 0.99, 1e-6, 0.05)
    assert torch.allclose(p, pt.detach(), rtol=1e-12, atol=1e-14)
    assert torch.allclose(m, opt.state[pt]["exp_avg"], rtol=1e-12) and torch.allclose(v, opt.state[pt]["exp_avg_sq"], rtol=1e-12)
    # AdamW (decoupled decay) against torch.optim.AdamW, from nonzero moments at step 3 as the footprint case starts; a scaled
    # gradient is the same update on the scaled gradient, the decay untouched
    m0 = 0.1 * torch.randn(50, generator=g2, dtype=F64)
    v0 = (0.1 * torch.randn(50, generator=g2, dtype=F64)) ** 2
    for gs in (1.0, 0.5):
        pt = p0.clone().requires_grad_(True)
        opt = torch.optim.AdamW([pt], lr=1e-2, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.05)
        opt.state[pt] = {"step": torch.tensor(2.0), "exp_avg": m0.clone(), "exp_avg_sq": v0.clone()}
        for _ in range(4):
            pt.grad = grad * gs
            opt.step()
        p, m, v = refs.adam(p0, grad, m0, v0, [3, 4, 5, 6], 1e-2, 0.8, 0.99, 1e-6, 0.05, gs, decoupled=True)
        assert torch.allclose(p, pt.detach(), rtol=1e-12, atol=1e-14)
        assert torch.allclose(m, opt.state[pt]["exp_avg"], rtol=1e-12) and torch.allclose(v, opt.state[pt]["exp_avg_sq"], rtol=1e-12)
        assert not torch.allclose(p, refs.adam(p0, grad, m0, v0, [3, 4, 5, 6], 1e-2, 0.8, 0.99, 1e-6, 0.05, gs)[0], rtol=1e-6)


def test_attention_bounds():
    g = torch.Generator().manual_seed(2)
    bf = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)  # noqa: E731
    B, H, Tq, Tk, D, scale = 2, 3, 7, 9, 16, 0.3
    q, dout, k, v = bf(B, H, Tq, D), bf(B, H, Tq, D), bf(B, H, Tk, D), bf(B, H, Tk, D)
    for causal, kk, vv in ((False, k, v), (True, k[:, :, :Tq], v[:, :, :Tq])):
        # the float64 values it returns are attention's forward and autograd gradients
        (o, lse, dq, dk, dv), tols = refs.attention_bounds(q, kk, vv, dout, scale, causal, q)
        (o2, lse2), grads = refs.with_grads(refs.attention, (q, kk, vv), dout, scale, causal)
        assert torch.allclose(o, o2, rtol=1e-12, atol=1e-14) and torch.allclose(lse, lse2, rtol=1e-12)
        for ours, theirs in zip((dq, dk, dv), grads):
            assert torch.allclose(ours, theirs, rtol=1e-10, atol=1e-12)
        assert [t.shape for t in tols] == [o.shape, dq.shape, dk.shape, dv.shape] and all((t > 0).all() for t in tols)
        # the row-layout wrapper is the same computation on [B T, H D] rows
        rows = lambda t: t.permute(0, 2, 1, 3).reshape(-1, H * D)  # noqa: E731
        r_vals, r_tols = refs.attention_bounds_rows(rows(q), rows(kk), rows(vv), rows(dout), B, H, scale, causal, rows(q))
        assert torch.allclose(r_vals[1], lse, rtol=1e-14)
        for a, b in zip((r_vals[0],) + r_vals[2:] + r_tols, (o, dq, dk, dv) + tols):
            assert torch.allclose(a, rows(b), rtol=1e-12, atol=1e-15)

    # nothing above the underflow floor (2^-126 flushes) where the quantity is exact: o with V = 0, every gradient with dO = 0
    (o, *_), (tol_o, *_) = refs.attention_bounds(q, k, torch.zeros_like(v), dout, scale, False, torch.zeros_like(q))
    assert torch.equal(o, torch.zeros_like(o, dtype=F64)) and (tol_o <= 2.0 ** -100).all()
    _, (_, *tol_grads) = refs.attention_bounds(q, k, v, torch.zeros_like(dout), scale, False, q)
    assert all((t <= 2.0 ** -100).all() for t in tol_grads)
    # one key: P = 1, out = v exactly, dS = 0, so dq = dk = 0 and their tolerance is only the fp32 rounding of dP and delta
    k1, v1 = k[:, :, :1], v[:, :, :1]
    (o, _, dq, dk, dv), (tol_o, tol_dq, tol_dk, tol_dv) = refs.attention_bounds(q, k1, v1, dout, scale, False, v1.expand(-1, -1, Tq, -1))
    assert torch.equal(o, v1.to(F64).expand_as(o)) and dq.abs().max() < 1e-12 and dk.abs().max() < 1e-12
    w = dout.to(F64).abs() @ v1.to(F64).abs().transpose(-1, -2)  # sum_d |dO_id| |v_d|: the magnitude of dP and delta
    assert (tol_dq <= 2.0 ** -14 * scale * (w @ k1.to(F64).abs())).all()
    assert (tol_dk <= 2.0 ** -14 * scale * (w.transpose(-1, -2) @ q.to(F64).abs())).all()
    assert (tol_dv >= 2.0 ** -8 * dv.abs()).all() and (tol_o >= 2.0 ** -8 * o.abs()).all()

    # monotone: a larger |V| never shrinks tol_o, a larger |dO| never shrinks tol_dv (and doubling either doubles them)
    grow = lambda t: (t.float() * (1 + torch.rand(t.shape, generator=g))).to(torch.bfloat16)  # noqa: E731
    for causal, kk, vv in ((False, k, v), (True, k[:, :, :Tq], v[:, :, :Tq])):
        base = refs.attention_bounds(q, kk, vv, dout, scale, causal, q)[1]
        bigger_v = refs.attention_bounds(q, kk, grow(vv), dout, scale, causal, q)[1]
        bigger_do = refs.attention_bounds(q, kk, vv, grow(dout), scale, causal, q)[1]
        assert (bigger_v[0] >= base[0]).all() and (bigger_do[3] >= base[3]).all()
        assert torch.allclose(refs.attention_bounds(q, kk, 2 * vv, dout, scale, causal, q)[1][0], 2 * base[0], rtol=1e-12)
        assert torch.allclose(refs.attention_bounds(q, kk, vv, 2 * dout, scale, causal, q)[1][3], 2 * base[3], rtol=1e-12)


def test_gemm_and_conv_references():
    g = torch.Generator().manual_seed(3)
    # the input gradient of the 3x3 convolution against autograd of F.conv2d
    xc = torch.randn(2, 5, 6, 8, generator=g, dtype=F64, requires_grad=True)
    w = torch.randn(4, 8, 3, 3, generator=g, dtype=F64)
    y = F.conv2d(xc.permute(0, 3, 1, 2), w, padding=1)
    dyc = torch.randn(y.shape, generator=g, dtype=F64)
    y.backward(dyc)
    assert torch.allclose(refs.conv3x3_dgrad(dyc.permute(0, 2, 3, 1), w), xc.grad.reshape(60, 8), rtol=1e-12, atol=1e-12)
    # exact operands: bf16 ints times 2^exp per row, the cancelling pair in place, the budget enforced
    ea, eb = refs.exponents(5, -20, 20, 1), refs.exponents(3, -20, 20, 2)
    A, B = refs.exact_operands(5, 3, 100, ea, eb, cancel=refs.cancel_pairs(100, "kblock"))
    assert (A[:, 63].double() == 2.0 ** (10 + ea)).all() and (B[:, 64].double() == -(2.0 ** (10 + eb))).all()
    units = (A.double() * torch.exp2(-ea)[:, None]).abs() @ (B.double() * torch.exp2(-eb)[:, None]).abs().t()
    assert units.max() < refs.EXACT_BUDGET and torch.equal(units, units.round())
    x, wc = refs.exact_conv_operands(2, 4, 4, 64, 8, refs.exponents(2, -3, 3, 3), refs.exponents(8, -3, 3, 4))
    assert x.dtype == wc.dtype == torch.bfloat16 and x.shape == (2, 4, 4, 64) and wc.shape == (8, 64, 3, 3)
    xw, dyw = refs.exact_wgrad_operands(1, 8, 8, 64, 8, refs.exponents(64, -3, 3, 5), refs.exponents(8, -3, 3, 6)[None, :])
    assert xw.shape == (1, 8, 8, 64) and dyw.shape == (64, 8)
    assert refs.splitk_ranges(200, 5) == [(0, 64), (64, 128), (128, 192), (192, 200)]
    # t = bf16(fp32(acc + bias)): ties go to even (257 -> 256, 259 -> 260); the fp32 rounding comes first (2^24 + 1 + 2^-30)
    acc = torch.tensor([[257.0, 259.0, 2.0 ** 24 + 1]], dtype=F64)
    t = refs.gemm_t(acc, torch.tensor([0.0, 0.0, 2.0 ** -30], dtype=torch.bfloat16))
    assert t.float().tolist() == [[256.0, 260.0, 2.0 ** 24]]
    # the bf16 adds and the clamp of epilogue 11
    big = torch.finfo(torch.bfloat16).max
    s = refs.add_bf16(torch.tensor([big, -big, 1.0, float("nan")]).to(torch.bfloat16), torch.tensor([big, -big, 2.0 ** -8, 0.0]).to(torch.bfloat16), clamp=True)
    assert s[:3].float().tolist() == [big, -big, 1.0] and torch.isnan(s[3])
    # the epilogues of functions of t against torch: GELU, dGELU, QuickGELU (eager's roundings on bf16 tensors), GEGLU and dGEGLU
    tb = (torch.randn(6, 16, generator=g) * 2).to(torch.bfloat16)
    hb = (torch.randn(6, 16, generator=g) * 2).to(torch.bfloat16)
    out = refs.gemm_epilogue(1, tb)
    assert torch.equal(out["out0"][0], tb) and out["out0"][1] is None
    assert torch.allclose(out["out1"][0], F.gelu(tb.double()), rtol=1e-12, atol=1e-15)
    hd = hb.double().requires_grad_(True)
    F.gelu(hd).backward(tb.double())
    assert torch.allclose(refs.gemm_epilogue(3, tb, hb)["out0"][0], hd.grad, rtol=1e-12, atol=1e-15)
    eager = tb * torch.sigmoid(tb * 1.702)  # bf16 CPU tensors: one rounding per op
    assert torch.equal(refs.bf16(refs.gemm_epilogue(5, tb)["out1"][0]), eager)
    hq = hb.clone().requires_grad_(True)
    (hq * torch.sigmoid(hq * 1.702)).backward(tb)
    ref6, tol6 = refs.gemm_epilogue(6, tb, hb)["out0"]
    assert ((hq.grad.double() - ref6).abs() <= tol6).all()
    hg = torch.cat([tb, hb], 1)
    ref7, _ = refs.gemm_epilogue(7, hg)["out1"]
    assert torch.allclose(ref7, tb.double() * F.gelu(hb.double()).to(torch.bfloat16).double(), rtol=1e-12, atol=1e-15)
    hgd = hg.double().requires_grad_(True)
    (hgd[:, :16] * F.gelu(hgd[:, 16:])).backward(tb.double())
    ref8, tol8 = refs.gemm_epilogue(8, tb, hg)["out0"]
    assert ((ref8 - hgd.grad).abs() <= tol8).all()
    aux = torch.randn(6, 16, generator=g)
    assert torch.equal(refs.gemm_epilogue(2, tb, aux)["out0"][0], aux + tb.float())
    assert torch.equal(refs.gemm_epilogue(9, tb, hb)["out0"][0], (tb.float() + hb.float()).to(torch.bfloat16))


def test_resample_and_per_image_references():
    """The stride-2 / nearest-2x convolution references and their gradients against torch's autograd of the same fp32 ops, and the
    per-image column sums against a loop over images."""
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 8, 6, 5, generator=g)  # channels-last [B, H, W, Cin]
    w = torch.randn(4, 5, 3, 3, generator=g)
    xf, wf = x.permute(0, 3, 1, 2).clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = F.conv2d(xf, wf, stride=2, padding=1)
    dy = torch.randn(y.shape, generator=g)
    y.backward(dy)
    dy_nhwc = dy.permute(0, 2, 3, 1)
    assert torch.allclose(refs.conv3x3_s2(x, w).float(), y.detach().permute(0, 2, 3, 1), atol=1e-5)
    assert torch.allclose(refs.conv3x3_s2_dgrad(dy_nhwc, w, 8, 6).float(), xf.grad.permute(0, 2, 3, 1), atol=1e-5)
    assert torch.allclose(refs.conv3x3_s2_wgrad(dy_nhwc, x).float(), wf.grad.permute(0, 2, 3, 1).reshape(4, -1), atol=1e-4)
    up = F.conv2d(F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="nearest"), w, padding=1)
    assert torch.allclose(refs.conv3x3_up2(x, w).float(), up.permute(0, 2, 3, 1), atol=1e-5)
    per, tot = refs.colsum_per_image(x)
    assert torch.allclose(per.float(), torch.stack([x[b].reshape(-1, 5).sum(0) for b in range(2)]), atol=1e-5)
    assert torch.allclose(tot.float(), x.reshape(-1, 5).sum(0), atol=1e-5)


def test_fcnn_reference():
    """fcnn_step against torch's autograd of the same float64 network (Linear, ReLU, l1_loss, mse_loss) on an arena with gaps and a
    layer without bias, with ReLU inputs and residuals planted at exactly 0; fcnn_bounds returns the same values."""
    g = torch.Generator().manual_seed(8)
    dims, woff, boff, P = [5, 7, 6, 3], [50, 0, 100], [90, -1, 120], 126
    halves = lambda *shape: torch.randint(-6, 7, shape, generator=g).to(F64) / 2  # noqa: E731  (sums exact: the zeros below are 0)
    params = torch.full((P,), float("nan"), dtype=F64)
    x = halves(9, 5)
    for l in range(3):
        params[woff[l]:woff[l] + dims[l] * dims[l + 1]] = halves(dims[l] * dims[l + 1])
        if boff[l] >= 0:
            params[boff[l]:boff[l] + dims[l + 1]] = halves(dims[l + 1])
    # pre-activation of unit 2, row 4 exactly 0 (the bias cancels it)
    W0 = params[woff[0]:woff[0] + 35].view(7, 5)
    params[boff[0] + 2] = -(x[4] @ W0[2])
    y, dpred = halves(9, 3) + 0.25, halves(9, 3)
    keys = [(woff[l], dims[l] * dims[l + 1]) for l in range(3)] + [(boff[l], dims[l + 1]) for l in range(3) if boff[l] >= 0]

    def autograd(target, w, use_dpred):
        leaves = [params[o:o + n].clone().requires_grad_(True) for o, n in keys]
        W = [leaves[l].view(dims[l + 1], dims[l]) for l in range(3)]
        b = {0: leaves[3], 2: leaves[4]}
        a = x
        for l in range(3):
            a = F.linear(a, W[l], b.get(l))
            if l < 2:
                a = torch.relu(a)
        pred = a
        if use_dpred:
            pred.backward(target)
            loss = None
        else:
            loss = w[0] * F.l1_loss(pred, target) + w[1] * F.mse_loss(pred, target)
            loss.backward()
        grads = torch.zeros(P, dtype=F64)
        for (o, n), t in zip(keys, leaves):
            grads[o:o + n] = t.grad
        return pred.detach(), loss, grads

    _, acts = refs.fcnn_forward(x, refs.fcnn_layers(params, dims, woff, boff))
    y_zero = y.clone()
    y_zero[1, 2] = acts[-1][1, 2]  # residual exactly 0: sign(0) = 0
    assert acts[1][4, 2] == 0
    for kw, w in ((dict(y=y_zero), (0.5, 2.0)), (dict(y=y), (1.0, 0.0)), (dict(dpred=dpred), (1.0, 1.0))):
        pred, loss, grads = refs.fcnn_step(x, params, dims, woff, boff, w_mae=w[0], w_mse=w[1], **kw)
        want_pred, want_loss, want_grads = autograd(kw.get("y", kw.get("dpred")), w, "dpred" in kw)
        assert torch.allclose(pred, want_pred, rtol=1e-12, atol=1e-12)
        assert (loss is None) == (want_loss is None) and (loss is None or torch.allclose(loss, want_loss, rtol=1e-12))
        bad = ~torch.isclose(grads, want_grads, rtol=1e-10, atol=1e-12)
        assert not bad.any(), (kw.keys(), torch.nonzero(bad).flatten().tolist(), grads[bad], want_grads[bad])
        gaps = torch.ones(P, dtype=torch.bool)
        for o, n in keys:
            gaps[o:o + n] = False
        assert (grads[gaps] == 0).all() and not torch.signbit(grads).logical_and(grads == 0).any()
        (p2, l2, g2), (tp, tl, tg) = refs.fcnn_bounds(x, params, dims, woff, boff, w_mae=w[0], w_mse=w[1], **kw)
        assert torch.equal(p2, pred) and torch.equal(g2, grads) and (l2 is None or torch.equal(l2, loss))
        assert tp.shape == pred.shape and tg.shape == grads.shape and (tp > 0).all() and (tg[~gaps] >= 0).all()
        assert (tl is None) == (loss is None) and (tl is None or tl > 0)
