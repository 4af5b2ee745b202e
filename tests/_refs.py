"""What the GPU tests compare the kernels against: seeded inputs, error measures and float64 references.

Every reference computes in torch.float64 on the device its inputs are on and returns everything its tests compare against.  A
backward is the autograd of the same float64 maths (``with_grads``), except for the losses, whose gradients are closed forms.
``test_refs.py`` checks each reference against torch's own op on small inputs."""
import math

import torch
import torch.nn.functional as F

F64 = torch.float64
GROUPS = 32  # GroupNorm(32), as in the SD-UNet


# ---- inputs ------------------------------------------------------------------------------------------------------------------------
def rand_bf16(*shape, scale=1.0, seed=0):
    """bf16(N(0, 1) * scale) on the GPU, drawn in fp32 from a CPU generator: the same tensor on every machine."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to("cuda")


def peaked_qkv(B, H, Tq, Tk, D, scale, causal, seed):
    """float64 [B, H, T, D] q, k, v whose scaled scores peak at 100..200 for one key per query row.  The dominant key sits in the
    first key block (row % 3 == 0), at the last key (row % 3 == 1: the last block, a partial tile when Tk % 64 != 0; on causal rows
    the diagonal, the row's last visible key) or at a random key of the last block (causal: any visible key).  Every other row has a
    runner-up key within 3 of the peak, so that its gradients are not all rounding noise."""
    g = torch.Generator().manual_seed(seed)
    k = torch.randn(B, H, Tk, D, generator=g, dtype=F64)
    v = torch.randn(B, H, Tk, D, generator=g, dtype=F64)
    i = torch.arange(Tq).expand(B, H, Tq)
    r1 = torch.randint(0, 1 << 30, (B, H, Tq), generator=g)
    r2 = torch.randint(0, 1 << 30, (B, H, Tq), generator=g)
    blk = min(Tk, 64)
    if causal:
        j1 = torch.where(i % 3 == 0, torch.zeros_like(i), torch.where(i % 3 == 1, i, r1 % (i + 1)))
        j2 = r2 % (i + 1)
    else:
        j1 = torch.where(i % 3 == 0, r1 % blk, torch.where(i % 3 == 1, torch.full_like(i, Tk - 1), Tk - 1 - r1 % blk))
        j2 = r2 % Tk
    two = (i % 2 == 0) & (j2 != j1)
    peak = 100 + 100 * torch.rand(B, H, Tq, generator=g, dtype=F64)
    t1 = peak / scale
    t2 = (peak - 3 * torch.rand(B, H, Tq, generator=g, dtype=F64)) / scale
    k1 = k.gather(2, j1[..., None].expand(B, H, Tq, D))
    k2 = k.gather(2, j2[..., None].expand(B, H, Tq, D))
    g11, g12, g22 = (k1 * k1).sum(-1), (k1 * k2).sum(-1), (k2 * k2).sum(-1)
    det = torch.where(two, g11 * g22 - g12 * g12, torch.ones_like(g11))
    a = torch.where(two, (t1 * g22 - t2 * g12) / det, t1 / g11)  # q = a k1 + c k2: q.k1 = t1 (and q.k2 = t2)
    c = torch.where(two, (t2 * g11 - t1 * g12) / det, torch.zeros_like(g11))
    q = a[..., None] * k1 + c[..., None] * k2 + 0.05 * torch.randn(B, H, Tq, D, generator=g, dtype=F64)
    return q, k, v


# ---- error measures ----------------------------------------------------------------------------------------------------------------
def relerr(a, ref):
    """Relative L2 error of ``a`` against ``ref``, in float64."""
    ref = ref.to(F64)
    return ((a.to(F64) - ref).norm() / ref.norm().clamp_min(1e-300)).item()


def first_bad(bad):
    idx = torch.nonzero(bad)
    return tuple(idx[0].tolist()) if idx.numel() else None


def assert_ulp(got, ref, what, ulps=1.0, floor=1e-6, mag=None):
    """No element of ``got`` further from ``ref`` than ``ulps`` bf16 ulps taken relative to ``mag`` (2^-7 |mag| each; default
    mag = |ref|) plus ``floor`` x max|ref|, the last bits of fp32 sums that cancel.  NaN counts as too far."""
    g, r = got.to(F64), ref.to(F64)
    mag = r.abs() if mag is None else mag.to(F64)
    tol = ulps * 2.0 ** -7 * mag + floor * r.abs().max().clamp_min(1e-30)
    pos = first_bad(~((g - r).abs() <= tol))
    assert pos is None, f"{what}: element {pos} = {g[pos].item()} vs reference {r[pos].item()}"


def assert_bf16_close(got, ref, what, max_ulps=1.01):
    """``got`` (bf16 values) is bf16(ref) rounded at the same point: it differs from bf16(ref) only by rare one-ulp flips where the
    kernel's fp32 sums and the reference's differ in their last bits, and no element by more than ``max_ulps`` ulp."""
    r = ref.to(torch.bfloat16).to(F64)
    rel = relerr(got, r)
    # well inside the 1e-3 relative target of BASELINE.json for a single op
    assert rel < 3e-4, f"{what}: relative L2 error {rel}"
    significant = r.abs() > 1e-4 * r.abs().max()  # ignore -0.0 vs -1e-11 style differences
    flips = ((got.to(F64) != r) & significant).sum().item() / max(1, significant.sum().item())
    assert flips < 2e-2, f"{what}: {flips:.3e} of the significant elements are not bit-identical to bf16(reference)"
    assert_ulp(got, r, what, ulps=max_ulps, floor=1e-3)


def bf16_ulps_off(got, ref):
    """How many elements of ``got`` are more than one bf16 ulp (the spacing of bf16 at bf16(ref)) from bf16(ref); NaN counts.  Near
    zero the ulp is floored at 2^-16 of the largest |ref|: there fp32 arithmetic leaves absolute errors that mean nothing at the
    tensor's scale.  A count, to be compared with eager's on the same inputs."""
    r = ref.to(torch.bfloat16).to(F64)
    ulp = torch.exp2(torch.floor(torch.log2(r.abs().clamp_min(1e-300))) - 7)
    tol = ulp.clamp_min(2.0 ** -16 * ref.to(F64).abs().max().item())
    return int((~((got.to(F64) - r).abs() <= tol)).sum().item())


# ---- float64 references ------------------------------------------------------------------------------------------------------------
def with_grads(fn, inputs, dout, *args):
    """``fn(*inputs, *args)`` on float64 leaf copies of ``inputs``, its first output back-propagated from ``dout``:
    (the outputs, detached; the gradients of ``inputs``)."""
    leaves = [t.detach().to(F64).requires_grad_(True) for t in inputs]
    outs = fn(*leaves, *args)
    outs[0].backward(dout.to(F64))
    return tuple(o.detach() for o in outs), tuple(t.grad for t in leaves)


def attention(q, k, v, scale, causal):
    """Attention of q [B, H, Tq, D] over k / v [B, H, Tk, D]: (out [B, H, Tq, D], lse [B, H, Tq]).  ``causal`` hides key j from
    query i when j > i."""
    s = (q.to(F64) @ k.to(F64).transpose(-1, -2)) * scale
    if causal:
        s = s.masked_fill(torch.ones(s.shape[-2], s.shape[-1], dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    lse = torch.logsumexp(s, -1)
    return (s - lse[..., None]).exp() @ v.to(F64), lse


def attention_rows(q, k, v, B, H, scale, causal):
    """``attention`` on the kernels' row layout: q [B Tq, H Dh], k / v [B Tk, H Dh] (head h at columns h Dh; column views of a
    packed buffer are fine): (out [B Tq, H Dh], lse [B, H, Tq])."""
    heads = lambda t: t.reshape(B, -1, H, t.shape[1] // H).permute(0, 2, 1, 3)  # noqa: E731
    o, lse = attention(heads(q), heads(k), heads(v), scale, causal)
    return o.permute(0, 2, 1, 3).reshape(q.shape[0], -1), lse


def packed_attention(qkv, B, T, H, scale=0.125, causal=False):
    """``attention`` of packed rows qkv [B T, 3 H 64] (q | k | v): (out [B T, H 64], lse [B, H, T])."""
    D = H * 64
    return attention_rows(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], B, H, scale, causal)


BF16_U = 2.0 ** -8   # unit roundoff of bf16 (8 significant bits): |bf16(x) - x| <= 2^-8 |x|
FP32_U = 2.0 ** -24  # unit roundoff of fp32: a sum of n exact products is off by at most n 2^-24 times the sum of their magnitudes
FP32_TINY = 2.0 ** -126  # smallest normal fp32 (and bf16): flush-to-zero arithmetic rounds anything smaller to 0
ATTN_C = 2.0         # attention_bounds: tolerance = ATTN_C x the first-order error bound


def attention_bounds(q, k, v, dout, scale, causal, out):
    """Per-element error bounds for the attention kernels, on ``attention``'s layout: q / out / dout [B, H, Tq, D], k / v
    [B, H, Tk, D], ``out`` the kernel's own bf16 output, which its backward reads.  Returns ((o, lse, dq, dk, dv), (tol_o, tol_dq,
    tol_dk, tol_dv)): the float64 forward and gradients of ``attention`` at these inputs, and for each of o, dq, dk, dv a tensor
    of its shape that |kernel - float64| must not exceed at any element.

    The tolerances follow the kernels' rounding points (attention_sm90.cu): fp32 scores and softmax, P rounded to bf16 as the
    A operand of P V and P^T dO, delta = rowsum(dO o out) from the bf16 ``out``, dS = P o (dP - delta) rounded to bf16 as an
    operand, fp32 accumulation everywhere, dQ / dK scaled in fp32 at the end, every output rounded to bf16 once.  With
    u = 2^-8 (bf16), g_n = n 2^-24 (an fp32 sum of n exact bf16 x bf16 products), t = 2^-126, |X| elementwise, P the float64
    softmax and M the 0 / 1 matrix of visible keys:

    scores   S = scale Q K^T over D products, then the fp32 multiply by scale log2(e): each is off by E_ij = g_{D+2} scale (|Q||K|^T)_ij.
             Softmax moves by at most its exponent's change:  |dP_ij| <= P_ij (E_ij + Ebar_i),  Ebar_i = sum_j P_ij E_ij + 2^-24 (1 +
             |lse_i|)  (the second term: the stored fp32 lse that the backward recomputes P from).
    underflow  exp2 runs as ex2.approx.ftz: a probability below t (a score 87 or more under its row's maximum) becomes 0, as does
             any fp32 value below t, so every P_ij and dS_ij of a visible key and every stored output is also off by up to t.
    out      o = bf16(sum_j bf16(p_ij) v_j / l_i), p_ij = exp(S_ij - max_j S_ij) and l_i >= 1:
             tol_o = C [(u + 2 g_Tk) P|V| + (P o (E + Ebar)) |V| + t M|V| + u |o| + t]   (P V and l each over Tk terms).
    delta    from the kernel's out:  |d delta_i| <= sum_d |dO_id| |out_id - o_id| + g_D sum_d |dO_id| |out_id|.
    dP       = dO V^T in fp32:  |d dP_ij| <= g_D (|dO||V|^T)_ij.
    dS       = bf16(P o (dP - delta)):
             |d dS| <= u |dS| + P o (g_D |dO||V|^T + d delta) + (E + Ebar) o |dS| + t M o (|dP - delta| + 1).
    dV       = bf16(sum_i bf16(P_ij) dO_i):  tol_dv = C [(u + g_Tq) P^T|dO| + (P o (E + Ebar))^T |dO| + t M^T|dO| + u |dv| + t].
    dQ       = bf16(scale sum_j bf16(dS_ij) K_j):  tol_dq = C [scale (|d dS| |K| + g_Tk |dS||K|) + u |dq| + t];
    dK       likewise over the queries:  tol_dk = C [scale (|d dS|^T |Q| + g_Tq |dS|^T|Q|) + u |dk| + t].

    C = ATTN_C = 2 covers what the first-order bound drops: products of two error terms and the few-ulp fp32 error of the
    exp2 / log / reciprocal approximations.  Where a quantity is exact in both -- o with V = 0, every gradient with dO = 0 -- the
    tolerance falls to the underflow floor, a few t.  Masked (causal) keys have P = 0 and add nothing."""
    qd, kd, vd, dod, od = (t.to(F64) for t in (q, k, v, dout, out))
    Tq, Tk, D = qd.shape[-2], kd.shape[-2], qd.shape[-1]
    s = (qd @ kd.transpose(-1, -2)) * scale
    seen = torch.ones(Tq, Tk, dtype=F64, device=s.device)
    if causal:
        seen = seen.tril()
        s = s.masked_fill(seen == 0, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = (s - lse[..., None]).exp()
    o = p @ vd
    dp_delta = dod @ vd.transpose(-1, -2) - (dod * o).sum(-1)[..., None]
    ds = p * dp_delta
    dq, dk, dv = scale * (ds @ kd), scale * (ds.transpose(-1, -2) @ qd), p.transpose(-1, -2) @ dod

    gD, u, t = (D + 2) * FP32_U, BF16_U, FP32_TINY
    aq, ak, av, ado = qd.abs(), kd.abs(), vd.abs(), dod.abs()
    e = gD * scale * (aq @ ak.transpose(-1, -2))
    e = e + (p * e).sum(-1, keepdim=True) + FP32_U * (1 + lse.abs())[..., None]  # E + Ebar
    pe = p * e
    ddelta = (ado * (od - o).abs()).sum(-1) + gD * (ado * od.abs()).sum(-1)
    dds = u * ds.abs() + p * (gD * (ado @ av.transpose(-1, -2)) + ddelta[..., None]) + e * ds.abs() + t * seen * (dp_delta.abs() + 1)
    tol_o = ATTN_C * ((u + 2 * Tk * FP32_U) * (p @ av) + pe @ av + t * (seen @ av) + u * o.abs() + t)
    tol_dv = ATTN_C * ((u + Tq * FP32_U) * (p.transpose(-1, -2) @ ado) + pe.transpose(-1, -2) @ ado + t * (seen.transpose(-1, -2) @ ado) +
                       u * dv.abs() + t)
    tol_dq = ATTN_C * (scale * ((dds + Tk * FP32_U * ds.abs()) @ ak) + u * dq.abs() + t)
    tol_dk = ATTN_C * (scale * ((dds + Tq * FP32_U * ds.abs()).transpose(-1, -2) @ aq) + u * dk.abs() + t)
    return (o, lse, dq, dk, dv), (tol_o, tol_dq, tol_dk, tol_dv)


def attention_bounds_rows(q, k, v, dout, B, H, scale, causal, out):
    """``attention_bounds`` on the kernels' row layout (as ``attention_rows``): q / out / dout [B Tq, H Dh], k / v [B Tk, H Dh].
    Everything comes back in that layout (lse [B, H, Tq])."""
    heads = lambda t: t.reshape(B, -1, H, t.shape[1] // H).permute(0, 2, 1, 3)  # noqa: E731
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(-1, t.shape[1] * t.shape[3])  # noqa: E731
    (o, lse, dq, dk, dv), tols = attention_bounds(heads(q), heads(k), heads(v), heads(dout), scale, causal, heads(out))
    return (rows(o), lse, rows(dq), rows(dk), rows(dv)), tuple(rows(t) for t in tols)


def layernorm(x, gamma, beta, eps):
    """LayerNorm over the last dim of x [rows, dim], two-pass variance: (y, mean [rows], rstd [rows], var [rows])."""
    xd = x.to(F64)
    mean = xd.mean(-1)
    var = ((xd - mean[:, None]) ** 2).mean(-1)
    rstd = (var + eps).rsqrt()
    return (xd - mean[:, None]) * rstd[:, None] * gamma.to(F64) + beta.to(F64), mean, rstd, var


def groupnorm(x, gamma, beta, eps, silu):
    """GroupNorm(32) (+ SiLU) of channels-last x [B, HW, C], two-pass variance: (y, mean [B, 32], rstd [B, 32], var [B, 32])."""
    B, HW, C = x.shape
    xg = x.to(F64).view(B, HW, GROUPS, C // GROUPS)
    mean = xg.mean(dim=(1, 3))
    var = ((xg - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    rstd = (var + eps).rsqrt()
    z = ((xg - mean[:, None, :, None]) * rstd[:, None, :, None]).reshape(B, HW, C) * gamma.to(F64) + beta.to(F64)
    return (F.silu(z) if silu else z), mean, rstd, var


def log_softmax(x):
    """Log-softmax over the last dim; -inf logits stay -inf."""
    xd = x.to(F64)
    m = xd.max(-1, keepdim=True).values
    return xd - m - (xd - m).exp().sum(-1, keepdim=True).log()


def softmax_xent(logits, labels):
    """Softmax cross-entropy of logits [B, C] with integer labels: (loss per row [B], gradient of the mean loss [B, C])."""
    lsm = log_softmax(logits)
    rows = -lsm.gather(1, labels[:, None])[:, 0]
    return rows, (lsm.exp() - F.one_hot(labels, lsm.shape[1]).to(F64)) / lsm.shape[0]


def symmetric_xent(logits):
    """CLIP's contrastive loss (CE(L) + CE(L^T)) / 2 of square logits [B, B], targets on the diagonal: (loss, gradient [B, B])."""
    labels = torch.arange(logits.shape[0], device=logits.device)
    rows, d = softmax_xent(logits, labels)
    cols, dt = softmax_xent(logits.t(), labels)
    return 0.5 * (rows.mean() + cols.mean()), 0.5 * (d + dt.t())


def conv3x3(x, w):
    """3x3 / stride 1 / zero padding 1 convolution of channels-last x [B, H, W, Cin] with w [Cout, Cin, 3, 3]: [B H W, Cout]."""
    B, H, W, _ = x.shape
    y = F.conv2d(x.to(F64).permute(0, 3, 1, 2), w.to(F64), padding=1)
    return y.permute(0, 2, 3, 1).reshape(B * H * W, -1)


def conv3x3_wgrad(dy, x):
    """Weight gradient of ``conv3x3`` for dy [B H W, Cout]: [Cout, 9 Cin] in the kernels' packed order (tap, then channel)."""
    B, H, W, Cin = x.shape
    cols = F.unfold(x.to(F64).permute(0, 3, 1, 2), 3, padding=1)  # [B, Cin 9, HW], k = (ci, ky, kx)
    cols = cols.view(B, Cin, 9, H * W).permute(0, 3, 2, 1).reshape(B * H * W, 9 * Cin)  # k = (tap, ci)
    return dy.to(F64).t() @ cols


def conv3x3_dgrad(dy, w):
    """Input gradient of ``conv3x3`` for dy [B, H, W, Cout] and w [Cout, Cin, 3, 3]: [B H W, Cin]."""
    B, H, W, _ = dy.shape
    dx = F.conv_transpose2d(dy.to(F64).permute(0, 3, 1, 2), w.to(F64), padding=1)
    return dx.permute(0, 2, 3, 1).reshape(B * H * W, -1)


def _nchw(t):
    return t.to(F64).permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def conv3x3_s2(x, w):
    """3x3 / stride 2 / zero padding 1 convolution of channels-last x [B, H, W, Cin] with w [Cout, Cin, 3, 3]: [B, H/2, W/2, Cout]."""
    return _nhwc(F.conv2d(_nchw(x), w.to(F64), stride=2, padding=1))


def conv3x3_up2(x, w):
    """Nearest 2x upsampling of channels-last x [B, H, W, Cin], then ``conv3x3`` with w: [B, 2H, 2W, Cout]."""
    return _nhwc(F.conv2d(F.interpolate(_nchw(x), scale_factor=2, mode="nearest"), w.to(F64), padding=1))


def conv3x3_s2_dgrad(dy, w, H, W):
    """Input gradient of ``conv3x3_s2`` for dy [B, H/2, W/2, Cout] and w [Cout, Cin, 3, 3]: [B, H, W, Cin]."""
    B, Cin = dy.shape[0], w.shape[1]
    return _nhwc(torch.nn.grad.conv2d_input((B, Cin, H, W), w.to(F64), _nchw(dy), stride=2, padding=1))


def conv3x3_s2_wgrad(dy, x):
    """Weight gradient of ``conv3x3_s2`` for dy [B, H/2, W/2, Cout]: [Cout, 9 Cin] in the kernels' packed order (tap, then channel)."""
    w_shape = (dy.shape[3], x.shape[3], 3, 3)
    return torch.nn.grad.conv2d_weight(_nchw(x), w_shape, _nchw(dy), stride=2, padding=1).permute(0, 2, 3, 1).reshape(w_shape[0], -1)


def colsum_per_image(x):
    """Column sums of x [B, ..., C] per image and over all rows: (per_image [B, C], total [C])."""
    xd = x.to(F64).reshape(x.shape[0], -1, x.shape[-1])
    return xd.sum(1), xd.sum((0, 1))


# ---- exact operands for the GEMM and the 3x3 convolution ---------------------------------------------------------------------------
# bf16 operands that are small integers times a power of two per row of A and per column of B (per image and per output channel
# for the convolution): every product of one output shares the unit 2^(row exponent + column exponent).  With sum_k |a_k b_k|
# below EXACT_BUDGET units, every product and every partial sum -- in any order, in any adder of at least 23 bits that aligns or
# truncates -- is an exact multiple of that unit, so the fp32 accumulator holds the float64 value exactly and the kernels' bf16
# results are fixed to the bit.  The exponents stay inside fp32's normal range: no expected value depends on flush-to-zero.
EXACT_BUDGET = 2 ** 22
INT_BUDGET = 2 ** 20  # the random integers' share; a cancelling pair (products +-2^20) takes at most the other 2^21
CANCEL = 2 ** 10      # operand magnitude of a cancelling pair


def bf16(x):
    """bf16 of x, rounded once to fp32 first: what a kernel's fp32 value becomes when it stores bf16."""
    return x.to(torch.float32).to(torch.bfloat16)


def exact_ints(shape, K, seed):
    """Integers uniform in [-q, q], q in {1, 3, 7, 15} the largest with K q^2 <= INT_BUDGET (float64, CPU)."""
    q = max(q for q in (1, 3, 7, 15) if K * q * q <= INT_BUDGET)
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-q, q + 1, tuple(shape), generator=g).to(F64)


def exact_scaled(ints, exp):
    """bf16 ints * 2^exp (``exp`` broadcast to ``ints``), checked to be exact."""
    v = ints * torch.exp2(torch.as_tensor(exp, dtype=F64))
    out = v.to(torch.bfloat16)
    assert torch.equal(out.to(F64), v), "operand not exact in bf16"
    return out


def exponents(n, lo, hi, seed):
    """n exponents uniform in [lo, hi] (float64, CPU)."""
    return torch.randint(lo, hi + 1, (n,), generator=torch.Generator().manual_seed(seed)).to(F64)


def cancel_pairs(K, kind):
    """k positions (+, -) of the cancelling pair: inside one k16 step, across the first two 64-deep k-blocks, or at the two ends of
    the reduction (a split apart whenever there are two splits); None without cancellation."""
    if kind is None:
        return None
    k = {"k16": (K - 16, K - 13) if K >= 16 else None, "kblock": (63, 64) if K > 64 else None, "split": (0, K - 1) if K > 1 else None}[kind]
    assert k is not None, f"no {kind} cancellation at K = {K}"
    return k


def exact_operands(M, N, K, a_exp, b_exp, cancel=None, seed=0):
    """A [M, K] and B [N, K] (bf16, CPU): integers times 2^a_exp[m] per row of A and 2^b_exp[n] per row of B.  ``cancel`` = (k+, k-,
    ...): both columns of a pair in A hold 2^10, B holds +2^10 at k+ and -2^10 at k-, so every output gets products +2^20 and -2^20
    units that cancel next to the small terms.  Asserts the exactness budget (one pair fits in it)."""
    ia, ib = exact_ints((M, K), K, seed), exact_ints((N, K), K, seed + 1)
    for kp, kn in zip(cancel[::2], cancel[1::2]) if cancel is not None else ():
        ia[:, kp] = ia[:, kn] = CANCEL
        ib[:, kp], ib[:, kn] = CANCEL, -CANCEL
    worst = (ia.abs() @ ib.abs().t()).max().item()
    assert worst < EXACT_BUDGET, f"sum |a b| = {worst} units, over the 2^22 budget"
    return exact_scaled(ia, a_exp[:, None]), exact_scaled(ib, b_exp[:, None])


def exact_conv_operands(B, H, W, Cin, Cout, x_exp, w_exp, seed=0):
    """x [B, H, W, Cin] and w [Cout, Cin, 3, 3] (bf16, CPU) for ``conv3x3``: integers times 2^x_exp[b] per image and 2^w_exp[co] per
    output channel.  Asserts the exactness budget over the 9 Cin products of every output."""
    ix, iw = exact_ints((B, H, W, Cin), 9 * Cin, seed), exact_ints((Cout, Cin, 3, 3), 9 * Cin, seed + 1)
    worst = conv3x3(ix.abs(), iw.abs()).max().item()
    assert worst < EXACT_BUDGET, f"sum |x w| = {worst} units, over the 2^22 budget"
    return exact_scaled(ix, x_exp[:, None, None, None]), exact_scaled(iw, w_exp[:, None, None, None])


def exact_wgrad_operands(B, H, W, Cin, Cout, x_exp, dy_exp, seed=0):
    """x [B, H, W, Cin] and dy [B H W, Cout] (bf16, CPU) for ``conv3x3_wgrad``: integers times 2^x_exp[ci] per input channel and
    2^dy_exp[co] per output channel.  Asserts the exactness budget over the B H W products of every weight."""
    ix, idy = exact_ints((B, H, W, Cin), B * H * W, seed), exact_ints((B * H * W, Cout), B * H * W, seed + 1)
    worst = conv3x3_wgrad(idy.abs(), ix.abs()).max().item()
    assert worst < EXACT_BUDGET, f"sum |dy x| = {worst} units, over the 2^22 budget"
    return exact_scaled(ix, x_exp), exact_scaled(idy, dy_exp)


# ---- the GEMM epilogues at their rounding points ------------------------------------------------------------------------------------
GELU_ATOL = 2e-6  # the GEMM's fast erf is accurate to ~1e-7 absolute where GELU is nearly zero, per unit of the factor scaling it


def gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def splitk_ranges(K, splits):
    """[k0, k1) of each split-K plane: the 64-deep k-blocks divided as evenly as the GEMM divides them, at most one split each."""
    nkb = (K + 63) // 64
    s = min(splits, nkb)
    return [(nkb * sp // s * 64, min(K, nkb * (sp + 1) // s * 64)) for sp in range(s)]


def gemm_t(acc, bias=None):
    """t = bf16(acc + bias) as the GEMM rounds it: the fp32 sum of the fp32 accumulator and the bf16 bias, then bf16.  ``acc`` is the
    exact float64 product (which the fp32 accumulator holds exactly on exact operands)."""
    s = acc.to(F64) if bias is None else acc.to(F64) + bias.to(F64)
    return bf16(s)


def add_bf16(t, aux, clamp=False):
    """bf16(float(t) + float(aux)) in fp32 (epilogues 9, 10, 11); ``clamp`` (11): +-inf become +-bf16 max, NaN stays."""
    s = (t.float() + aux.float()).to(torch.bfloat16)
    if clamp:
        big = torch.finfo(torch.bfloat16).max
        s = torch.where(torch.isinf(s), torch.where(s > 0, big, -big).to(torch.bfloat16), s)
    return s


def gemm_epilogue(epi, t, aux=None):
    """The outputs of GEMM epilogue ``epi`` given t: bf16(acc + bias), or bf16(acc) for the backward epilogues 3, 6 and 8 (for 7, t is
    hg [M, 2F]; for 8, da [M, F]).  ``aux``: the epilogue's aux rows (10: already one row per pixel).  Returns {name: (expected, tol)}:
    tol None means bit for bit (bf16 or fp32 values); otherwise |got - expected| <= tol elementwise, float64, for the outputs that are
    transcendental functions of t.  Their ulp counts are the ones the footprint and exhaustive GELU tests allow."""
    td = t.to(F64)
    u = 2.0 ** -7

    def tol(ulps, ref, factor=1.0, mag=None):
        return ulps * u * (ref.abs() if mag is None else mag) + GELU_ATOL * (factor.abs() if torch.is_tensor(factor) else factor)

    if epi in (0, 1, 5, 7):
        out = {"out0": (t, None)}
        if epi == 1:
            ref = gelu(td)
            out["out1"] = (ref, tol(1, ref))
        elif epi == 5:  # eager's three bf16 roundings: 1.702 h, sigmoid, the product
            ref = td * bf16(torch.sigmoid(bf16(1.702 * td).to(F64))).to(F64)
            out["out1"] = (ref, tol(2, ref))
        elif epi == 7:
            Fd = t.shape[1] // 2
            h, gate = td[:, :Fd], td[:, Fd:]
            ref = h * bf16(gelu(gate)).to(F64)
            out["out1"] = (ref, tol(1, ref, h))
        return out
    if epi == 2:
        return {"out0": (aux.float() + t.float(), None)}
    if epi in (9, 10, 11):
        return {"out0": (add_bf16(t, aux, clamp=epi == 11), None)}
    h = aux.to(F64)
    if epi == 3:
        ref = td * gelu_grad(h)
        return {"out0": (ref, tol(2, ref, td))}
    if epi == 6:  # autograd of h * sigmoid(1.702 h) on bf16 tensors, one rounding per kernel; the two paths into h may cancel
        s = bf16(torch.sigmoid(bf16(1.702 * h).to(F64))).to(F64)
        gh1 = bf16(td * s).to(F64)
        gt = bf16(bf16(bf16(td * h).to(F64) * bf16(1 - s).to(F64)).to(F64) * s).to(F64)
        gh2 = bf16(1.702 * gt).to(F64)
        ref = gh1 + gh2
        return {"out0": (ref, tol(3, ref, td, gh1.abs() + gh2.abs()))}
    if epi == 8:  # dh = bf16(da g), dgate = bf16(gelu'(gate) bf16(da h)), g = bf16(gelu(gate))
        Fd = t.shape[1]
        hh, gate = h[:, :Fd], h[:, Fd:]
        dh = td * bf16(gelu(gate)).to(F64)
        dgate = gelu_grad(gate) * bf16(td * hh).to(F64)
        ref = torch.cat([dh, dgate], 1)
        return {"out0": (ref, tol(2, ref, torch.cat([td, td * hh], 1)))}
    raise ValueError(f"no reference for epilogue {epi}")


def adam(p, g, m, v, steps, lr, b1, b2, eps, wd, grad_scale=1.0, decoupled=False):
    """Adam with L2 weight decay (torch.optim.Adam's update) over the step numbers ``steps``: (params, exp_avg, exp_avg_sq).
    ``decoupled``: AdamW (torch.optim.AdamW's update), p <- p (1 - lr wd) first and no L2 term.  grad_scale multiplies only the
    gradient."""
    p, m, v = p.to(F64).clone(), m.to(F64).clone(), v.to(F64).clone()
    for t in steps:
        if decoupled:
            p = p * (1 - lr * wd)
        gg = g.to(F64) * grad_scale + (0.0 if decoupled else wd * p)
        m = b1 * m + (1 - b1) * gg
        v = b2 * v + (1 - b2) * gg * gg
        p = p - lr / (1 - b1 ** t) * m / (v.sqrt() / math.sqrt(1 - b2 ** t) + eps)
    return p, m, v


# ---- the fused FCNN step ----------------------------------------------------------------------------------------------------------------
# b200_fcnn_step (csrc/mlp.cu) runs Linear -> ReLU -> ... -> Linear in fp32, one thread per sample, every sum an FFMA chain in a fixed
# order: the forward z = fma(W_jk, a_k, ...) from z = b_j (or +0) over k; the output gradient of the multi_task[mae, mse] loss
# (w_mae sign(d) + 2 w_mse d) * inv with d = pred - y and inv = fp32(1 / (M nout)), or a given dpred; per 128-row block, each weight
# gradient fma(d_j[r], a_k[r], ...) over the block's 128 rows (rows past M carry d = 0), each bias gradient the plain sum of those d_j,
# the loss sum_j (w_mae |d| + w_mse d^2) summed over the block then times inv; each input gradient fma(d_j, W_jk, ...) over j, kept
# where the stored activation is > 0; finally b200_colsum_finish adds the block partials.
FCNN_BUDGET = 2 ** 24  # an fp32 sum of multiples of q whose magnitudes add up to less than 2^24 q is exact in any order
FCNN_C = 2.0           # fcnn_bounds: tolerance = FCNN_C x the first-order error bound


def fcnn_layers(params, dims, woff, boff):
    """[(W_l [dims[l+1], dims[l]], b_l [dims[l+1]] or None)] of the arena ``params`` (float64 views)."""
    p = params.to(F64)
    return [(p[woff[l]:woff[l] + dims[l] * dims[l + 1]].view(dims[l + 1], dims[l]),
             p[boff[l]:boff[l] + dims[l + 1]] if boff[l] >= 0 else None) for l in range(len(dims) - 1)]


def fcnn_forward(x, layers):
    """(pre-activations z_l, activations a_l) of the network: a_0 = x, a_{l+1} = relu(z_{l+1}) except the output a_L = z_L."""
    acts, pre = [x.to(F64)], []
    for l, (W, b) in enumerate(layers):
        z = acts[-1] @ W.t() + (0.0 if b is None else b) + 0.0
        pre.append(z)
        acts.append(torch.relu(z) if l + 1 < len(layers) else z)
    return pre, acts


def fcnn_step(x, params, dims, woff, boff, y=None, dpred=None, w_mae=1.0, w_mse=1.0):
    """The fused FCNN step in float64: (pred [M, nout], loss (0-dim; None with dpred), gradient arena [P]).  With ``y`` the loss is
    w_mae mean|pred - y| + w_mse mean (pred - y)^2, the mean over all M nout elements; otherwise ``dpred`` is d(pred).  torch's rules:
    the L1 gradient is sign(d), 0 at d = 0; the ReLU gradient is 0 where the activation is 0 (threshold_backward), the boundary z = 0
    included.  The arena's gaps get gradient 0.  An exact zero comes out as +0, as in the kernel, whose sums start from +0.

    The kernel's one rounding that no choice of operands removes is its fp32 inv = 1 / (M nout): it is exact only when M nout is a power
    of two, so only then can the kernel's loss and gradients of the fused loss equal these bit for bit."""
    layers = fcnn_layers(params, dims, woff, boff)
    _, acts = fcnn_forward(x, layers)
    pred = acts[-1]
    loss = None
    if y is not None:
        d = pred - y.to(F64)
        n = d.numel()
        loss = (w_mae * d.abs() + w_mse * d * d).sum() / n
        g = (w_mae * torch.sign(d) + 2 * w_mse * d) / n + 0.0
    else:
        g = dpred.to(F64)
    grads = torch.zeros(params.numel(), dtype=F64, device=pred.device)
    for l in reversed(range(len(layers))):
        W, b = layers[l]
        grads[woff[l]:woff[l] + W.numel()] = (g.t() @ acts[l]).reshape(-1) + 0.0
        if b is not None:
            grads[boff[l]:boff[l] + b.numel()] = g.sum(0) + 0.0
        if l > 0:
            g = torch.where(acts[l] > 0, g @ W, torch.zeros_like(acts[l])) + 0.0
    return pred, loss, grads


def fcnn_bounds(x, params, dims, woff, boff, y=None, dpred=None, w_mae=1.0, w_mse=1.0):
    """(pred, loss, grads) of ``fcnn_step`` and, for each, a tolerance of its shape that |kernel - float64| must not exceed anywhere.

    First-order propagation of the kernel's fp32 roundings, with u = 2^-24, g_n = n u for a fixed-order sum of n terms (an FFMA chain
    rounds once per term), |X| elementwise and B = ceil(blocks / 8) + 8 the adds of b200_colsum_finish:
    forward   dz_{l+1} = g_{in} (|b| + |a_l| |W|^T) + da_l |W|^T;  da_{l+1} = dz_{l+1} (ReLU does not expand an error); tol_pred = C dz_L.
    residual  dd = dz_L + u |d|.
    dpred     dg = 0.  Fused loss: dg = [2 w_mse dd + 4 u (w_mae + 2 w_mse |d|)] / n (the product 2 w_mse d, the add, the product with
              inv and inv's own rounding), plus 2 w_mae / n where |d| <= dd: there sign(d) may flip.
    loss      tol = C [sum (w_mae + 2 w_mse |d|) dd + (3 u + g_{nout + 9 + B}) sum (w_mae |d| + w_mse d^2)] / n: each term's two products
              and add, then the thread's sum over nout, the 32-lane tree (5), the four warps (2), the product with inv and its error (2).
    weights   tol = C [g_{128 + B} |D|^T |a_l| + dD^T |a_l| + |D|^T da_l], D the layer's output gradient; biases C [g_{128 + B} sum |D| +
              sum dD].
    inputs    t = D W: dt = g_out |D| |W| + dD |W|; kept where a_l > 0, and where |z_l| <= dz_l the kernel may mask otherwise: there
              the error may be |t| + dt.
    C = FCNN_C = 2 covers the products of two error terms the first order drops."""
    u, C = FP32_U, FCNN_C
    layers = fcnn_layers(params, dims, woff, boff)
    pre, acts = fcnn_forward(x, layers)
    pred = acts[-1]
    M, nout = pred.shape
    blocks = -(-M // 128)
    B = -(-blocks // 8) + 8
    da, dzs = torch.zeros_like(acts[0]), []
    for l, (W, b) in enumerate(layers):
        mag = acts[l].abs() @ W.abs().t() + (0.0 if b is None else b.abs())
        da = dims[l] * u * mag + da @ W.abs().t()
        dzs.append(da)
    loss = tol_loss = None
    if y is not None:
        d = pred - y.to(F64)
        n = d.numel()
        dd = da + u * d.abs()
        terms = w_mae * d.abs() + w_mse * d * d
        loss = terms.sum() / n
        tol_loss = C * (((w_mae + 2 * w_mse * d.abs()) * dd).sum() + (3 * u + (nout + 9 + B) * u) * terms.sum()) / n
        g = (w_mae * torch.sign(d) + 2 * w_mse * d) / n + 0.0
        dg = (2 * w_mse * dd + 4 * u * (w_mae + 2 * w_mse * d.abs())) / n + (2 * w_mae / n) * (d.abs() <= dd)
    else:
        g = dpred.to(F64)
        dg = torch.zeros_like(g)
    grads = torch.zeros(params.numel(), dtype=F64, device=pred.device)
    tol = torch.zeros_like(grads)
    dacts = [torch.zeros_like(acts[0])] + dzs  # the error of each activation
    for l in reversed(range(len(layers))):
        W, b = layers[l]
        a, ag = acts[l], acts[l].abs()
        grads[woff[l]:woff[l] + W.numel()] = (g.t() @ a).reshape(-1) + 0.0
        tol[woff[l]:woff[l] + W.numel()] = C * ((128 + B) * u * (g.abs().t() @ ag) + dg.t() @ ag + g.abs().t() @ dacts[l]).reshape(-1)
        if b is not None:
            grads[boff[l]:boff[l] + b.numel()] = g.sum(0) + 0.0
            tol[boff[l]:boff[l] + b.numel()] = C * ((128 + B) * u * g.abs().sum(0) + dg.sum(0))
        if l > 0:
            t = g @ W
            dt = dims[l + 1] * u * (g.abs() @ W.abs()) + dg @ W.abs()
            live, unsure = a > 0, pre[l - 1].abs() <= dacts[l]
            g = torch.where(live, t, torch.zeros_like(t)) + 0.0
            dg = torch.where(live, dt, torch.zeros_like(dt)) + torch.where(unsure, t.abs() + dt, torch.zeros_like(dt))
    return (pred, loss, grads), (C * dzs[-1], tol_loss, tol)


def _quantum(v):
    """The largest power of two that divides the dyadic float v (> 0)."""
    q = 2.0 ** math.floor(math.log2(abs(v)))
    while v / q != round(v / q):
        q /= 2
    return q


FCNN_FANS = (64.0, 16.0, 8.0, 4.0, 2.0, 1.0)  # exact_fcnn_operands tries the densest weights first


def exact_fcnn_operands(dims, M, bias, seed, *, y=False, w_mae=1.0, w_mse=1.0, fan=None, gaps=True, arena_len=None, layout=None):
    """fp32 operands of the fused FCNN step on which every product and partial sum of the kernel is exact, so that its pred, loss
    and gradients equal ``fcnn_step``'s bit for bit.  ``bias``: one bool per layer.  Returns a dict: x [M, dims[0]], y or dpred
    [M, nout], params (the arena, NaN in every gap), woff, boff, and the planted zeros: relu_zeros [(layer, row, unit)] whose ReLU
    input is exactly 0, residual_zeros [(row, unit)] where pred - y is exactly 0.

    Values are small integers times a power of two: x in [-3, 3] 2^ex; W_l in {-1, 0, 1} (one nonzero in 16 is +-3; hidden layers
    three quarters positive, or all where a unit has one input, so that units stay alive) times 2^e_l, each weight nonzero with probability fan / min(in, out), so that
    activation l is a multiple of q_l = 2^(ex + e_0 + ... + e_{l-1}); b_l in [-2, 4] q_{l+1} (the output layer's in [-4, 4]); dpred
    in [-3, 3] 2^ed; y = pred + {-2, -1, 1, 2} q_L.  Exponents differ per layer, so a value taken from the wrong layer is off by a power
    of two.  Planted zeros: in hidden layers with a bias, the bias of every unit j = 1 mod 3 is minus its pre-activation on one row
    (a ReLU input of exactly 0); in hidden layers without one, one unit's weights are all 0; residuals 2, 7, 12, ... (row-major) are
    exactly 0.

    Asserts that every intermediate stays under FCNN_BUDGET units of its quantum, measured on the network run on absolute values:
    forward sums, y and the residuals, the loss terms summed over all rows, the output gradient, every weight and bias gradient
    summed over all M rows (which bounds each 128-row block and the sum of the blocks), and every input gradient.  Without ``fan``
    the densest of FCNN_FANS that keeps the budget is taken.  ``y=True`` (the fused loss) needs M nout a power of two: the kernel's
    fp32 1 / (M nout) is exact only then.  ``layout`` = (woff, boff, P) places the tensors as given; otherwise they go in a shuffled
    order with gaps of 0..5 floats (``gaps``), the arena padded to ``arena_len``."""
    if fan is None:
        for f in FCNN_FANS[:-1]:
            try:
                return exact_fcnn_operands(dims, M, bias, seed, y=y, w_mae=w_mae, w_mse=w_mse, fan=f, gaps=gaps, arena_len=arena_len,
                                           layout=layout)
            except AssertionError as err:
                if "budget" not in str(err):
                    raise
        fan = FCNN_FANS[-1]
    L, nout = len(dims) - 1, dims[-1]
    n = M * nout
    assert not y or n & (n - 1) == 0, f"the fused loss is exact only for M nout a power of two, not {n}"
    g = torch.Generator().manual_seed(seed)
    ri = lambda lo, hi, shape=(): torch.randint(lo, hi + 1, shape, generator=g).to(F64)  # noqa: E731
    ex, ed = int(ri(-3, 3)), int(ri(-3, 3))
    cum = [ex]  # log2 of each activation's quantum: steps of -2..2, kept within [-4, 4]
    for _ in range(L):
        cum.append(min(4, max(-4, cum[-1] + int(ri(-2, 2)))))
    es = [c1 - c0 for c0, c1 in zip(cum, cum[1:])]
    qs = [2.0 ** c for c in cum]
    x = ri(-3, 3, (M, dims[0])) * qs[0]
    Ws, bs, relu_zeros, a = [], [], [], x
    for l in range(L):
        n_in, n_out, hidden = dims[l], dims[l + 1], l + 1 < L
        u = lambda: torch.rand(n_out, n_in, generator=g, dtype=F64)  # noqa: E731
        sign = torch.where(u() < (0.5 if not hidden else 0.25 if n_in > 1 else 0.0), -1.0, 1.0)
        mag = torch.where(u() < 1 / 16, 3.0, 1.0)
        wi = torch.where(u() < fan / min(n_in, n_out), sign * mag, 0.0).to(F64)
        if hidden and not bias[l] and n_out > 1:
            j = int(ri(0, n_out - 1))
            wi[j] = 0.0
            relu_zeros += [(l, r, j) for r in range(M)]
        W = wi * 2.0 ** es[l]
        z = a @ W.t() + 0.0
        b = None
        if bias[l]:
            b = ri(-2 if hidden else -4, 4, (n_out,)) * qs[l + 1]
            if hidden:
                for j in range(1, n_out, 3):
                    r = int(ri(0, M - 1))
                    b[j] = -z[r, j] + 0.0
                    relu_zeros.append((l, r, j))
            z = z + b + 0.0
        Ws.append(W)
        bs.append(b)
        a = torch.relu(z) if hidden else z
    pred, residual_zeros = a, []
    if y:
        di = ri(1, 2, (M, nout)) * torch.where(torch.rand(M, nout, generator=g) < 0.5, -1.0, 1.0).to(F64)
        di.view(-1)[2::5] = 0.0
        residual_zeros = [divmod(i, nout) for i in range(2, n, 5)]
        target = pred + di * qs[L] + 0.0
    else:
        target = ri(-3, 3, (M, nout)) * 2.0 ** ed

    def check(units, what):
        worst = units.max().item()
        assert worst < FCNN_BUDGET, f"{what}: {worst:.0f} units, over the 2^24 budget"

    A = [x.abs()]
    for l in range(L):
        A.append(A[l] @ Ws[l].abs().t() + (0.0 if bs[l] is None else bs[l].abs()))
        check(A[l + 1] / qs[l + 1], f"layer {l} forward sum")
    if y:
        d = pred - target
        check(target.abs() / qs[L], "y")
        check(d.abs() / qs[L], "residual")
        qt = min([_quantum(w) * q for w, q in ((w_mae, qs[L]), (w_mse, qs[L] ** 2)) if w != 0] or [1.0])
        check((w_mae * d.abs() + w_mse * d * d).sum() / qt, "loss sum")
        D = ((w_mae * torch.sign(d) + 2 * w_mse * d) / n).abs()
        G = min([_quantum(w) * q for w, q in ((w_mae, 1.0), (w_mse, 2 * qs[L])) if w != 0] or [1.0]) / n
    else:
        D, G = target.abs(), 2.0 ** ed
    check(D / G, "output gradient")
    for l in reversed(range(L)):
        check((D.t() @ A[l]) / (G * qs[l]), f"layer {l} weight gradient")
        check(D.sum(0) / G, f"layer {l} bias gradient")
        if l > 0:
            D, G = D @ Ws[l].abs(), G * 2.0 ** es[l]
            check(D / G, f"layer {l} input gradient")
    assert min(qs + [G]) >= 2.0 ** -100, "a quantum near fp32's subnormal range"

    names = [("w", l) for l in range(L)] + [("b", l) for l in range(L) if bias[l]]
    if layout is not None:
        woff, boff, P = list(layout[0]), list(layout[1]), layout[2]
    else:
        if gaps:
            names = [names[i] for i in torch.randperm(len(names), generator=g).tolist()]
        woff, boff, cur = [0] * L, [-1] * L, 0
        for kind, l in names:
            cur += int(ri(0, 5)) if gaps else 0
            (woff if kind == "w" else boff)[l] = cur
            cur += dims[l] * dims[l + 1] if kind == "w" else dims[l + 1]
        P = cur + (int(ri(1, 3)) if gaps else 0)
        if arena_len is not None:
            assert arena_len >= P, f"the network needs {P} floats, more than arena_len {arena_len}"
            P = arena_len
    params = torch.full((P,), float("nan"), dtype=F64)
    for l in range(L):
        params[woff[l]:woff[l] + Ws[l].numel()] = Ws[l].reshape(-1)
        if bs[l] is not None:
            params[boff[l]:boff[l] + dims[l + 1]] = bs[l]
    out = dict(x=x.float(), params=params.float(), woff=woff, boff=boff, relu_zeros=relu_zeros, residual_zeros=residual_zeros)
    out["y" if y else "dpred"] = target.float()
    for name in ("x", "params", "y" if y else "dpred"):
        v, t = out[name].double(), {"x": x, "params": params}.get(name, target)
        assert torch.equal(v[~t.isnan()], t[~t.isnan()]), f"{name} not exact in fp32"
    return out
