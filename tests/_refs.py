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


def adam(p, g, m, v, steps, lr, b1, b2, eps, wd, grad_scale=1.0):
    """Adam with L2 weight decay (torch.optim.Adam's update) over the step numbers ``steps``: (params, exp_avg, exp_avg_sq)."""
    p, m, v = p.to(F64).clone(), m.to(F64).clone(), v.to(F64).clone()
    for t in steps:
        gg = g.to(F64) * grad_scale + wd * p
        m = b1 * m + (1 - b1) * gg
        v = b2 * v + (1 - b2) * gg * gg
        p = p - lr / (1 - b1 ** t) * m / (v.sqrt() / math.sqrt(1 - b2 ** t) + eps)
    return p, m, v
