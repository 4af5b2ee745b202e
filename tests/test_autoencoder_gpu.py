"""The KL autoencoder's decoder on native kernels (carefree-learn_b200/autoencoder.py) and what it added to the kernels.  Every test
needs an H100 (pytest -m gpu).

  1. 3x3 and fused upsampling convolutions on rows 256 and 512 pixels wide: bit for bit on exactly representable inputs, and on
     random inputs within their rounding bound of float64 while writing exactly their outputs;
  2. GroupNorm at the decoder's largest activation (B 8, 512 x 512 pixels, 256 channels) against float64;
  3. the row softmax, and the single-head attention op at C 128 / 512 and T 1,024 / 4,096, within a bound derived from their
     bf16 rounding points;
  4. the decoder against the float64 oracle and eager bf16 autocast of it (tiny config; f8 at 256 and 512 px);
  5. determinism, layouts and dtypes of the latent, and no parameter or autograd state touched."""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import B200Error, ops  # noqa: E402
from cflearn_b200.autoencoder import AttentionAutoEncoderKLB200, spatial_attention  # noqa: E402
from _refs import (assert_bf16_close, assert_ulp, bf16, conv3x3, conv3x3_up2, exact_conv_operands, exponents, first_bad,  # noqa: E402
                   groupnorm, relerr)
from test_kernel_footprint_gpu import Case, S, assert_equal, call, covers, rand  # noqa: E402
import ae_oracle as ao  # noqa: E402

DEV = "cuda"
F64 = torch.float64
U = 2.0 ** -8  # one bf16 rounding: relative error at most 2^-8 (8 significant bits)


# ---- 1. wide rows -------------------------------------------------------------------------------------------------------------------
def _conv(up, x, wp, epi=0, aux=None):
    f = ops.conv3x3_up2 if up else ops.conv3x3
    return f(x, wp, epilogue=epi, aux=aux)


@pytest.mark.gpu
@pytest.mark.parametrize("up", [False, True], ids=["conv3x3", "up2"])
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 3, 256, 128, 72), (1, 2, 512, 64, 264), (3, 1, 256, 64, 8)])
def test_wide_rows_exact(up, B, H, W, Cin, Cout):
    """Integers times per-image and per-channel powers of 2: every fp32 sum is exact, so the output is bf16 of the float64 result."""
    seed = B * H * W + Cin + Cout + up
    x, w = exact_conv_operands(B, H, W, Cin, Cout, exponents(B, -10, 10, seed), exponents(Cout, -10, 10, seed + 1), seed)
    out = _conv(up, x.to(DEV), ops.pack_conv3x3_weight(w).to(DEV))
    ref = (conv3x3_up2(x.to(DEV), w.to(DEV)) if up else conv3x3(x.to(DEV), w.to(DEV))).reshape(-1, Cout)
    assert_equal(out.reshape(-1, Cout).cpu(), bf16(ref).cpu(), f"{'up2' if up else 'conv3x3'} {B}x{H}x{W}x{Cin}->{Cout}")


@pytest.mark.gpu
@pytest.mark.parametrize("epi", [0, 10])
@pytest.mark.parametrize("up", [False, True], ids=["conv3x3", "up2"])
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 2, 256, 64, 200), (1, 2, 512, 128, 72)])
def test_wide_rows_footprint(up, epi, B, H, W, Cin, Cout):
    """Random inputs behind NaN guards (the halo must come from the TMA zero fill): every output element written once, nothing
    else, the same bits twice, and each value within its rounding bound of float64."""
    x = rand((B, H, W, Cin), 21)
    w = rand((Cout, Cin, 3, 3), 22, 0.7 / math.sqrt(9 * Cin))
    bias = rand((Cout,), 23, 0.1)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    Ho, Wo = (2 * H, 2 * W) if up else (H, W)
    M, ldo = B * Ho * Wo, Cout + 8
    name = "b200_conv3x3_up2_nhwc_bf16" if up else "b200_conv3x3_nhwc_bf16"
    c = Case(f"{name} epi {epi} {B}x{H}x{W}x{Cin}->{Cout}")
    gx, gw, gb = c.input("x", x.reshape(1, -1)), c.input("w", wp), c.input("bias", bias)
    aux_v = rand((B, Cout), 24) if epi == 10 else None
    aux = c.input("aux", aux_v, ldo) if epi == 10 else None
    out = c.output("out0", M, Cout, ldo, torch.bfloat16, back_rows=128)
    r = c.run(lambda: call(name, gx.ptr(), gw.ptr(), gb.ptr(), out.ptr(), aux.ptr() if aux else None, ldo, B, H, W, Cin, Cout, epi, S()))
    acc = (conv3x3_up2(x, w).reshape(M, Cout) if up else conv3x3(x, w)) + bias.double()
    if epi == 0:
        assert_ulp(r["out0"], acc, c.name)
    else:
        # bf16(acc) may round the other way from the float64 sum (one ulp of acc, 2^-7 |acc|), then the sum rounds (half an ulp,
        # 2^-8 |sum|): 1.5 ulps of |bf16(acc)| + |aux|, which also covers the sums where the two cancel
        term, per_pixel = bf16(acc).double(), aux_v.double().repeat_interleave(Ho * Wo, 0)
        assert_ulp(r["out0"], term + per_pixel, c.name, ulps=1.5, floor=1e-6, mag=term.abs() + per_pixel.abs())


# ---- 2. GroupNorm at the decoder's largest activation ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_at_512px_batch_8(silu):
    """B 8 x 262,144 pixels x 256 channels (2^29 elements): the statistics of every image and the output of the last one (the
    largest offsets) against float64."""
    B, HW, C = 8, 512 * 512, 256
    g = torch.Generator(device=DEV).manual_seed(7)
    x = (torch.randn(B, HW, C, device=DEV, generator=g) * 3 + 1).to(torch.bfloat16)
    gamma = 1 + 0.1 * torch.randn(C, device=DEV, generator=g)
    beta = 0.1 * torch.randn(C, device=DEV, generator=g)
    y, mean, rstd = ops.groupnorm_silu_fwd(x, gamma, beta, 1e-6, silu=silu)
    for b in range(B):
        ref_y, ref_m, ref_r, _ = groupnorm(x[b:b + 1], gamma, beta, 1e-6, silu)
        assert torch.allclose(mean[b].double(), ref_m[0], rtol=1e-5, atol=1e-5), f"mean of image {b}"
        assert torch.allclose(rstd[b].double(), ref_r[0], rtol=1e-5), f"rstd of image {b}"
        if b == B - 1:
            assert_bf16_close(y[b], ref_y[0], f"groupnorm y of image {b}")
        del ref_y


# ---- 3. softmax and attention ----------------------------------------------------------------------------------------------------------
@covers("b200_softmax_rows_bf16")
@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols,lds,ldp", [(3, 1, 1, 8), (130, 1000, 1003, 1008), (64, 4096, 4096, 4096)])
def test_softmax_rows(rows, cols, lds, ldp):
    """Strided rows behind guards; each element within one bf16 rounding (2^-8 relative) plus the fp32 errors of the exponential's
    argument, of the exponential and of the row sum, of float64 softmax."""
    g = torch.Generator().manual_seed(rows + cols)
    s = torch.randn(rows, cols, generator=g, dtype=F64) * torch.exp2(torch.randint(-4, 7, (rows, 1), generator=g).to(F64))
    s = s.float()
    scale = 1.0 / math.sqrt(512)
    c = Case(f"softmax_rows {rows}x{cols}")
    gs = c.input("s", s, lds)
    p = c.output("p", rows, cols, ldp, torch.bfloat16)
    r = c.run(lambda: call("b200_softmax_rows_bf16", gs.ptr(), lds, p.ptr(), ldp, rows, cols, scale, S()))
    arg = scale * (s.double() - s.double().max(dim=1, keepdim=True).values)
    ref = torch.softmax(arg, dim=1)
    tol = ref * (2.0 ** -8 + 2.0 ** -22 * (1 + arg.abs()) + 2.0 ** -23 * cols) + 2.0 ** -126
    bad = first_bad(~((r["p"].double() - ref).abs() <= tol))
    assert bad is None, f"{c.name}: element {bad} = {r['p'][bad].item()} vs {ref[bad].item()}"


def _attention_params(C, seed):
    g = torch.Generator().manual_seed(seed)
    P = [1 + 0.1 * torch.randn(C, generator=g), 0.05 * torch.randn(C, generator=g)]
    for _ in range(4):
        P += [torch.randn(C, C, 1, 1, generator=g) / math.sqrt(C), 0.02 * torch.randn(C, generator=g)]
    return [t.to(DEV) for t in P]


def attention_bound(x, P):
    """float64 reference of ``spatial_attention`` on x bf16 [B, H, W, C] and a first-order bound of the kernels' error: one bf16
    rounding (U |t|) at y, q / k / v, P, O, the projection and the residual sum, propagated through the later linear maps in
    absolute values, and through the softmax as |dp_j| <= p_j (e_j + sum_i p_i e_i)."""
    gw, gb, wq, bq, wk, bk, wv, bv, wo, bo = [t.to(F64) for t in P]
    B, H, W, C = x.shape
    T = H * W
    xd = x.to(F64).view(B, T, C)
    y = groupnorm(x.view(B, T, C), gw, gb, 1e-6, False)[0]
    ey = U * y.abs() + 1e-5  # (+ the fp32 statistics' last bits where y is near 0)
    proj = lambda w, b: (y @ w.view(C, C).t() + b, ey @ w.view(C, C).abs().t())  # noqa: E731
    (q, eq0), (k, ek0), (v, ev0) = proj(wq, bq), proj(wk, bk), proj(wv, bv)
    eq, ek, ev = eq0 + U * q.abs(), ek0 + U * k.abs(), ev0 + U * v.abs()
    scale = 1.0 / math.sqrt(C)
    s = scale * q @ k.transpose(1, 2)
    es = scale * (eq @ k.abs().transpose(1, 2) + q.abs() @ ek.transpose(1, 2))
    p = torch.softmax(s, dim=-1)
    ep = p * (es + (p * es).sum(-1, keepdim=True)) + U * p
    o = p @ v
    eo = ep @ v.abs() + p @ ev + U * o.abs()
    z = o @ wo.view(C, C).t() + bo
    ez = eo @ wo.view(C, C).abs().t() + U * z.abs()
    out = xd + z
    return out.view(B, H, W, C), (ez + U * out.abs()).view(B, H, W, C)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [128, 512])
@pytest.mark.parametrize("B,H,W", [(2, 32, 32), (1, 64, 64)])
def test_spatial_attention(B, H, W, C):
    P = _attention_params(C, seed=C + H)
    g = torch.Generator().manual_seed(B * H + C)
    x = (torch.randn(B, H, W, C, generator=g) * 2).to(torch.bfloat16).to(DEV)
    got = spatial_attention(x, P)
    ref, err = attention_bound(x, P)
    bad = first_bad(~((got.to(F64) - ref).abs() <= 2.0 * err + 1e-6))
    assert bad is None, f"attention B {B} T {H * W} C {C}: element {bad} = {got[bad].item()} vs {ref[bad].item()} (bound {err[bad].item()})"
    assert torch.equal(got, spatial_attention(x, P)), "not bit-identical on a rerun"


# ---- 4. the decoder ----------------------------------------------------------------------------------------------------------------
def _model(name, seed=0):
    cfg = ao.ae_config(name)
    m = AttentionAutoEncoderKLB200(cfg.pop("img_size"), cfg.pop("in_channels"), cfg.pop("out_channels"), cfg.pop("inner_channels"),
                                   cfg.pop("latent_channels"), cfg.pop("channel_multipliers"), **cfg)
    sd = ao.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=seed)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), {k: v.to(DEV) for k, v in sd.items()}


def _latent(B, E, side, seed):
    return torch.randn(B, E, side, side, generator=torch.Generator().manual_seed(seed)).to(DEV)


@pytest.fixture
def cudnn_benchmark():
    """cudnn.benchmark on for eager's convolutions (as the decode benchmark runs them), restored afterwards so that no later
    test depends on it."""
    before = torch.backends.cudnn.benchmark
    torch.backends.cudnn.benchmark = True
    yield
    torch.backends.cudnn.benchmark = before


def _eager(sd, z, no_head=False):
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        return ao.decode(sd, z.contiguous(memory_format=torch.channels_last), no_head=no_head)


def _float64(sd, z, no_head=False):
    with torch.no_grad():
        return ao.decode({k: v.double() for k, v in sd.items()}, z.double(), no_head=no_head)


def _assert_parity(ours, eager, f64, what, slack=1e-3):
    """test_unet_gpu's criterion: no further from float64 than 1.5x eager bf16's distance, and no further from eager than 2x."""
    floor = relerr(eager, f64)
    to_f64, to_eager = relerr(ours, f64), relerr(ours, eager)
    print(f"{what}: ours vs float64 {to_f64:.3e}, vs eager {to_eager:.3e}; eager vs float64 {floor:.3e}")
    assert to_f64 <= 1.5 * floor + slack, f"{what}: ours vs float64 {to_f64:.3e}, eager bf16 vs float64 {floor:.3e}"
    assert to_eager <= 2.0 * floor + slack, f"{what}: ours vs eager {to_eager:.3e}, eager bf16 vs float64 {floor:.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("B,side", [(1, 8), (2, 8), (2, 16)])
@pytest.mark.parametrize("no_head", [False, True])
def test_tiny_decoder_matches_oracle(B, side, no_head, cudnn_benchmark):
    m, sd = _model("kl_tiny")
    z = _latent(B, 4, side, seed=B + side)
    out = m.decode(ao_inputs(z, no_head))
    assert out.dtype == torch.bfloat16 and out.is_contiguous(memory_format=torch.channels_last)
    _assert_parity(out, _eager(sd, z, no_head), _float64(sd, z, no_head), f"kl_tiny B {B} {side}x{side} no_head={no_head}")


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("side", [32, 64])
def test_f8_decoder_matches_oracle(B, side, cudnn_benchmark):
    m, sd = _model("kl_f8")
    z = _latent(B, 4, side, seed=B * side)
    out = m.decode(z)
    assert tuple(out.shape) == (B, 3, 8 * side, 8 * side) and out.is_contiguous(memory_format=torch.channels_last)
    eager = _eager(sd, z)
    f64 = _float64(sd, z)
    _assert_parity(out, eager, f64, f"kl_f8 B {B} {8 * side} px")


class ao_inputs:  # noqa: N801  (the reference's DecoderInputs, duck-typed)
    def __init__(self, z, no_head=False, apply_tanh=None):
        self.z, self.no_head, self.apply_tanh = z, no_head, apply_tanh


# ---- 5. modes ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_decode_is_deterministic_and_touches_nothing():
    m, _ = _model("kl_f8")
    z = _latent(2, 4, 32, seed=3)
    before = {k: v.clone() for k, v in m.state_dict().items()}
    a = m.decode(z)
    b = m.decode(ao_inputs(z.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)))
    assert torch.equal(a, b), "fp32 NCHW and bf16 channels-last latents (the same values) decode differently"
    assert torch.equal(a, m.decode(z)), "two decodes differ"
    assert not a.requires_grad and a.grad_fn is None
    assert all(p.grad is None for p in m.parameters())
    assert all(torch.equal(before[k], v) for k, v in m.state_dict().items())
    z.requires_grad_(True)
    assert not m.decode(z).requires_grad
    with pytest.raises(B200Error, match="CPU|cuda|CUDA"):
        m.decode(z.detach().cpu())
