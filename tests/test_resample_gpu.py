"""The SD-UNet's resampling layers on native kernels (include/b200_cflearn_ext.h): the stride-2 convolution with its input and weight
gradients, the fused nearest-2x upsampling convolution, the nearest copy and its 2x2-sum backward, and ResDownsampleB200 /
ResUpsampleB200 against oracle/unet_oracle.py::_sequential.  Every test needs an H100 (pytest -m gpu).

  1. bit for bit on exactly representable operands (every product and partial sum exact in fp32), against float64;
  2. random operands against float64, rounded at the kernels' rounding points;
  3. footprint: each entry writes exactly its outputs (test_kernel_footprint_gpu's guarded buffers);
  4. the modules at the six SD-v1.5 512 px shapes against eager bf16 autocast and fp32, determinism, memory, a short chain."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import ops  # noqa: E402
from cflearn_b200.unet_blocks import ResDownsampleB200, ResUpsampleB200, ResidualBlockWithTimeEmbeddingB200  # noqa: E402
from _refs import (bf16, conv3x3_s2, conv3x3_s2_dgrad, conv3x3_s2_wgrad, conv3x3_up2, exact_ints, exact_scaled, exponents,  # noqa: E402
                   first_bad, relerr)
from test_kernel_footprint_gpu import Case, S, assert_equal, call, covers, rand  # noqa: E402

DEV = "cuda"
F64 = torch.float64
CL = torch.channels_last


def packed(w):
    """[Cout, Cin, 3, 3] -> [Cout, 9 Cin], tap-major: the kernels' weight and weight-gradient layout."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)


# float64 references on channels-last tensors (CPU)
ref_down, ref_up, ref_down_dgrad, ref_down_wgrad = conv3x3_s2, conv3x3_up2, conv3x3_s2_dgrad, conv3x3_s2_wgrad


def sum2x2_ref(x):
    """The kernel's order: (0, 0), (0, 1), (1, 0), (1, 1) in fp32 from zero, one rounding."""
    f = x.float()
    s = torch.zeros_like(f[:, ::2, ::2])
    for i in (0, 1):
        for j in (0, 1):
            s = s + f[:, i::2, j::2]
    return s.to(torch.bfloat16)


def exact_conv(B, H, W, Cin, Cout, seed):
    """x [B, H, W, Cin] (integers times 2^e per image) and w [Cout, Cin, 3, 3] (times 2^e per output channel): every output of any
    3x3 convolution of them, upsampled or strided, is an exact fp32 sum."""
    x = exact_scaled(exact_ints((B, H, W, Cin), 9 * Cin, seed), exponents(B, -6, 6, seed + 2)[:, None, None, None])
    w = exact_scaled(exact_ints((Cout, Cin, 3, 3), 9 * Cin, seed + 1), exponents(Cout, -6, 6, seed + 3)[:, None, None, None])
    return x, w


def dev(t):
    return t.to(DEV).contiguous()


# ---- geometry: each grid class of the tiles, odd batches, B = 1, M and N tile edges ---------------------------------------------
# (B, H, W, Cin, Cout): H x W is the lower-resolution side.  Down grids (H/2 x W/2): 8 x 8 (two images per tile), 16 x 16 (8 rows
# per tile), 32 x 32 (4 rows), 64 x 64 (2 rows), 1 x 128 (one row); up grids (H x W): 8 x 8, 16 x 16, 32 x 32, 4 x 32, 2 x 64.
# Cout 8 / 248 / 264 / 520: one partial N tile, just below / above one 256-column tile, past two.
DOWN = [(1, 16, 16, 64, 8), (3, 16, 16, 128, 264), (2, 32, 32, 64, 248), (1, 64, 64, 64, 72), (1, 128, 128, 64, 8),
        (5, 2, 256, 64, 16), (8, 16, 16, 64, 520)]
UP = [(1, 8, 8, 64, 8), (3, 8, 8, 128, 264), (2, 16, 16, 64, 248), (1, 32, 32, 64, 72), (3, 4, 32, 64, 16), (1, 2, 64, 64, 520)]
DOWN_WGRAD = [s for s in DOWN if s[2] // 2 <= 64 and (s[1] // 2) * (s[2] // 2) % 64 == 0]


# ---- 1. bit for bit ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("epi", [0, 10])
@pytest.mark.parametrize("B,H,W,Cin,Cout", DOWN)
def test_down_exact(B, H, W, Cin, Cout, epi):
    x, w = exact_conv(B, H, W, Cin, Cout, seed=B + H + Cout)
    expect = bf16(ref_down(x, w))
    aux = None
    if epi == 10:  # eager's bias: a second bf16 add on the rounded convolution
        aux = exact_scaled(exact_ints((B, Cout), 1, 7), exponents(B, -3, 3, 8)[:, None])
        expect = (expect.float() + aux.float()[:, None, None, :]).to(torch.bfloat16)
    out = ops.conv3x3_s2(dev(x), dev(ops.pack_conv3x3_weight(w)), epilogue=epi, aux=None if aux is None else dev(aux))
    assert_equal(out.cpu(), expect, f"conv3x3_s2 {B}x{H}x{W}x{Cin}->{Cout} epilogue {epi}")


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,Cout,Cin", DOWN)
def test_down_dgrad_exact(B, H, W, Cout, Cin):
    """dy scaled per image, w per input channel (the output channel of this call)."""
    dy = exact_scaled(exact_ints((B, H // 2, W // 2, Cout), 9 * Cout, H), exponents(B, -6, 6, 1)[:, None, None, None])
    w = exact_scaled(exact_ints((Cout, Cin, 3, 3), 9 * Cout, W), exponents(Cin, -6, 6, 2)[None, :, None, None])
    dx = ops.conv3x3_s2_dgrad(dev(dy), dev(ops.pack_conv3x3_weight_s2_dgrad(w)))
    assert_equal(dx.cpu(), bf16(ref_down_dgrad(dy, w, H, W)), f"conv3x3_s2 dgrad {B}x{H}x{W} {Cout}->{Cin}")


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,Cin,Cout", DOWN_WGRAD)
def test_down_wgrad_exact(B, H, W, Cin, Cout):
    """x scaled per input channel, dy per output channel; unrounded fp32 sums of the split-K planes."""
    K = B * (H // 2) * (W // 2)
    x = exact_scaled(exact_ints((B, H, W, Cin), K, 5), exponents(Cin, -6, 6, 6))
    dy = exact_scaled(exact_ints((B, H // 2, W // 2, Cout), K, 7), exponents(Cout, -6, 6, 8))
    got = ops.conv3x3_s2_wgrad(dev(dy), dev(x), round_bf16=False)
    assert_equal(got.cpu(), ref_down_wgrad(dy, x).float(), f"conv3x3_s2 wgrad {B}x{H}x{W}x{Cin}->{Cout}")


@pytest.mark.gpu
@pytest.mark.parametrize("epi", [0, 10])
@pytest.mark.parametrize("B,H,W,Cin,Cout", UP)
def test_up_exact(B, H, W, Cin, Cout, epi):
    x, w = exact_conv(B, H, W, Cin, Cout, seed=B + H + Cout)
    expect = bf16(ref_up(x, w))
    aux = None
    if epi == 10:
        aux = exact_scaled(exact_ints((B, Cout), 1, 7), exponents(B, -3, 3, 8)[:, None])
        expect = (expect.float() + aux.float()[:, None, None, :]).to(torch.bfloat16)
    out = ops.conv3x3_up2(dev(x), dev(ops.pack_conv3x3_weight(w)), epilogue=epi, aux=None if aux is None else dev(aux))
    assert_equal(out.cpu(), expect, f"conv3x3_up2 {B}x{H}x{W}x{Cin}->{Cout} epilogue {epi}")


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,C", [(1, 8, 8, 8), (3, 16, 16, 1280), (2, 32, 32, 640), (1, 5, 7, 24)])
def test_nearest_and_sum2x2_exact(B, H, W, C):
    x = rand((B, H, W, C), H + C)
    up = ops.upsample_nearest2x(dev(x)).cpu()
    assert torch.equal(up.view(torch.int16), x.repeat_interleave(2, 1).repeat_interleave(2, 2).view(torch.int16))
    hi = rand((B, 2 * H, 2 * W, C), H + C + 1, scale=3.0)
    assert_equal(ops.sum2x2(dev(hi)).cpu(), sum2x2_ref(hi), f"sum2x2 {B}x{H}x{W}x{C}")


# ---- 2. random operands ---------------------------------------------------------------------------------------------------------
def assert_rounded(got, ref, absref, what):
    """got is ref rounded once to bf16 from an fp32 sum: within half a bf16 ulp of ref plus the fp32 accumulation error."""
    bad = (got.double() - ref).abs() > 2.0 ** -8 * ref.abs() + 1e-5 * absref + 1e-30
    assert first_bad(bad) is None, f"{what}: element {first_bad(bad)} = {got[first_bad(bad)].item()} vs {ref[first_bad(bad)].item()}"


SD = [(8, 64, 64, 320, 320, False), (8, 32, 32, 640, 640, False), (8, 16, 16, 1280, 1280, False),
      (8, 8, 8, 1280, 1280, True), (8, 16, 16, 1280, 1280, True), (8, 32, 32, 640, 640, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(3, 16, 16, 320, 320), (2, 32, 32, 640, 200)])
def test_random_kernels(B, H, W, Cin, Cout):
    x = rand((B, H, W, Cin), 1)
    w = rand((Cout, Cin, 3, 3), 2, (9 * Cin) ** -0.5)
    what = f"{B}x{H}x{W}x{Cin}->{Cout}"
    assert_rounded(ops.conv3x3_s2(dev(x), dev(ops.pack_conv3x3_weight(w))).cpu(), ref_down(x, w), ref_down(x.abs(), w.abs()), "down " + what)
    assert_rounded(ops.conv3x3_up2(dev(x), dev(ops.pack_conv3x3_weight(w))).cpu(), ref_up(x, w), ref_up(x.abs(), w.abs()), "up " + what)
    if Cout % 64 == 0:
        dy = rand((B, H // 2, W // 2, Cout), 3)
        assert_rounded(ops.conv3x3_s2_dgrad(dev(dy), dev(ops.pack_conv3x3_weight_s2_dgrad(w))).cpu(), ref_down_dgrad(dy, w, H, W),
                       ref_down_dgrad(dy.abs(), w.abs(), H, W), "down dgrad " + what)
        got = ops.conv3x3_s2_wgrad(dev(dy), dev(x)).cpu()  # rounded to bf16, then widened
        assert torch.equal(got, got.to(torch.bfloat16).float())
        assert_rounded(got, ref_down_wgrad(dy, x), ref_down_wgrad(dy.abs(), x.abs()), "down wgrad " + what)


# ---- 3. footprint ---------------------------------------------------------------------------------------------------------------
@covers("b200_conv3x3_s2_nhwc_bf16", "b200_conv3x3_up2_nhwc_bf16")
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["b200_conv3x3_s2_nhwc_bf16", "b200_conv3x3_up2_nhwc_bf16"])
@pytest.mark.parametrize("epi", [0, 2, 10, 11])
def test_resample_conv_footprint(entry, epi):
    B, H, W, Cin, Cout = 3, 16, 16, 64, 200
    up = "up2" in entry
    Ho, Wo = (2 * H, 2 * W) if up else (H // 2, W // 2)
    M, ldo = B * Ho * Wo, Cout + 8
    x = rand((B, H, W, Cin), 11)
    w = rand((Cout, Cin, 3, 3), 12, (9 * Cin) ** -0.5)
    bias = rand((Cout,), 13, 0.1)
    c = Case(f"{entry} epilogue {epi}")
    gx, gw, gb = c.input("x", x.reshape(1, -1)), c.input("w", packed(w).contiguous()), c.input("bias", bias)
    dtype = torch.float32 if epi == 2 else torch.bfloat16
    aux_v = {2: rand((M, Cout), 14, dtype=torch.float32), 10: rand((B, Cout), 14), 11: rand((M, Cout), 14)}.get(epi)
    aux = c.input("aux", aux_v, ldo) if epi else None
    out = c.output("out0", M, Cout, ldo, dtype, back_rows=128)
    r = c.run(lambda: call(entry, gx.ptr(), gw.ptr(), gb.ptr(), out.ptr(), aux.ptr() if aux else None, ldo, B, H, W, Cin, Cout, epi, S()))
    acc = (ref_up(x, w) if up else ref_down(x, w)).reshape(M, Cout) + bias.double()
    t = bf16(acc).float()
    if epi == 10:
        aux_v = aux_v.repeat_interleave(Ho * Wo, 0)
    ref = (t if epi == 0 else (t + aux_v.float()).to(dtype)).double()
    got = r["out0"].double()
    # one fp32 accumulation apart: t may round to the neighbouring bf16 (1 ulp <= 2^-7 |t|), then the sum rounds again (half an ulp
    # <= 2^-8 (|t| + |aux|)); t and aux may cancel
    scale = t.double().abs() + (aux_v.double().abs() if epi else 0.0)
    ok = (got - ref).abs() <= 2.0 ** -6 * scale + 1e-5 * acc.abs().max()
    assert first_bad(~ok) is None, f"{c.name}: element {first_bad(~ok)}"


@covers("b200_conv3x3_s2_dgrad_nhwc_bf16")
@pytest.mark.gpu
def test_down_dgrad_footprint():
    B, H, W, Cin, Cout = 3, 16, 16, 200, 64
    dy = rand((B, H // 2, W // 2, Cout), 21)
    w = rand((Cout, Cin, 3, 3), 22, (9 * Cout) ** -0.5)
    c = Case("conv3x3_s2 dgrad")
    gdy, gw = c.input("dy", dy.reshape(1, -1)), c.input("w", ops.pack_conv3x3_weight_s2_dgrad(w))
    dx = c.output("dx", B * H * W, Cin, dtype=torch.bfloat16, back_rows=128)
    r = c.run(lambda: call("b200_conv3x3_s2_dgrad_nhwc_bf16", gdy.ptr(), gw.ptr(), dx.ptr(), B, H, W, Cin, Cout, S()))
    assert_rounded(r["dx"], ref_down_dgrad(dy, w, H, W).reshape(-1, Cin), ref_down_dgrad(dy.abs(), w.abs(), H, W).reshape(-1, Cin),
                   c.name)


@covers("b200_conv3x3_s2_wgrad_nhwc_bf16")
@pytest.mark.gpu
def test_down_wgrad_footprint():
    B, H, W, Cin, Cout = 3, 16, 16, 64, 200
    x = rand((B, H, W, Cin), 31)
    M = B * (H // 2) * (W // 2)
    dy = rand((M, Cout), 32)
    splits = 2
    c = Case("conv3x3_s2 wgrad")
    gdy, gx = c.input("dy", dy, ld=Cout + 8), c.input("x", x.reshape(1, -1))
    part = c.output("partials", splits * Cout, 9 * Cin, back_rows=128)
    r = c.run(lambda: call("b200_conv3x3_s2_wgrad_nhwc_bf16", gdy.ptr(), Cout + 8, gx.ptr(), part.ptr(), B, H, W, Cin, Cout, splits, S()))
    planes = r["partials"].double().view(splits, Cout, 9 * Cin)
    nkb = M // 64
    for sp in range(splits):
        p0, p1 = nkb * sp // splits * 64, nkb * (sp + 1) // splits * 64
        dy_sp = torch.zeros(M, Cout, dtype=F64)
        dy_sp[p0:p1] = dy.double()[p0:p1]
        dy4 = dy_sp.view(B, H // 2, W // 2, Cout)
        ref, absref = ref_down_wgrad(dy4, x), ref_down_wgrad(dy4.abs(), x.abs())
        bad = (planes[sp] - ref).abs() > 1e-5 * absref + 1e-30
        assert first_bad(bad) is None, f"{c.name}: split {sp} element {first_bad(bad)}"


@covers("b200_upsample_nearest2x_bf16", "b200_sum2x2_bf16")
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["b200_upsample_nearest2x_bf16", "b200_sum2x2_bf16"])
def test_copy_footprint(entry):
    B, H, W, C = 3, 5, 7, 24
    lo, hi = rand((B, H, W, C), 41), rand((B, 2 * H, 2 * W, C), 42)
    c = Case(entry)
    if "upsample" in entry:
        gx, out = c.input("x", lo.reshape(1, -1)), c.output("out", 1, hi.numel(), dtype=torch.bfloat16)
        expect = lo.repeat_interleave(2, 1).repeat_interleave(2, 2)
    else:
        gx, out = c.input("x", hi.reshape(1, -1)), c.output("out", 1, lo.numel(), dtype=torch.bfloat16)
        expect = sum2x2_ref(hi)
    r = c.run(lambda: call(entry, gx.ptr(), out.ptr(), B, H, W, C, S()))
    assert_equal(r["out"].view(-1), expect.reshape(-1), entry)


# ---- 4. modules -------------------------------------------------------------------------------------------------------------------
def _module(up, Cin, Cout, seed):
    import unet_oracle as uo

    m = (ResUpsampleB200 if up else ResDownsampleB200)(Cin, True, out_channels=Cout)
    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=seed)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def _oracle(sd, net, up_grad):
    """Eager bf16 autocast and fp32 runs of oracle/unet_oracle.py::_sequential on the layer's state dict."""
    import unet_oracle as uo

    refs = []
    for autocast in (True, False):
        sdg = {"0." + k: v.detach().clone().to(DEV).requires_grad_(True) for k, v in sd.items()}
        x = (net if autocast else net.float()).detach().clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            y = uo._sequential(sdg, "", x, None, None, 1)
        (y.float() * up_grad).sum().backward()
        refs.append({"out": y, "net": x.grad, **{k[2:]: v.grad for k, v in sdg.items()}})
    return refs


def _run(m, net, up_grad):
    x = net.detach().clone().requires_grad_(True)
    y = m(x)
    (y.float() * up_grad).sum().backward()
    assert y.dtype == torch.bfloat16 and y.is_contiguous(memory_format=CL)
    assert x.grad.dtype == torch.bfloat16 and x.grad.shape == x.shape
    return {"out": y, "net": x.grad, **{k: p.grad for k, p in m.named_parameters()}}


def _inputs(B, C, H, W, Cout, up, seed, fmt=CL):
    g = torch.Generator().manual_seed(seed)
    net = torch.randn(B, C, H, W, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=fmt)
    s = 2 if up else 0.5
    up_grad = torch.randn(B, Cout, int(H * s), int(W * s), generator=g).to(DEV)
    return net, up_grad


def _check(ours, eager, fp32):
    for k in ours:
        floor = relerr(eager[k], fp32[k])
        assert relerr(ours[k], fp32[k]) <= 1.5 * floor + 1e-6, (k, relerr(ours[k], fp32[k]), floor)
        assert relerr(ours[k], eager[k]) <= 2.0 * floor + 1e-6, (k, relerr(ours[k], eager[k]), floor)


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,Cin,Cout,up", SD)
def test_module_parity(B, H, W, Cin, Cout, up):
    m, sd = _module(up, Cin, Cout, seed=H + Cin + up)
    net, up_grad = _inputs(B, Cin, H, W, Cout, up, seed=H)
    ours = _run(m, net, up_grad)
    eager, fp32 = _oracle(sd, net, up_grad)
    _check(ours, eager, fp32)


@pytest.mark.gpu
@pytest.mark.parametrize("up", [False, True])
def test_memory_format_and_determinism(up):
    m, _ = _module(up, 640, 640, seed=5)
    net, up_grad = _inputs(3, 640, 16, 16, 640, up, seed=6)
    runs = []
    for x in (net, net.contiguous(), net):
        m.zero_grad(set_to_none=True)
        runs.append(_run(m, x, up_grad))
    for r in runs[1:]:
        for k in runs[0]:
            assert torch.equal(r[k], runs[0][k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("up", [False, True])
def test_node_holds_its_input(up):
    """After the forward the node keeps the input itself and the parameters, nothing derived from them."""
    m, _ = _module(up, 320, 320, seed=7)
    net, _ = _inputs(2, 320, 32, 32, 320, up, seed=8)
    x = net.detach().requires_grad_(True)
    packed_ = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: packed_.append(t) or t, lambda t: t):
        m(x)
    params = [m.conv.weight if up else m.net.weight]
    assert len(packed_) == 2
    assert packed_[0].data_ptr() == x.data_ptr() and packed_[0].shape == x.shape
    assert packed_[1] is params[0] or packed_[1].data_ptr() == params[0].data_ptr()


@pytest.mark.gpu
def test_chain_against_oracle():
    """ResBlock(320) -> Downsample -> ResBlock(320 -> 640) -> Upsample(640) at 64 x 64, B 2, against the same oracle chain."""
    import unet_oracle as uo

    B, side, tdim = 2, 64, 1280
    mods = torch.nn.Sequential(ResidualBlockWithTimeEmbeddingB200(320, norm_eps=1e-5, time_embedding_channels=tdim),
                               ResDownsampleB200(320, True),
                               ResidualBlockWithTimeEmbeddingB200(320, 640, norm_eps=1e-5, time_embedding_channels=tdim),
                               ResUpsampleB200(640, True, out_channels=640))
    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in mods.state_dict().items()], seed=9)
    mods.load_state_dict(sd, strict=True)
    mods = mods.to(DEV)
    g = torch.Generator().manual_seed(10)
    net = torch.randn(B, 320, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=CL)
    tn = torch.randn(B, tdim, generator=g).to(DEV).to(torch.bfloat16)
    up_grad = torch.randn(B, 640, side, side, generator=g).to(DEV)

    x = net.detach().clone().requires_grad_(True)
    y = x
    for i, mod in enumerate(mods):
        y = mod(y, tn) if i in (0, 2) else mod(y)
    loss = (y.float() * up_grad).sum()
    loss.backward()
    ours = {"loss": loss.detach(), "net": x.grad, **{k: p.grad for k, p in mods.named_parameters()}}
    refs = []
    for autocast in (True, False):
        sdg = {k: v.detach().clone().to(DEV).requires_grad_(True) for k, v in sd.items()}
        xr = (net if autocast else net.float()).detach().clone().requires_grad_(True)
        t = tn if autocast else tn.float()
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            yr = uo._sequential(sdg, "", xr, t, None, 1)
        lr = (yr.float() * up_grad).sum()
        lr.backward()
        refs.append({"loss": lr.detach(), "net": xr.grad, **{k: v.grad for k, v in sdg.items()}})
    eager, fp32 = refs
    assert abs(ours["loss"].item() - fp32["loss"].item()) <= 1.5 * abs(eager["loss"].item() - fp32["loss"].item()) + 1e-3 * abs(fp32["loss"].item())
    _check({k: v for k, v in ours.items() if k != "loss"}, eager, fp32)
