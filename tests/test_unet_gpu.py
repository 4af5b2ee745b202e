"""The assembled SD-v1.5 UNet on native kernels (carefree-learn_b200/unet.py) and the two kernels it adds
(include/b200_cflearn_ext.h: channel padding, the noise-prediction loss).  Every test needs an H100 (pytest -m gpu).

  1. the pad kernel bit for bit against torch's cast, and its footprint;
  2. the loss kernel: float64 on exact inputs, eager's gradient bit for bit, determinism, footprints;
  3. the padded stem and head convolutions bit for bit against unpadded float64 convolutions on exact operands;
  4. every top-level child teacher-forced on eager's own input of its stage (SD-v1.5, 64 x 64, B 2);
  5. the whole model, loss and every gradient against eager bf16 autocast and fp32 of oracle/unet_oracle.py;
  6. use_checkpoint, determinism, memory formats and latent dtypes; 7. one CUDA-graph capture of the step."""
import os
import re
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import ops  # noqa: E402
from cflearn_b200.unet import UNetDiffuserB200, head_conv, head_conv_bwd, noise_prediction_loss, stem_conv, stem_conv_bwd  # noqa: E402
from _refs import bf16, conv3x3, conv3x3_dgrad, conv3x3_wgrad, exact_ints, exact_scaled, relerr  # noqa: E402
from test_kernel_footprint_gpu import Case, S, assert_equal, call  # noqa: E402

DEV = "cuda"
F64 = torch.float64
CL = torch.channels_last
NCHW = torch.contiguous_format

# widths all multiples of 64 (the blocks refuse the 32-channel unet_tiny): start 64, multipliers (1, 2), one res block per
# level, transformers at both levels with 2 heads, context width 64; 16 x 16 latents
SMALL = dict(in_channels=4, out_channels=4, num_heads=2, context_dim=64, start_channels=64, num_res_blocks=1,
             attention_downsample_rates=(1, 2), channel_multipliers=(1, 2))


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


# ---- 1. channel padding ------------------------------------------------------------------------------------------------------------
def _pad_input(B, C, H, W, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g) * torch.exp2(torch.randint(-20, 20, (B, C, H, W), generator=g).float())
    flat = x.view(-1)
    n = min(8, flat.numel())
    # ties to even both ways, signed zero, infinities, an fp32 subnormal
    flat[:n] = torch.tensor([1 + 2 ** -8, 1 + 3 * 2 ** -8, -0.0, float("inf"), -float("inf"), 1e-40, -(1 + 2 ** -8), 3.0])[:n]
    return x.to(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("C", [4, 8, 60])
@pytest.mark.parametrize("fmt", [NCHW, CL], ids=["nchw", "channels_last"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_pad_channels_is_torchs_cast(dtype, fmt, C, B):
    x = _pad_input(B, C, 8, 16, dtype, seed=B * 100 + C).to(DEV).contiguous(memory_format=fmt)
    out = ops.pad_channels(x, 64)
    ref = torch.zeros(B, 8, 16, 64, dtype=torch.bfloat16, device=DEV)
    ref[..., :C] = x.permute(0, 2, 3, 1).to(torch.bfloat16)
    assert_equal(out.cpu(), ref.cpu(), f"pad {dtype} {fmt} C {C} B {B}")
    assert (_bits(out[..., C:]) == 0).all()  # +0, not -0


@pytest.mark.gpu
@pytest.mark.parametrize("x_f32,cl", [(1, 0), (1, 1), (0, 0), (0, 1)])
def test_pad_channels_footprint(x_f32, cl):
    B, C, H, W, Cp = 3, 5, 6, 7, 24
    x = _pad_input(B, C, H, W, torch.float32 if x_f32 else torch.bfloat16, seed=5)
    src = x.permute(0, 2, 3, 1).contiguous() if cl else x
    c = Case(f"pad_channels f32={x_f32} cl={cl}")
    gx = c.input("x", src.reshape(1, -1))
    out = c.output("out", B * H * W, Cp, dtype=torch.bfloat16)
    r = c.run(lambda: call("b200_pad_channels_bf16", gx.ptr(), x_f32, cl, out.ptr(), B, C, H, W, Cp, S()))
    ref = torch.zeros(B, H, W, Cp, dtype=torch.bfloat16)
    ref[..., :C] = x.permute(0, 2, 3, 1).to(torch.bfloat16)
    assert_equal(r["out"], ref.view(-1, Cp), c.name)


# ---- 2. the noise-prediction loss ---------------------------------------------------------------------------------------------------
def _eager_loss(pred, noise, scale=1.0):
    """DDPMStep.loss_fn at its defaults under bf16 autocast: (loss, d loss / d pred)."""
    p = pred.detach().clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = F.mse_loss(p, noise, reduction="none").mean(dim=(1, 2, 3)).mean()
    (loss * scale).backward()
    return loss.detach(), p.grad


def _ours_loss(pred, noise, scale=1.0):
    p = pred.detach().clone().requires_grad_(True)
    loss = noise_prediction_loss(p, noise)
    (loss * scale).backward()
    return loss.detach(), p.grad


def _loss_inputs(B, C, H, W, fmt, noise_dtype, seed, exact=False):
    g = torch.Generator().manual_seed(seed)
    if exact:  # small dyadic values: every difference, square and partial sum is exact in fp32
        pred = torch.randint(-15, 16, (B, C, H, W), generator=g).to(F64) * 2 ** -3
        noise = torch.randint(-15, 16, (B, C, H, W), generator=g).to(F64) * 2 ** -4
    else:
        pred, noise = torch.randn(B, C, H, W, generator=g, dtype=F64), torch.randn(B, C, H, W, generator=g, dtype=F64)
    return (pred.to(torch.bfloat16).to(DEV).contiguous(memory_format=fmt),
            noise.to(noise_dtype).to(DEV).contiguous(memory_format=fmt))


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("noise_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_loss_is_float64_on_exact_inputs(noise_dtype, B):
    pred, noise = _loss_inputs(B, 4, 16, 16, CL, noise_dtype, seed=B, exact=True)
    ref = ((pred.double() - noise.double()) ** 2).mean(dim=(1, 2, 3)).mean()
    loss = noise_prediction_loss(pred, noise)
    assert loss.item() == ref.float().item(), (loss.item(), ref.item())


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W", [(1, 8, 8), (2, 64, 64), (3, 16, 32), (8, 64, 64)])
@pytest.mark.parametrize("fmt", [NCHW, CL], ids=["nchw", "channels_last"])
@pytest.mark.parametrize("noise_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_loss_gradient_is_eagers(noise_dtype, fmt, B, H, W):
    pred, noise = _loss_inputs(B, 4, H, W, fmt, noise_dtype, seed=B * H)
    for scale in (1.0, 0.37):
        e_loss, e_grad = _eager_loss(pred, noise, scale)
        loss, grad = _ours_loss(pred, noise, scale)
        assert grad.dtype == torch.bfloat16 and grad.stride() == pred.stride()
        assert_equal(grad.cpu(), e_grad.cpu(), f"dpred B {B} {H}x{W} scale {scale}")
    # the fixed-order fp32 sum against float64: every term is positive, so the error is at most depth * u * the loss, depth = the
    # longest chain of fp32 roundings (one thread's N / 1024 terms, the 5-level warp tree, 32 warps, the image mean, the batch)
    ref = ((pred.double() - noise.double()) ** 2).mean(dim=(1, 2, 3)).mean().item()
    N = pred[0].numel()
    depth = N // 1024 + 1 + 5 + 32 + 1 + B + 1 + 3
    assert abs(loss.item() - ref) <= depth * 2.0 ** -24 * ref, (loss.item(), ref)


def _scales(B, N, g0):
    """The two candidate scales, from IEEE fp32 arithmetic on the host (numpy: a true division is a division)."""
    f = np.float32
    rec, div = f(f(g0) * (f(1) / f(B))) * (f(1) / f(N)), f(f(g0) / f(B)) / f(N)
    return torch.tensor(float(rec), dtype=torch.float32), torch.tensor(float(div), dtype=torch.float32)


def _split_orders(B, N, g0, count=32):
    """d = pred - noise values (fp32) for which the two candidate orders of the gradient's scale, fl(fl(g0 fl(1/B)) fl(1/N)) (the
    reciprocals ATen's CUDA division by a scalar multiplies by) and fl(fl(g0 / B) / N) (true division), give different bf16
    gradients.  Returns (d, the true-division order's gradients of d)."""
    g_rec, g_div = _scales(B, N, g0)
    assert g_rec != g_div, "these shapes do not separate the two orders"
    d = torch.rand(1 << 22, generator=torch.Generator().manual_seed(B * N)) * 3.5 + 0.5
    rec, div = ((2 * d) * g_rec).to(torch.bfloat16), ((2 * d) * g_div).to(torch.bfloat16)
    split = torch.nonzero(rec.view(torch.int16) != div.view(torch.int16))[:count, 0]
    assert split.numel() == count
    return d[split], div[split]


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,g0", [(3, 24, 40, 1.0), (2, 24, 40, 0.37), (1, 48, 64, 1.3)])
def test_loss_gradient_order_is_eagers(B, H, W, g0):
    """Shapes (N = 4 H W not a power of two) and values where multiplying by fp32 reciprocals and dividing give different bits:
    the kernel follows eager, and eager here is not the true-division order."""
    N = 4 * H * W
    d, div_grad = _split_orders(B, N, g0)
    pred = torch.zeros(B * N, dtype=torch.bfloat16)
    noise = torch.randn(B * N, generator=torch.Generator().manual_seed(1))
    pos = torch.arange(d.numel()) * (B * N // d.numel())
    noise[pos] = -d  # pred - noise = d exactly
    pred, noise = pred.view(B, 4, H, W).to(DEV), noise.view(B, 4, H, W).to(DEV)
    _, e_grad = _eager_loss(pred, noise, g0)
    _, grad = _ours_loss(pred, noise, g0)
    assert_equal(grad.cpu(), e_grad.cpu(), f"dpred B {B} {H}x{W} g0 {g0}")
    assert (e_grad.reshape(-1)[pos].cpu().view(torch.int16) != div_grad.view(torch.int16)).all()


@pytest.mark.gpu
def test_loss_is_deterministic():
    pred, noise = _loss_inputs(8, 4, 64, 64, CL, torch.float32, seed=3)
    a, b = _ours_loss(pred, noise), _ours_loss(pred, noise)
    assert torch.equal(_bits(a[0]), _bits(b[0])) and torch.equal(_bits(a[1]), _bits(b[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("noise_f32", [1, 0])
def test_loss_footprint(noise_f32):
    B, N = 3, 4 * 9 * 7
    pred, noise = _loss_inputs(B, 4, 9, 7, NCHW, torch.float32 if noise_f32 else torch.bfloat16, seed=7)
    pred, noise = pred.cpu().reshape(B, N), noise.cpu().reshape(B, N)
    ref64 = ((pred.double() - noise.double()) ** 2).mean(dim=1).mean()
    c = Case(f"noise_prediction_loss f32={noise_f32}")
    gp, gn = c.input("pred", pred), c.input("noise", noise)
    loss = c.output("loss", 1, 1)
    r = c.run(lambda: call("b200_noise_prediction_loss_bf16", gp.ptr(), gn.ptr(), noise_f32, loss.ptr(), None, None, B, N, S()))
    assert abs(r["loss"].item() - ref64.item()) <= 64 * 2.0 ** -24 * ref64.item()
    c = Case(f"noise_prediction_loss grad f32={noise_f32}")
    gp, gn, go = c.input("pred", pred), c.input("noise", noise), c.input("grad_out", torch.tensor([0.37]))
    dpred = c.output("dpred", B, N, dtype=torch.bfloat16)
    r = c.run(lambda: call("b200_noise_prediction_loss_bf16", gp.ptr(), gn.ptr(), noise_f32, None, dpred.ptr(), go.ptr(), B, N, S()))
    _, e_grad = _eager_loss(pred.view(B, 4, 9, 7).to(DEV), noise.view(B, 4, 9, 7).to(DEV), 0.37)
    assert_equal(r["dpred"], e_grad.cpu().reshape(B, N), c.name)


# ---- 3. the padded stem and head convolutions ---------------------------------------------------------------------------------------
def _exact(shape, exp, seed):
    return exact_scaled(exact_ints(shape, 1, seed).clamp(-1, 1), exp)  # {-1, 0, 1} 2^exp: every sum below is exact in fp32


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W", [(1, 16, 16), (3, 8, 8), (2, 64, 64)])
@pytest.mark.parametrize("fmt", [NCHW, CL], ids=["nchw", "channels_last"])
def test_stem_is_the_4_channel_convolution(B, H, W, fmt):
    C, Cout = 4, 320
    x, w = _exact((B, H, W, C), -2, 1), _exact((Cout, C, 3, 3), -3, 2)
    bias, dy = _exact((Cout,), -4, 3), _exact((B, H, W, Cout), -4, 4)
    net = x.permute(0, 3, 1, 2).to(DEV).contiguous(memory_format=fmt).float()
    out, xp, wp = stem_conv(net, w.float().to(DEV), bias.float().to(DEV))
    ref = bf16(bf16(conv3x3(x, w)).double() + bias.double()).view(B, H, W, Cout)
    assert_equal(out.cpu(), ref, "stem forward")
    dx, dw, db = stem_conv_bwd(dy.to(DEV), xp, wp, C, True)
    assert_equal(dx.contiguous().cpu(), bf16(conv3x3_dgrad(dy, w)).view(B, H, W, C), "stem input gradient")
    ref_dw = bf16(conv3x3_wgrad(dy.reshape(-1, Cout), x)).float().view(Cout, 3, 3, C).permute(0, 3, 1, 2)
    assert_equal(dw.cpu(), ref_dw.contiguous(), "stem weight gradient")
    assert_equal(db.cpu(), bf16(dy.double().reshape(-1, Cout).sum(0)).float(), "stem bias gradient")


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,C,Co", [(1, 16, 16, 64, 4), (3, 8, 8, 320, 4), (2, 64, 64, 320, 4), (2, 16, 16, 128, 8)])
def test_head_is_the_unpadded_convolution(B, H, W, C, Co):
    y, w = _exact((B, H, W, C), -2, 11), _exact((Co, C, 3, 3), -3, 12)
    bias, dout = _exact((Co,), -4, 13), _exact((B, H, W, Co), -4, 14)
    out, wp = head_conv(y.to(DEV), w.float().to(DEV), bias.float().to(DEV))
    ref = bf16(bf16(conv3x3(y, w)).double() + bias.double()).view(B, H, W, Co)
    assert_equal(out.cpu(), ref, "head forward")
    for fmt in (NCHW, CL):
        d = dout.permute(0, 3, 1, 2).to(DEV).contiguous(memory_format=fmt)
        dy, dw, db = head_conv_bwd(d, y.to(DEV), wp)
        assert_equal(dy.cpu(), bf16(conv3x3_dgrad(dout, w)).view(B, H, W, C), "head input gradient")
        ref_dw = bf16(conv3x3_wgrad(dout.reshape(-1, Co), y)).float().view(Co, 3, 3, C).permute(0, 3, 1, 2)
        assert_equal(dw.cpu(), ref_dw.contiguous(), "head weight gradient")
        assert_equal(db.cpu(), bf16(dout.double().reshape(-1, Co).sum(0)).float(), "head bias gradient")


# ---- the model and its oracle --------------------------------------------------------------------------------------------------------
def _model(cfg, seed=0, **kw):
    import unet_oracle as uo

    m = UNetDiffuserB200(cfg["in_channels"], cfg["out_channels"], use_spatial_transformer=True, num_heads=cfg["num_heads"],
                         context_dim=cfg["context_dim"], start_channels=cfg["start_channels"], num_res_blocks=cfg["num_res_blocks"],
                         attention_downsample_rates=cfg["attention_downsample_rates"],
                         channel_multipliers=cfg["channel_multipliers"], **kw)
    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=seed)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def _batch(cfg, B, side, seed, ctx_len=77, width=None):
    width = width or side
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cfg["in_channels"], side, width, generator=g)
    ts = torch.randint(0, 1000, (B,), generator=g)
    ctx = torch.randn(B, ctx_len, cfg["context_dim"], generator=g)
    noise = torch.randn(B, cfg["out_channels"], side, width, generator=g)
    return x.to(DEV), ts.to(DEV), ctx.to(DEV), noise.to(DEV)


def _ours_step(m, x, ts, ctx, noise):
    m.zero_grad(set_to_none=True)
    pred = m(x, timesteps=ts, context=ctx)
    loss = noise_prediction_loss(pred, noise)
    loss.backward()
    return {"out": pred.detach(), "loss": loss.detach(), **{k: p.grad for k, p in m.named_parameters()}}


def _oracle_step(sd, cfg, x, ts, ctx, noise, autocast):
    import unet_oracle as uo

    params = {k: v.detach().clone().to(DEV).requires_grad_(True) for k, v in sd.items()}
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        out = uo.forward(params, x, ts, ctx, cfg)
        loss = F.mse_loss(out, noise, reduction="none").mean(dim=(1, 2, 3)).mean()
    loss.backward()
    return {"out": out.detach(), "loss": loss.detach(), **{k: v.grad for k, v in params.items()}}


NEAR_CANCELLING = re.compile(r"\.blocks\.\d+\.norm[123]\.bias$")  # LayerNorm bias gradients inside the transformer blocks


def _assert_parity(ours, eager, fp32, slack=1e-3):
    """test_model_gpu's criterion on every entry: no further from fp32 than 1.5x eager bf16's distance, and no further from eager
    than 2x eager's own distance from fp32.  One named exception, reported when used: the gradients of the transformer blocks'
    LayerNorm biases (``NEAR_CANCELLING``), sums over every token of a gradient whose terms largely cancel, so that any bf16
    pipeline's error there is a large share of the value (eager bf16 itself is 0.55-2 % from fp32 on the ones beyond the
    criterion at these sizes).  Ours measures up to 2.0x eager's distance on them; they are held to 3x."""
    assert ours.keys() == eager.keys()
    worst, relaxed = [], []
    for k in eager:
        floor = relerr(eager[k], fp32[k])
        to_fp32, to_eager = relerr(ours[k], fp32[k]), relerr(ours[k], eager[k])
        worst.append((to_fp32 / max(floor, 1e-12), k))
        f_fp32, f_eager = 1.5, 2.0
        if (to_fp32 > f_fp32 * floor + slack or to_eager > f_eager * floor + slack) and NEAR_CANCELLING.search(k):
            f_fp32, f_eager = 3.0, 3.0
            relaxed.append(f"{k} ({to_fp32:.2e} vs fp32, eager {floor:.2e})")
        assert to_fp32 <= f_fp32 * floor + slack, f"{k}: ours vs fp32 {to_fp32:.3e}, eager bf16 vs fp32 {floor:.3e}"
        assert to_eager <= f_eager * floor + slack, f"{k}: ours vs eager {to_eager:.3e}, eager bf16 vs fp32 {floor:.3e}"
    print("worst (ours vs fp32) / (eager vs fp32):", max(worst), "; held to 3x:", relaxed or "none")


def _sd_cfg():
    import unet_oracle as uo

    return uo.unet_config("sd_v1_5")


# ---- 4. stage by stage, teacher-forced -----------------------------------------------------------------------------------------------
def _stage_fn(name, cfg, params):
    """Stage ``name`` of oracle/unet_oracle.py::forward as a function of (input, time_net, context)."""
    import unet_oracle as uo

    if name == "time_embedding":
        return lambda emb, t, c: F.linear(F.silu(F.linear(emb, params["time_embedding.0.weight"], params["time_embedding.0.bias"])),
                                          params["time_embedding.2.weight"], params["time_embedding.2.bias"])
    if name == "head":
        return lambda net, t, c: F.conv2d(F.silu(F.group_norm(net, 32, params["head.0.weight"], params["head.0.bias"], 1e-5)),
                                          params["head.2.weight"], params["head.2.bias"], padding=1)
    return lambda net, t, c: uo._sequential(params, name + ".", net, t, c, cfg["num_heads"])


def _stage_inputs(cfg, params, x, ts, ctx):
    """Eager bf16 autocast of oracle/unet_oracle.py::forward: [(stage name, eager's input of that stage)], eager's time_net."""
    import unet_oracle as uo

    run = lambda name, net: _stage_fn(name, cfg, params)(net, t, ctx)  # noqa: E731
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        emb = uo.timestep_embedding(ts, cfg["start_channels"], torch.float32)
        t = _stage_fn("time_embedding", cfg, params)(emb, None, None)
        stages, skips, net, i = [("time_embedding", emb)], [], x, 0
        while any(k.startswith(f"input_blocks.{i}.") for k in params):
            stages.append((f"input_blocks.{i}", net))
            net = run(f"input_blocks.{i}", net)
            skips.append(net)
            i += 1
        stages.append(("residual", net))
        net, i = run("residual", net), 0
        while any(k.startswith(f"output_blocks.{i}.") for k in params):
            net = torch.cat([net, skips.pop()], dim=1)
            stages.append((f"output_blocks.{i}", net))
            net = run(f"output_blocks.{i}", net)
            i += 1
        stages.append(("head", net))
    return stages, t


def _ours_stage(m, name, net, t, ctx):
    if name == "time_embedding":
        return m._time_mlp(net)
    if name == "input_blocks.0":
        return m._stem(net)
    if name == "head":
        return m._head(net)
    return m._run(m.get_submodule(name), net, t, ctx)


@pytest.mark.gpu
def test_every_stage_on_eagers_input():
    """SD-v1.5 at 64 x 64, B 2: each top-level child on eager's own input of its stage (with eager's time_net and context), forward
    and backward for one random upstream gradient, within DESIGN.md section 5's stage bound of 5e-3 (relative L2) of eager bf16, or
    of 2x eager bf16's own distance from fp32 on the same input where that is larger."""
    cfg = _sd_cfg()
    m, sd = _model(cfg)
    x, ts, ctx, _ = _batch(cfg, 2, 64, seed=1)
    params = {k: v.to(DEV) for k, v in sd.items()}
    stages, t_eager = _stage_inputs(cfg, params, x, ts, ctx)
    ctx_bf = ctx.to(torch.bfloat16)
    report = []
    for n, (name, inp) in enumerate(stages):
        prefix = name + "."
        up, results = None, []
        for mode in ("eager", "fp32", "ours"):
            leaf = inp.detach().clone()
            leaf = leaf.float() if mode == "fp32" else leaf
            leaf.requires_grad_(name != "time_embedding")
            if mode == "ours":
                m.zero_grad(set_to_none=True)
                y = _ours_stage(m, name, leaf, t_eager, ctx_bf)
                ps = {k: p for k, p in m.named_parameters() if k.startswith(prefix)}
            else:
                ps = {k: v.detach().clone().requires_grad_(True) for k, v in params.items() if k.startswith(prefix)}
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "eager"):
                    y = _stage_fn(name, cfg, dict(params, **ps))(leaf, t_eager if mode == "eager" else t_eager.float(), ctx)
            if up is None:
                up = torch.randn(y.shape, generator=torch.Generator().manual_seed(n)).to(DEV)
            (y.float() * up).sum().backward()
            res = {"out": y.detach(), **{k: p.grad for k, p in ps.items()}}
            if leaf.requires_grad:
                res["input"] = leaf.grad
            results.append(res)
        eager, fp32, ours = results
        for k in eager:
            err, floor = relerr(ours[k], eager[k]), relerr(eager[k], fp32[k])
            report.append((err, name, k))
            assert err <= max(5e-3, 2.0 * floor), f"{name} {k}: ours vs eager {err:.3e}, eager vs fp32 {floor:.3e}"
    print("worst stage error vs eager:", max(report))


# ---- 5. the whole model against the oracle ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W", [(1, 16, 16), (3, 16, 16), (2, 48, 64)])
def test_small_unet_matches_oracle(B, H, W):
    m, sd = _model(SMALL)
    x, ts, ctx, noise = _batch(SMALL, B, H, seed=B, ctx_len=7, width=W)
    ours = _ours_step(m, x, ts, ctx, noise)
    _assert_parity(ours, _oracle_step(sd, SMALL, x, ts, ctx, noise, True), _oracle_step(sd, SMALL, x, ts, ctx, noise, False))


@pytest.mark.gpu
def test_sd_v1_5_matches_oracle():
    cfg = _sd_cfg()
    m, sd = _model(cfg)
    x, ts, ctx, noise = _batch(cfg, 2, 64, seed=2)
    ours = {k: v.detach().cpu() for k, v in _ours_step(m, x, ts, ctx, noise).items()}
    del m
    eager = {k: v.cpu() for k, v in _oracle_step(sd, cfg, x, ts, ctx, noise, True).items()}
    fp32 = {k: v.cpu() for k, v in _oracle_step(sd, cfg, x, ts, ctx, noise, False).items()}
    _assert_parity(ours, eager, fp32)


# ---- 6. modes ----------------------------------------------------------------------------------------------------------------------
def _same(a, b):
    for k in a:
        assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), k


@pytest.mark.gpu
def test_checkpoint_is_bit_identical_and_lowers_the_peak():
    """At 64 x 64 latents, where the activations every block keeps until backward outweigh the parameters and workspaces."""
    x, ts, ctx, noise = _batch(SMALL, 2, 64, seed=4, ctx_len=7)
    peaks, results = {}, {}
    for flag in (False, True):
        m, _ = _model(SMALL, use_checkpoint=flag)
        _ours_step(m, x, ts, ctx, noise)  # warm-up: workspaces
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        results[flag] = {k: v.clone() for k, v in _ours_step(m, x, ts, ctx, noise).items()}
        torch.cuda.synchronize()
        peaks[flag] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        del m
    _same(results[True], results[False])
    print(f"small UNet B 2, 64 x 64: peak over the step {peaks[False]:.1f} MiB stored, {peaks[True]:.1f} MiB checkpointed")
    assert peaks[True] < peaks[False]


@pytest.mark.gpu
def test_runs_formats_and_dtypes_are_bit_identical():
    m, _ = _model(SMALL)
    x, ts, ctx, noise = _batch(SMALL, 3, 16, seed=5, ctx_len=7)
    x = x.to(torch.bfloat16).float()  # values a bf16 latent holds exactly
    ref = {k: v.clone() for k, v in _ours_step(m, x, ts, ctx, noise).items()}
    assert ref["out"].dtype == torch.bfloat16 and ref["out"].is_contiguous(memory_format=CL)
    for variant in (x, x.contiguous(memory_format=CL), x.to(torch.bfloat16), x.to(torch.bfloat16).contiguous(memory_format=CL)):
        _same(_ours_step(m, variant, ts, ctx, noise), ref)
    _same(_ours_step(m, x, ts.float(), ctx.to(torch.bfloat16), noise), ref)  # float timesteps, a bf16 context


@pytest.mark.gpu
def test_latent_gradient_when_asked():
    m, _ = _model(SMALL)
    x, ts, ctx, noise = _batch(SMALL, 1, 16, seed=6, ctx_len=7)
    leaf = x.clone().requires_grad_(True)
    noise_prediction_loss(m(leaf, timesteps=ts, context=ctx), noise).backward()
    assert leaf.grad is not None and leaf.grad.dtype == torch.float32 and leaf.grad.abs().sum() > 0


# ---- 7. one CUDA graph --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_graphed_step_replays_the_eager_step():
    m, _ = _model(SMALL)
    static = list(_batch(SMALL, 3, 16, seed=7, ctx_len=7))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _ours_step(m, *static)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    m.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        pred = m(static[0], timesteps=static[1], context=static[2])
        loss = noise_prediction_loss(pred, static[3])
        loss.backward()
    new = _batch(SMALL, 3, 16, seed=8, ctx_len=7)
    with torch.no_grad():
        for s, n in zip(static, new):
            s.copy_(n)
    graph.replay()
    torch.cuda.synchronize()
    got = {"out": pred.detach().clone(), "loss": loss.detach().clone(), **{k: p.grad.clone() for k, p in m.named_parameters()}}
    graph.replay()  # replays are identical too
    torch.cuda.synchronize()
    _same({"out": pred.detach(), "loss": loss.detach(), **{k: p.grad for k, p in m.named_parameters()}}, got)
    del pred, loss
    graph.reset()
    _same(_ours_step(m, *new), got)
