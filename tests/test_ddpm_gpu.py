"""DDPMB200 on an H100 (pytest -m gpu): the fused noising kernel bit for bit against eager's q_sample and behind guarded buffers,
the gradient arena bit for bit against the UNet's autograd gradients (stored and use_checkpoint, small and SD-v1.5), gradient
accumulation in the arena, train_step against torch noising + the UNet + the loss, ArenaAdamW in lock-step with
torch.optim.AdamW, and the graphed step against the eager one."""
import json
import os
import shutil
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: E402,F401
from cflearn_b200 import ops  # noqa: E402
from cflearn_b200.ddpm import DDPMB200, noise_tables  # noqa: E402
from cflearn_b200.optim import ArenaAdamW  # noqa: E402
from cflearn_b200.trainer import B200TrainStep  # noqa: E402
from cflearn_b200.unet import UNetDiffuserB200, enable_grad_arena, noise_prediction_loss  # noqa: E402
from test_kernel_footprint_gpu import Case, S, call, covers  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GOLDEN = os.path.join(ROOT, "tests", "golden")
SMALL = dict(in_channels=4, out_channels=4, num_heads=2, context_dim=64, start_channels=64, num_res_blocks=1,
             attention_downsample_rates=(1, 2), channel_multipliers=(1, 2))


def _sd_cfg():
    d = json.load(open(os.path.join(GOLDEN, "unet_sd_v1_5_state_dict_keys.json")))
    return {k: tuple(v) if isinstance(v, list) else v for k, v in d["config"].items()}


def _weights(m, seed):
    import unet_oracle as uo

    return uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=seed)


def _unet(cfg, **kw):
    cfg = dict(cfg)
    return UNetDiffuserB200(cfg.pop("in_channels"), cfg.pop("out_channels"), use_spatial_transformer=True, **cfg, **kw)


def _ddpm(cfg, **kw):
    cfg = dict(cfg)
    return DDPMB200(64, cfg.pop("in_channels"), cfg.pop("out_channels"), use_spatial_transformer=True, **cfg, **kw)


def _batch(cfg, B, side, seed, ctx_len=7):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cfg["in_channels"], side, side, generator=g)
    ts = torch.randint(0, 1000, (B,), generator=g)
    ctx = torch.randn(B, ctx_len, cfg["context_dim"], generator=g)
    noise = torch.randn(B, cfg["out_channels"], side, side, generator=g)
    return x.to(DEV), ts.to(DEV), ctx.to(DEV), noise.to(DEV)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


# ---- the noising kernel ---------------------------------------------------------------------------------------------------------------
def _torch_q_sample_pad(x0, noise, t, a, s, cp=64):
    w_net, w_noise = a[t].view(-1, 1, 1, 1), s[t].view(-1, 1, 1, 1)  # extract_to
    net = (w_net * x0 + w_noise * noise).to(torch.bfloat16)  # q_sample in fp32, then autocast's cast at the stem
    return torch.nn.functional.pad(net.permute(0, 2, 3, 1), (0, cp - x0.shape[1])).contiguous()


@pytest.mark.parametrize("channels_last", [False, True])
def test_q_sample_pad_is_eagers_bit_for_bit_at_every_timestep(channels_last):
    a, s = (t.to(DEV) for t in noise_tables())
    g = torch.Generator(device=DEV).manual_seed(1)
    t = torch.arange(1000, device=DEV)
    x0 = torch.randn(1000, 4, 8, 16, device=DEV, generator=g) * 3
    noise = torch.randn(1000, 4, 8, 16, device=DEV, generator=g)
    if channels_last:
        x0, noise = x0.contiguous(memory_format=torch.channels_last), noise.contiguous(memory_format=torch.channels_last)
    out, bad = ops.q_sample_pad(x0, noise, t, a, s, 64)
    want = _torch_q_sample_pad(x0, noise, t, a, s)
    assert torch.equal(_bits(out), _bits(want)) and int(bad.item()) == 0
    assert (_bits(out[..., 4:]) == 0).all()  # +0 padding


def test_q_sample_pad_bad_timestep_sets_the_flag():
    """A timestep outside [0, T) sets the flag and NaNs its image; the images around it are exact.  (The kernel tests the range
    before it loads a table entry; an out-of-range load itself is not observable here: its image is NaN either way.)"""
    a, s = (t.to(DEV) for t in noise_tables(timesteps=50))
    t = torch.tensor([0, -1, 49, 50, 7, 1 << 40], device=DEV)
    x0 = torch.randn(6, 3, 8, 8, device=DEV)
    noise = torch.randn(6, 3, 8, 8, device=DEV)
    out, bad = ops.q_sample_pad(x0, noise, t, a, s, 8)
    assert int(bad.item()) == 1
    good = torch.tensor([0, 2, 4], device=DEV)
    want = _torch_q_sample_pad(x0[good], noise[good], t[good], a, s, 8)
    assert torch.equal(_bits(out[good]), _bits(want))
    for b in (1, 3, 5):
        assert torch.isnan(out[b, ..., :3].float()).all() and (_bits(out[b, ..., 3:]) == 0).all()


# (B, C, H, W, Cp): one group of 8 channels with C = 4 and many groups; odd C, whose last pair holds one real channel
# (c + 1 < C fails); odd C across two real groups
Q_SAMPLE_SHAPES = [(2, 4, 8, 16, 64), (3, 5, 6, 7, 24), (2, 9, 3, 5, 16)]
Q_SAMPLE_T = 37


@covers("b200_q_sample_pad_bf16")
@pytest.mark.parametrize("timesteps", ["in_range", "out_of_range", "flag_already_set"])
@pytest.mark.parametrize("channels_last", [0, 1])
@pytest.mark.parametrize("B,C,H,W,Cp", Q_SAMPLE_SHAPES)
def test_q_sample_pad_footprint(B, C, H, W, Cp, channels_last, timesteps):
    """Guarded buffers (test_kernel_footprint_gpu): the tables are [T] with poison on both sides, so a read of entry -1 or T NaNs
    an image; every image with a timestep in range is eager's bit for bit.  Timesteps 0 and T - 1 are in every in-range batch;
    out of range, image 1 has T (and image 2, if any, -1).  The flag is only ever set, never cleared."""
    a, s = noise_tables(timesteps=Q_SAMPLE_T)
    g = torch.Generator().manual_seed(B * 100 + C)
    x0 = torch.randn(B, C, H, W, generator=g) * 3
    noise = torch.randn(B, C, H, W, generator=g)
    t = torch.tensor([0, Q_SAMPLE_T - 1, 17][:B])
    if timesteps == "out_of_range":
        t[1:] = torch.tensor([Q_SAMPLE_T, -1][:B - 1])
    good = (t >= 0) & (t < Q_SAMPLE_T)
    layout = (lambda v: v.permute(0, 2, 3, 1)) if channels_last else (lambda v: v)
    c = Case(f"q_sample_pad {B}x{C}x{H}x{W} Cp {Cp} cl {channels_last} {timesteps}")
    gx, gn = c.input("x0", layout(x0).reshape(1, -1)), c.input("noise", layout(noise).reshape(1, -1))
    gt, ga, gs = c.input("timesteps", t), c.input("sqrt_alphas_cumprod", a), c.input("sqrt_one_minus_alphas_cumprod", s)
    flag = c.inout("bad_flag", torch.tensor([int(timesteps == "flag_already_set")], dtype=torch.int32))
    out = c.output("out", B * H * W, Cp, dtype=torch.bfloat16)
    r = c.run(lambda: call("b200_q_sample_pad_bf16", gx.ptr(), gn.ptr(), channels_last, gt.ptr(), ga.ptr(), gs.ptr(), Q_SAMPLE_T,
                           flag.ptr(), out.ptr(), B, C, H, W, Cp, S()), nan_ok=("out",) if timesteps == "out_of_range" else ())
    assert r["bad_flag"].item() == int(timesteps != "in_range"), c.name
    got = r["out"].view(B, H, W, Cp)
    want = _torch_q_sample_pad(x0[good].to(DEV), noise[good].to(DEV), t[good].to(DEV), a.to(DEV), s.to(DEV), Cp).cpu()
    assert torch.equal(_bits(got[good]), _bits(want)), c.name
    for b in torch.nonzero(~good).flatten().tolist():
        assert torch.isnan(got[b, ..., :C].float()).all() and (_bits(got[b, ..., C:]) == 0).all(), f"{c.name}: image {b}"


# ---- the gradient arena ----------------------------------------------------------------------------------------------------------------
def _step(m, x, ts, ctx, noise):
    loss = noise_prediction_loss(m(x, timesteps=ts, context=ctx), noise)
    loss.backward()
    return loss.detach()


def _pair(cfg, use_checkpoint, seed=0):
    ref = _unet(cfg, use_checkpoint=use_checkpoint)
    sd = _weights(ref, seed)
    ref.load_state_dict(sd, strict=True)
    ref = ref.to(DEV)
    m = _unet(cfg, use_checkpoint=use_checkpoint)
    m.load_state_dict(sd, strict=True)
    arena = enable_grad_arena(m)  # on the host: the forward builds the arena on the device the module moved to
    m = m.to(DEV)
    return ref, m, arena


@pytest.mark.parametrize("cfg,B,side", [("small", 3, 16), ("sd", 1, 64)])
@pytest.mark.parametrize("use_checkpoint", [False, True])
def test_arena_gradients_are_autograds_bit_for_bit(cfg, B, side, use_checkpoint):
    cfg = SMALL if cfg == "small" else _sd_cfg()
    ref, m, arena = _pair(cfg, use_checkpoint)
    A = arena.arena
    seen = []
    # torch runs a leaf's post-accumulate hook even when its node returned no gradient for it: what the hook sees must be the
    # arena view the op's backward filled, with nothing added or allocated by autograd
    for name, p in m.named_parameters():
        p.register_post_accumulate_grad_hook(
            lambda q, name=name: seen.append((name, q.grad is not None and q.grad.data_ptr() == A.g(name).data_ptr())))
    x, ts, ctx, noise = _batch(cfg, B, side, seed=3, ctx_len=77 if cfg is not SMALL else 7)
    l_ref = _step(ref, x, ts, ctx, noise)
    l_m = _step(m, x, ts, ctx, noise)
    assert torch.equal(l_ref, l_m)
    assert sorted(k for k, _ in seen) == sorted(k for k, _ in m.named_parameters())  # every parameter's hook ran once
    assert all(ok for _, ok in seen), [k for k, ok in seen if not ok]
    assert A.grad.device == DEV
    for (k, p), (_, q) in zip(m.named_parameters(), ref.named_parameters()):
        assert p.grad.data_ptr() == A.grad.data_ptr() + 4 * A.offsets[k], k
        assert torch.equal(_bits(p.grad), _bits(q.grad)), k


def test_arena_accumulates_the_fp32_sum_of_two_backwards():
    ref, m, arena = _pair(SMALL, False, seed=1)
    b1, b2 = _batch(SMALL, 2, 16, seed=4), _batch(SMALL, 2, 16, seed=5)
    fresh = []
    for b in (b1, b2):
        ref.zero_grad(set_to_none=True)
        _step(ref, *b)
        fresh.append({k: p.grad.clone() for k, p in ref.named_parameters()})
    for b in (b1, b2):  # no zero_grad in between: the second backward adds in the arena
        _step(m, *b)
    for k, p in m.named_parameters():
        assert torch.equal(_bits(p.grad), _bits(fresh[0][k] + fresh[1][k])), k


# ---- train_step ----------------------------------------------------------------------------------------------------------------------
def test_train_step_is_torch_noising_unet_and_loss_bit_for_bit():
    torch.manual_seed(0)
    m = _ddpm(SMALL)
    sd = _weights(m, 2)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV)
    ref = _unet(SMALL)
    ref.load_state_dict({k[len("unet."):]: v for k, v in sd.items()}, strict=True)
    ref = ref.to(DEV)
    x, ts, ctx, noise = _batch(SMALL, 3, 16, seed=6)
    loss = m.train_step(x, ctx, noise, ts)
    a, s = m.sqrt_alphas_cumprod, m.sqrt_one_minus_alphas_cumprod
    xt = a[ts].view(-1, 1, 1, 1) * x + s[ts].view(-1, 1, 1, 1) * noise  # DDPMQSampler.q_sample
    l_ref = _step(ref, xt, ts, ctx, noise)
    assert torch.equal(loss, l_ref) and int(m.last_bad_flag.item()) == 0
    for (k, p), (_, q) in zip(m.unet.named_parameters(), ref.named_parameters()):
        assert torch.equal(_bits(p.grad), _bits(q.grad)), k


def test_seeded_draws_are_randint_then_randn_like():
    m = _ddpm(SMALL).to(DEV)
    x, _, ctx, _ = _batch(SMALL, 4, 16, seed=7)
    torch.manual_seed(11)
    out = m(x, ctx)
    torch.manual_seed(11)
    ts = torch.randint(0, 1000, (4,), device=DEV)
    noise = torch.randn_like(x)
    assert torch.equal(out["timesteps"], ts) and torch.equal(out["noise"], noise)
    assert out["predictions"].shape == x.shape


# ---- AdamW -----------------------------------------------------------------------------------------------------------------------------
def test_arena_adamw_follows_torch_adamw_with_clipping_and_a_schedule():
    m = _ddpm(SMALL)
    m.load_state_dict(_weights(m, 3), strict=True)
    m = m.to(DEV)
    m.arena.ensure()
    clip = 0.05
    opt = ArenaAdamW(m, lr=1e-3, capturable=True)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: (i + 1) / 4)
    named = {k: p.detach().clone().requires_grad_(True) for k, p in m.unet.named_parameters()}
    params = list(named.values())
    topt = torch.optim.AdamW(params, lr=1e-3)  # weight_decay 0.01, torch's default
    tsched = torch.optim.lr_scheduler.LambdaLR(topt, lambda i: (i + 1) / 4)
    g = torch.Generator(device=DEV).manual_seed(9)
    norms = []
    for _ in range(3):
        G = torch.randn(m.arena.total, device=DEV, generator=g) * 1e-3
        m.arena.grad.copy_(G)
        for k in named:
            named[k].grad = m.arena.g(k).clone()
        opt.sync_hyper()
        opt.clip_grad_norm_(clip)
        opt.step()
        sched.step()
        norms.append(torch.nn.utils.clip_grad_norm_(params, clip).item())
        topt.step()
        tsched.step()
        for k, p in m.unet.named_parameters():
            assert torch.allclose(p, named[k], rtol=1e-5, atol=2e-7), (k, (p - named[k]).abs().max().item())
    assert max(norms) > clip


# ---- the graphed step ------------------------------------------------------------------------------------------------------------------
def _seam(sd, graph, static=None, lr=1e-4):
    m = _ddpm(SMALL)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV)
    opt = ArenaAdamW(m, lr=lr, capturable=True)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: 1.0 / (i + 1))
    return m, B200TrainStep(m, opt, scheduler=sched, clip_norm=1.0, graph=graph, static_inputs=static)


def test_graphed_step_equals_the_eager_seam():
    sd = _weights(_ddpm(SMALL), 4)
    batches = [_batch(SMALL, 2, 16, seed=10 + i) for i in range(3)]
    static = [torch.zeros_like(t) for t in (batches[0][0], batches[0][2], batches[0][3], batches[0][1])]
    m_e, s_e = _seam(sd, False)
    m_g, s_g = _seam(sd, True, static)
    for x, ts, ctx, noise in batches:
        l_e = s_e.step(x, ctx, noise, ts)
        l_g = s_g.step(x, ctx, noise, ts)
        assert torch.equal(l_e, l_g)
    for (k, p), (_, q) in zip(m_e.named_parameters(), m_g.named_parameters()):
        assert torch.equal(_bits(p), _bits(q)), k
    s_g.close()


def test_graph_replays_draw_fresh_noise():
    sd = _weights(_ddpm(SMALL), 5)
    x, _, ctx, _ = _batch(SMALL, 2, 16, seed=20)
    m, step = _seam(sd, True, [torch.zeros_like(x), torch.zeros_like(ctx)], lr=0.0)
    losses = [step.step(x, ctx).clone() for _ in range(3)]
    assert len({float(v) for v in losses}) == 3  # same latent, same weights (lr 0): only the draws differ
    step.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_unet_dp_check_world2():
    torchrun = shutil.which("torchrun")
    cmd = ([torchrun] if torchrun else [sys.executable, "-m", "torch.distributed.run"]) + [
        "--nproc-per-node", "2", os.path.join(ROOT, "tools", "unet_dp_check.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
