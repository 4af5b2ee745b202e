"""DDIM sampling on an H100 (pytest -m gpu): b200_ddim_step_bf16 bit for bit against the oracle's step in torch ops on CUDA at
every step of a 50-step schedule, guided and not, on inputs with signed zeros, large magnitudes and bf16 ties, its out-of-range
counter, and its footprint behind guarded buffers; DDPMB200.decode bit for bit against oracle/ddim_oracle.py's loop driving the
same native UNet, across the golden fixture's case matrix and at SD-v1.5, including the generator state after the call; the
graph cache; and a graphed training step unchanged by sampling between its steps."""
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: E402,F401
from cflearn_b200 import ops  # noqa: E402
from cflearn_b200.ddim import step_tables  # noqa: E402
from cflearn_b200.ddpm import DDPMB200, alphas_cumprod_table  # noqa: E402
from cflearn_b200.optim import ArenaAdamW  # noqa: E402
from cflearn_b200.trainer import B200TrainStep  # noqa: E402
import ddim_oracle  # noqa: E402
from test_kernel_footprint_gpu import Case, S as current_stream, call, covers, rand  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GOLDEN = os.path.join(ROOT, "tests", "golden")
SMALL = dict(in_channels=4, out_channels=4, num_heads=2, context_dim=64, start_channels=64, num_res_blocks=1,
             attention_downsample_rates=(1, 2), channel_multipliers=(1, 2))
CASES = torch.load(os.path.join(GOLDEN, "ddim_reference.pt"))["cases"]
SCHEDULES = {1000: dict(linear_start=1e-4, linear_end=2e-2), 37: dict(linear_start=8.5e-4, linear_end=1.2e-2)}
NAMES = ("s1m", "sqrt_a", "sqrt_ap", "c_dir", "sigma")


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _weights(m, seed):
    import unet_oracle as uo

    return uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=seed)


def _ddpm(cfg, side=64, **kw):
    cfg = dict(cfg)
    return DDPMB200(side, cfg.pop("in_channels"), cfg.pop("out_channels"), use_spatial_transformer=True, **cfg, **kw)


# ---- the step kernel -----------------------------------------------------------------------------------------------------------------------
def _step_inputs(B, C, H, W, guided, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, C, H, W, device=DEV, generator=g)
    noise = torch.randn(B, C, H, W, device=DEV, generator=g)
    ec = torch.randn(B, H, W, C, device=DEV, generator=g)
    eu = torch.randn(B, H, W, C, device=DEV, generator=g)
    # bf16 ties: ec in [1, 2) and eu in [0.5, 1) on bf16 grids, so that half of the differences sit halfway between bf16 values
    n = ec.numel() // 4
    ec.view(-1)[:n] = 1.0 + torch.randint(0, 128, (n,), device=DEV, generator=g).float() / 128
    eu.view(-1)[:n] = 0.5 + torch.randint(0, 128, (n,), device=DEV, generator=g).float() / 256
    # signed zeros and large magnitudes
    x.view(-1)[n:n + 64] = -0.0
    x.view(-1)[n + 64:n + 128] = 0.0
    ec.view(-1)[n:n + 32] = -0.0
    eu.view(-1)[n + 16:n + 48] = 0.0
    x.view(-1)[n + 128:n + 256] *= 1e30
    ec.view(-1)[n + 256:n + 384] *= 1e30
    noise.view(-1)[n + 384:n + 512] *= 1e20
    ec, eu = (t.to(torch.bfloat16).permute(0, 3, 1, 2) for t in (ec, eu))  # dense channels-last [B, C, H, W]
    return x, noise, ec, (eu if guided else None)


def _oracle_step(x, noise, ec, eu, scale, coef_row, temperature):
    e = ec if eu is None or scale == 1.0 else eu + scale * (ec - eu)  # _uncond_denoise's last line, bf16 tensor ops
    B = x.shape[0]
    c = {name: torch.full((B, 1, 1, 1), float(coef_row[j]), dtype=torch.float32, device=DEV) for j, name in enumerate(NAMES)}
    return ddim_oracle.update(x, e, c, noise, temperature)


@pytest.mark.parametrize("guided,copies,eta,temperature", [
    (False, 1, 0.0, 1.0), (False, 1, 0.7, 0.8), (True, 2, 0.0, 1.0), (True, 2, 0.7, 1.3), (True, 1, 0.7, 1.0),
])
def test_ddim_step_is_the_oracles_step_at_every_t_index(guided, copies, eta, temperature):
    B, C, H, W, Cp, S, scale = 3, 4, 8, 16, 64, 50, 7.5
    ts, coef = step_tables(torch.from_numpy(alphas_cumprod_table(1000)), "uniform", S, eta)
    coef_d, ts_d = coef.to(DEV), ts.to(DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    bad = torch.zeros(1, dtype=torch.int32, device=DEV)
    next_in = torch.full((copies * B, H, W, Cp), float("nan"), dtype=torch.bfloat16, device=DEV)
    next_ts = torch.full((copies * B,), -7, dtype=torch.int64, device=DEV)
    x, _, _, _ = _step_inputs(B, C, H, W, guided, seed=0)
    for i in range(S):
        _, noise, ec, eu = _step_inputs(B, C, H, W, guided, seed=100 + i)
        ref = _oracle_step(x, noise, ec, eu, scale, coef[i], temperature)
        prev_in, prev_ts = next_in.clone(), next_ts.clone()
        ops.ddim_step(ec, eu, scale, x, noise, coef_d, ts_d, temperature, step, bad, next_in, next_ts)
        assert torch.equal(_bits(x), _bits(ref)), f"step {i}"
        assert int(step.item()) == i + 1 and int(bad.item()) == 0
        if i + 1 < S:
            want = F.pad(ref.to(torch.bfloat16).permute(0, 2, 3, 1), (0, Cp - C)).repeat(copies, 1, 1, 1)
            assert torch.equal(_bits(next_in), _bits(want)), f"next_in after step {i}"
            assert (next_ts == ts[i + 1]).all()
        else:  # no next step: nothing written
            assert torch.equal(_bits(next_in), _bits(prev_in)) and torch.equal(next_ts, prev_ts)


def test_guidance_at_scale_one_is_the_conditional_output():
    B, C, H, W = 2, 4, 8, 8
    ts, coef = step_tables(torch.from_numpy(alphas_cumprod_table(1000)), "uniform", 50, 0.0)
    x, noise, ec, eu = _step_inputs(B, C, H, W, True, seed=3)
    ref = _oracle_step(x, noise, ec, None, 1.0, coef[0], 1.0)
    step, bad = torch.zeros(1, dtype=torch.int32, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
    ops.ddim_step(ec, eu, 1.0, x, noise, coef.to(DEV), ts.to(DEV), 1.0, step, bad,
                  torch.empty((B, H, W, 64), dtype=torch.bfloat16, device=DEV), torch.empty(B, dtype=torch.int64, device=DEV))
    assert torch.equal(_bits(x), _bits(ref))


@pytest.mark.parametrize("counter", [-1, 50, 1 << 30])
def test_out_of_range_counter_sets_the_flag_and_poisons_x(counter):
    B, C, H, W = 2, 4, 8, 8
    ts, coef = step_tables(torch.from_numpy(alphas_cumprod_table(1000)), "uniform", 50, 0.0)
    x, noise, ec, eu = _step_inputs(B, C, H, W, True, seed=4)
    step = torch.full((1,), counter, dtype=torch.int32, device=DEV)
    bad = torch.zeros(1, dtype=torch.int32, device=DEV)
    next_in = torch.zeros((2 * B, H, W, 64), dtype=torch.bfloat16, device=DEV)
    next_ts = torch.full((2 * B,), -7, dtype=torch.int64, device=DEV)
    ops.ddim_step(ec, eu, 7.5, x, noise, coef.to(DEV), ts.to(DEV), 1.0, step, bad, next_in, next_ts, increment=False)
    assert int(bad.item()) == 1 and torch.isnan(x).all()
    assert int(step.item()) == counter and not next_in.any() and (next_ts == -7).all()


# (B, C, H, W, Cp) of the noising kernel's footprint: C = 4 in one group of many; odd C with a half-real last pair; two real groups
DDIM_SHAPES = [(2, 4, 8, 16, 64), (3, 5, 6, 7, 24), (2, 9, 3, 5, 16)]
DDIM_STEPS = 7


@covers("b200_ddim_step_bf16")
@pytest.mark.parametrize("increment", [0, 1])
@pytest.mark.parametrize("counter", [0, 3, DDIM_STEPS - 1, -1, DDIM_STEPS])
@pytest.mark.parametrize("copies,scale", [(1, 7.5), (2, 7.5), (2, 1.0)], ids=["unguided", "guided", "guided_scale_1"])
@pytest.mark.parametrize("B,C,H,W,Cp", DDIM_SHAPES)
def test_ddim_step_footprint(B, C, H, W, Cp, copies, scale, counter, increment):
    """Guarded buffers (test_kernel_footprint_gpu): coef [S, 5] has poison rows at -1 and S, so a read of either NaNs x.  In range,
    x is the oracle's step bit for bit, and next_in / next_ts are written in full, or, on the last step, left exactly as they were.
    Out of range, only x (NaN), the flag and the counter change.  The counter ends at its start plus increment."""
    ts, coef = step_tables(torch.from_numpy(alphas_cumprod_table(1000)), "uniform", DDIM_STEPS, 0.7)
    temperature = 1.3
    x, noise, ec, eu = _step_inputs(B, C, H, W, copies == 2, seed=B * 100 + C)
    ok = 0 <= counter < DDIM_STEPS
    writes_next = ok and counter + 1 < DDIM_STEPS
    rows = lambda v: v.permute(0, 2, 3, 1).reshape(-1, C)  # noqa: E731  ([B, C, H, W] view of channels-last memory -> [B H W, C])
    c = Case(f"ddim_step {B}x{C}x{H}x{W} Cp {Cp} copies {copies} scale {scale} counter {counter} increment {increment}")
    ge = c.input("eps", rows(ec))
    gu = c.input("eps_uncond", rows(eu)) if eu is not None else None
    gx = c.inout("x", x.reshape(B * C, H * W))
    gn = c.input("noise", noise.reshape(B * C, H * W))
    gc, gts = c.input("coef", coef), c.input("ts_table", ts)
    step = c.inout("step_dev", torch.tensor([counter], dtype=torch.int32))
    flag = c.inout("bad_flag", torch.zeros(1, dtype=torch.int32))
    n_in = copies * B * H * W
    prior_in, prior_ts = rand((n_in, Cp), 7), torch.arange(copies * B, dtype=torch.int64) - 7
    if writes_next:
        nin, nts = c.output("next_in", n_in, Cp, dtype=torch.bfloat16), c.output("next_ts", 1, copies * B, dtype=torch.int64)
    else:
        nin, nts = c.inout("next_in", prior_in), c.inout("next_ts", prior_ts)
    r = c.run(lambda: call("b200_ddim_step_bf16", ge.ptr(), gu.ptr() if gu else None, scale, gx.ptr(), gn.ptr(), gc.ptr(), gts.ptr(),
                           DDIM_STEPS, temperature, step.ptr(), increment, flag.ptr(), nin.ptr(), nts.ptr(), copies, B, C, H, W, Cp,
                           current_stream()), nan_ok=() if ok else ("x",))
    assert r["step_dev"].item() == counter + increment and r["bad_flag"].item() == int(not ok), c.name
    if ok:
        ref = _oracle_step(x, noise, ec, eu, scale, coef[counter], temperature)
        assert torch.equal(_bits(r["x"]), _bits(ref.reshape(B * C, H * W).cpu())), f"{c.name}: x"
    else:
        assert torch.isnan(r["x"]).all(), f"{c.name}: x"
    if writes_next:
        want = F.pad(ref.to(torch.bfloat16).permute(0, 2, 3, 1), (0, Cp - C)).repeat(copies, 1, 1, 1).reshape(n_in, Cp).cpu()
        assert torch.equal(_bits(r["next_in"]), _bits(want)), f"{c.name}: next_in"
        assert (r["next_ts"] == ts[counter + 1]).all(), f"{c.name}: next_ts"
    else:
        assert torch.equal(_bits(r["next_in"]), _bits(prior_in)), f"{c.name}: next_in"
        assert torch.equal(r["next_ts"].view(-1), prior_ts), f"{c.name}: next_ts"


# ---- decode against the oracle loop on the same native UNet ------------------------------------------------------------------------------
def _denoiser(m):
    def denoise(image, ts, cond):
        with torch.no_grad():
            return m.unet.forward_padded(ops.pad_channels(image, 64), ts, cond)
    return denoise


def _contexts(case, B, D, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    cond = None if case["cond_tokens"] is None else torch.randn(B, case["cond_tokens"], D, device=DEV, generator=g)
    uncond = None if case["uncond_tokens"] is None else torch.randn(1, case["uncond_tokens"], D, device=DEV, generator=g)
    return cond, uncond


def _decode_and_oracle(m, case, z_shape, cond, uncond, seed):
    cfg = dict(eta=case["eta"], discretize=case["discretize"], unconditional_cond=uncond, temperature=case["temperature"],
               unconditional_guidance_scale=case["unconditional_guidance_scale"])
    m.switch_sampler("ddim", cfg)
    torch.manual_seed(seed)
    z = torch.randn(z_shape, device=DEV)
    out = m.decode(z, cond=cond, num_steps=case["num_steps"])
    state = torch.cuda.get_rng_state()
    torch.manual_seed(seed)
    z = torch.randn(z_shape, device=DEV)
    ref = ddim_oracle.sample(_denoiser(m), m.alphas_cumprod, z, cond=cond, unconditional_cond=uncond, num_steps=case["num_steps"],
                             eta=case["eta"], discretize=case["discretize"], temperature=case["temperature"],
                             unconditional_guidance_scale=case["unconditional_guidance_scale"],
                             has_condition_model=m.condition_model is not None)
    return out, state, ref, torch.cuda.get_rng_state()


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_decode_is_the_oracle_loop_on_the_native_unet(case):
    # without a context the UNet's cross-attention attends to its own tokens, which needs context_dim None (as in the reference)
    cfg = dict(SMALL, context_dim=SMALL["context_dim"] if case["cond_tokens"] else None)
    m = _ddpm(cfg, 16, timesteps=case["T"], condition_model="identity" if case["condition_model"] else None,
              **SCHEDULES[case["T"]])
    m.load_state_dict(_weights(m, 7), strict=True)
    m = m.to(DEV)
    cond, uncond = _contexts(case, 2, SMALL["context_dim"], seed=case["seed"])
    if "raises" in case:
        with pytest.raises(ValueError):
            m.decode(torch.zeros(2, 4, 16, 16, device=DEV), cond=cond, num_steps=case["num_steps"])
        return
    out, state, ref, ref_state = _decode_and_oracle(m, case, (2, 4, 16, 16), cond, uncond, seed=case["seed"])
    assert torch.equal(_bits(out), _bits(ref)) and torch.isfinite(out).all()
    assert torch.equal(state, ref_state)
    assert int(m.sampler.last_bad_flag.item()) == 0


def test_decode_at_sd_v1_5_with_guidance():
    d = json.load(open(os.path.join(GOLDEN, "unet_sd_v1_5_state_dict_keys.json")))
    cfg = {k: tuple(v) if isinstance(v, list) else v for k, v in d["config"].items()}
    m = _ddpm(cfg, 64, condition_model="identity")
    m.load_state_dict(_weights(m, 8), strict=True)
    m = m.to(DEV)
    case = dict(eta=0.0, discretize="uniform", temperature=1.0, unconditional_guidance_scale=7.5, num_steps=50,
                cond_tokens=77, uncond_tokens=77)
    cond, uncond = _contexts(case, 2, cfg["context_dim"], seed=9)
    out, state, ref, ref_state = _decode_and_oracle(m, case, (2, 4, 64, 64), cond, uncond, seed=9)
    assert torch.equal(_bits(out), _bits(ref)) and torch.isfinite(out).all()
    assert torch.equal(state, ref_state)


# ---- the graph cache --------------------------------------------------------------------------------------------------------------------
def test_graph_is_reused_recaptured_and_follows_the_weights():
    m = _ddpm(SMALL, 16, condition_model="identity",
              sampler_config=dict(unconditional_cond=torch.randn(1, 5, 64), unconditional_guidance_scale=7.5, default_steps=6))
    m.load_state_dict(_weights(m, 10), strict=True)
    m = m.to(DEV)
    m.sampler.unconditional_cond = m.sampler.unconditional_cond.to(DEV)
    cond = torch.randn(2, 5, 64, device=DEV)
    torch.manual_seed(1)
    a = m.sample(2, cond=cond)
    torch.manual_seed(1)
    b = m.sample(2, cond=cond)
    assert torch.equal(_bits(a), _bits(b)) and m.sampler.captures == 1
    assert a.abs().max() <= 1.0
    m.sample(3, cond=torch.randn(3, 5, 64, device=DEV))  # a new batch size
    assert m.sampler.captures == 2
    m.sample(3, cond=torch.randn(3, 5, 64, device=DEV), num_steps=4)  # a new step count
    assert m.sampler.captures == 3
    m.to("cpu").to(DEV)  # the parameters' storage moves
    torch.manual_seed(1)
    c = m.sample(2, cond=cond)
    assert m.sampler.captures == 4 and torch.equal(_bits(a), _bits(c))
    # an optimizer step changes the weights in place: the same graph samples with the new ones
    opt = ArenaAdamW(m, lr=1e-2)
    m.arena.grad.copy_(torch.randn(m.arena.total, device=DEV) * 1e-2)
    opt.step()
    torch.manual_seed(1)
    d = m.sample(2, cond=cond, clip_output=False)
    assert m.sampler.captures == 4
    torch.manual_seed(1)
    z = torch.randn(2, 4, 16, 16, device=DEV)
    ref = ddim_oracle.sample(_denoiser(m), m.alphas_cumprod, z, cond=cond, unconditional_cond=m.sampler.unconditional_cond,
                             num_steps=6, unconditional_guidance_scale=7.5)
    assert torch.equal(_bits(d), _bits(ref)) and not torch.equal(_bits(d.clip(-1, 1)), _bits(a))
    m.sampler.release()
    assert m.sampler._graph is None


# ---- sampling between graphed training steps ------------------------------------------------------------------------------------------
def _seam(sd):
    m = _ddpm(SMALL, 16)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV)
    opt = ArenaAdamW(m, lr=1e-4, capturable=True)
    static = [torch.zeros(2, 4, 16, 16, device=DEV), torch.zeros(2, 7, 64, device=DEV), torch.zeros(2, 4, 16, 16, device=DEV),
              torch.zeros(2, dtype=torch.int64, device=DEV)]
    return m, B200TrainStep(m, opt, clip_norm=1.0, graph=True, static_inputs=static)


def test_sampling_between_graphed_training_steps_changes_nothing():
    sd = _weights(_ddpm(SMALL, 16), 11)
    g = torch.Generator().manual_seed(12)
    batches = [(torch.randn(2, 4, 16, 16, generator=g).to(DEV), torch.randn(2, 7, 64, generator=g).to(DEV),
                torch.randn(2, 4, 16, 16, generator=g).to(DEV), torch.randint(0, 1000, (2,), generator=g).to(DEV)) for _ in range(3)]
    m_a, s_a = _seam(sd)
    m_b, s_b = _seam(sd)
    for x, ctx, noise, ts in batches:
        l_a = s_a.step(x, ctx, noise, ts)
        m_b.sample(2, cond=ctx, num_steps=3)
        l_b = s_b.step(x, ctx, noise, ts)
        assert torch.equal(l_a, l_b)
    for (k, p), (_, q) in zip(m_a.named_parameters(), m_b.named_parameters()):
        assert torch.equal(_bits(p), _bits(q)), k
    assert torch.equal(m_a.arena.grad, m_b.arena.grad)
    s_a.close()
    s_b.close()
