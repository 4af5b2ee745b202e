"""DDIM sampling's host surface, checked without a GPU: oracle/ddim_oracle.py against the reference's own DDIMSampler
(tests/golden/ddim_reference.pt, written by tools/make_golden_ddim.py) step by step and for the generator state after the call;
the native host tables (ddim.step_tables) against the oracle's fp32 scalars bit for bit; the refusals of DDPMB200's sampling
keywords and of DDIMSamplerB200; and the argument contract of b200_ddim_step_bf16 (fake pointers, never dereferenced: refused
calls stop at the argument checks)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: E402
from cflearn_b200 import _cabi  # noqa: E402
from cflearn_b200.ddim import DDIMSamplerB200, step_tables  # noqa: E402
from cflearn_b200.ddpm import DDPMB200, alphas_cumprod_table  # noqa: E402
import ddim_oracle  # noqa: E402

GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "ddim_reference.pt"))
CASES = GOLDEN["cases"]
ARG, ALIGN = -1, -2
FAKE = 1 << 20
SMALL = dict(num_heads=2, context_dim=64, start_channels=64, num_res_blocks=1, attention_downsample_rates=(1, 2),
             channel_multipliers=(1, 2), use_spatial_transformer=True)


def _inputs(case):
    """The case's seeded draws, as tools/make_golden_ddim.py made them: z first from the global generator, then the contexts."""
    shape, D = GOLDEN["shape"], GOLDEN["context_dim"]
    torch.manual_seed(case["seed"])
    z = torch.randn(shape)
    g = torch.Generator().manual_seed(1000 + case["seed"])
    cond = None if case["cond_tokens"] is None else torch.randn(shape[0], case["cond_tokens"], D, generator=g)
    uncond = None if case["uncond_tokens"] is None else torch.randn(1, case["uncond_tokens"], D, generator=g)
    return z, cond, uncond


def _oracle_kw(case):
    return dict(num_steps=case["num_steps"], eta=case["eta"], discretize=case["discretize"], temperature=case["temperature"],
                unconditional_guidance_scale=case["unconditional_guidance_scale"], has_condition_model=case["condition_model"])


def _alphas(case):
    return torch.from_numpy(alphas_cumprod_table(case["T"], None, "linear", **GOLDEN["schedules"][case["T"]]))


# ---- the oracle against the reference's own sampler ---------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_oracle_reproduces_the_reference_sampler(case):
    assert torch.equal(_alphas(case), case["alphas_cumprod"])
    z, cond, uncond = _inputs(case)
    assert torch.equal(z, case["z"])
    if "raises" in case:
        with pytest.raises(ValueError):
            ddim_oracle.sample(ddim_oracle.standin_denoise, case["alphas_cumprod"], z, cond=cond, unconditional_cond=uncond,
                               **_oracle_kw(case))
        return
    trace = []
    out = ddim_oracle.sample(ddim_oracle.standin_denoise, case["alphas_cumprod"], z, cond=cond, unconditional_cond=uncond,
                             trace=trace, **_oracle_kw(case))
    assert len(trace) == case["num_steps"] == case["steps"].shape[0]
    for i, img in enumerate(trace):
        assert torch.equal(img.view(torch.int32), case["steps"][i].view(torch.int32)), f"step {i}"
    assert torch.equal(out, case["steps"][-1])
    assert torch.equal(torch.get_rng_state(), case["rng_state"])


def test_the_fixture_covers_the_case_matrix():
    ok = [c for c in CASES if "raises" not in c]
    assert {c["T"] for c in ok} == {1000, 37} and {c["num_steps"] for c in ok} == {50, 7, 1}
    assert {c["discretize"] for c in ok} == {"uniform", "quad"}
    assert {c["eta"] for c in ok} == {0.0, 0.7} and {c["temperature"] for c in ok} == {1.0, 0.8}
    guided = [c for c in ok if c["unconditional_guidance_scale"] == 7.5 and c["cond_tokens"] and c["uncond_tokens"]
              and c["condition_model"]]
    assert any(c["cond_tokens"] == c["uncond_tokens"] for c in guided) and any(c["cond_tokens"] != c["uncond_tokens"] for c in guided)
    assert any(c["unconditional_guidance_scale"] == 1.0 and c["uncond_tokens"] for c in ok)
    assert any(c["cond_tokens"] is None for c in ok) and any(not c["condition_model"] and c["uncond_tokens"] for c in ok)
    assert [(c["T"], c["num_steps"], c["discretize"]) for c in CASES if "raises" in c] == [(37, 50, "uniform")]


# ---- the native host tables -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_step_tables_are_the_oracles_fp32_scalars(case):
    ac, S = case["alphas_cumprod"], case["num_steps"]
    if "raises" in case:
        with pytest.raises(ValueError):
            step_tables(ac, case["discretize"], S, case["eta"])
        return
    ts, coef = step_tables(ac, case["discretize"], S, case["eta"])
    assert ts.dtype == torch.int64 and coef.dtype == torch.float32 and coef.shape == (S, 5)
    tab = ddim_oracle.tables(ac, case["discretize"], S, case["eta"])
    for step in range(S):
        t_index = S - step - 1
        assert int(ts[step]) == tab["timesteps"][t_index]
        c = ddim_oracle.coefficients(ddim_oracle.step_scalars(tab, t_index, 2, torch.device("cpu")))
        for j, name in enumerate(("s1m", "sqrt_a", "sqrt_ap", "c_dir", "sigma")):
            assert torch.equal(coef[step, j].view(1).view(torch.int32), c[name][0].view(1).view(torch.int32)), (step, name)


def test_uniform_uses_the_first_num_steps_timesteps():
    ac = torch.from_numpy(alphas_cumprod_table(1000))
    assert len(ddim_oracle.ddim_timesteps(1000, "uniform", 7)) == 8
    ts, _ = step_tables(ac, "uniform", 7, 0.0)
    assert ts.tolist() == [997, 831, 665, 499, 333, 167, 1]


def test_step_tables_refuse_what_the_reference_refuses():
    ac = torch.from_numpy(alphas_cumprod_table(37, None, "linear", 8.5e-4, 1.2e-2))
    with pytest.raises(ValueError):
        step_tables(ac, "uniform", 50, 0.0)
    with pytest.raises(ValueError, match="unrecognized discretize"):
        step_tables(ac, "cubic", 5, 0.0)


# ---- DDPMB200's sampling keywords -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["basic", "plms", "klms", "k_euler", "k_euler_a", "k_heun", "k_dpmpp_2m", "solver", "lcm"])
def test_other_samplers_are_refused_by_name(name):
    with pytest.raises(NotImplementedError, match=f"sampler='{name}'"):
        DDPMB200(16, 4, 4, sampler=name, **SMALL)
    m = DDPMB200(16, 4, 4, **SMALL)
    with pytest.raises(NotImplementedError, match=name):
        m.switch_sampler(name)


@pytest.mark.parametrize("cm", ["clip", "identityx"])
def test_other_condition_models_are_still_refused(cm):
    with pytest.raises(NotImplementedError, match="condition_model"):
        DDPMB200(16, 4, 4, condition_model=cm, **SMALL)


@pytest.mark.parametrize("cfg,option", [(dict(noise_dropout=0.1), "noise_dropout"), (dict(quantize_denoised=True), "quantize_denoised")])
def test_sampler_config_refusals_name_the_option(cfg, option):
    with pytest.raises(NotImplementedError, match=option):
        DDPMB200(16, 4, 4, sampler_config=cfg, **SMALL)


@pytest.mark.parametrize("kw,option", [
    (dict(start_step=3), "start_step"), (dict(ref=torch.zeros(1)), "ref"), (dict(ref_mask=torch.zeros(1)), "ref_mask"),
    (dict(step_callback=lambda image: True), "step_callback"), (dict(noise_dropout=0.5), "noise_dropout"),
    (dict(quantize_denoised=True), "quantize_denoised"), (dict(cond={"context": torch.zeros(1)}), "dict conds"),
])
def test_decode_refusals_name_the_option(kw, option):
    m = DDPMB200(16, 4, 4, **SMALL)
    with pytest.raises(NotImplementedError, match=option):
        m.decode(torch.zeros(1, 4, 16, 16), num_steps=2, **kw)


def test_decode_refuses_a_cpu_latent_and_unknown_keywords():
    m = DDPMB200(16, 4, 4, **SMALL)
    with pytest.raises(cflearn_b200.B200Error, match="CUDA fp32 latent"):
        m.decode(torch.zeros(1, 4, 16, 16), num_steps=2)
    with pytest.raises(TypeError, match="unexpected keyword"):
        m.decode(torch.zeros(1, 4, 16, 16), num_steps=2, guidance=3.0)


def test_sampling_keywords_leave_the_state_dict_alone():
    base = DDPMB200(16, 4, 4, **SMALL).state_dict()
    for kw in (dict(condition_model="identity"), dict(sampler="ddim", sampler_config=dict(eta=0.5, default_steps=20)),
               dict(condition_model="identity", sampler_config=dict(unconditional_cond=torch.zeros(1, 3, 64)))):
        sd = DDPMB200(16, 4, 4, **SMALL, **kw).state_dict()
        assert list(sd) == list(base) and all(sd[k].shape == base[k].shape for k in sd), kw
    m = DDPMB200(16, 4, 4, condition_model="identity", **SMALL)
    assert isinstance(m.condition_model, torch.nn.Identity) and m.alphas_cumprod.dtype == torch.float64
    assert "alphas_cumprod" not in m.state_dict()
    c = torch.randn(2, 3, 64)
    assert m.get_cond(c) is c
    with pytest.raises(ValueError, match="condition_model"):
        DDPMB200(16, 4, 4, **SMALL).get_cond(c)


def test_sampler_takes_ddim_mixins_keywords():
    m = DDPMB200(16, 4, 4, sampler_config=dict(eta=0.3, discretize="quad", unconditional_guidance_scale=5.0, temperature=0.9,
                                               default_steps=12), **SMALL)
    s = m.sampler
    assert isinstance(s, DDIMSamplerB200) and s.default_steps == 12
    assert s.sample_kwargs == dict(eta=0.3, discretize="quad", unconditional_cond=None, unconditional_guidance_scale=5.0,
                                   temperature=0.9, noise_dropout=0.0, quantize_denoised=False)
    m.switch_sampler("ddim", dict(eta=0.0))
    assert m.sampler is not s and m.sampler.eta == 0.0 and m.sampler.default_steps == 50


# ---- b200_ddim_step_bf16's argument contract -------------------------------------------------------------------------------------------
def _status(name, *args):
    rc = getattr(_cabi.lib(), name)(*args)
    return rc, _cabi.last_error()


@pytest.mark.parametrize("kw,code,text", [
    (dict(B=0), ARG, "non-positive size"), (dict(C=0), ARG, "non-positive size"), (dict(H=0), ARG, "non-positive size"),
    (dict(W=0), ARG, "non-positive size"), (dict(Cp=0), ARG, "non-positive size"), (dict(S=0), ARG, "non-positive size"),
    (dict(Cp=60), ARG, "multiple of 8"), (dict(C=65), ARG, "at most Cp"), (dict(copies=3), ARG, "copies"),
    (dict(copies=0), ARG, "copies"), (dict(copies=2, eu=None), ARG, "needs eps_uncond"), (dict(inc=2), ARG, "increment"),
    (dict(B=1, C=1, H=46341, W=46341, Cp=8), ARG, "H * W"), (dict(B=1 << 21, H=1 << 10, W=1 << 10), ARG, "too many"),
    (dict(eps=None), ARG, "null pointer"), (dict(x=None), ARG, "null pointer"), (dict(noise=None), ARG, "null pointer"),
    (dict(coef=None), ARG, "null pointer"), (dict(ts=None), ARG, "null pointer"), (dict(step=None), ARG, "null pointer"),
    (dict(bad=None), ARG, "null pointer"), (dict(nin=None), ARG, "null pointer"), (dict(nts=None), ARG, "null pointer"),
    (dict(eps=FAKE + 1), ALIGN, "element size"), (dict(eu=FAKE + 1), ALIGN, "element size"), (dict(x=FAKE + 2), ALIGN, "element size"),
    (dict(noise=FAKE + 2), ALIGN, "element size"), (dict(coef=FAKE + 2), ALIGN, "element size"), (dict(ts=FAKE + 4), ALIGN, "element size"),
    (dict(step=FAKE + 2), ALIGN, "element size"), (dict(bad=FAKE + 1), ALIGN, "element size"), (dict(nts=FAKE + 4), ALIGN, "element size"),
    (dict(nin=FAKE + 8), ALIGN, "16-byte aligned"),
])
def test_ddim_step_refusals(kw, code, text):
    a = dict(eps=FAKE, eu=FAKE, scale=7.5, x=FAKE, noise=FAKE, coef=FAKE, ts=FAKE, S=50, temp=1.0, step=FAKE, inc=1, bad=FAKE,
             nin=FAKE, nts=FAKE, copies=1, B=2, C=4, H=8, W=8, Cp=64)
    a.update(kw)
    rc, msg = _status("b200_ddim_step_bf16", a["eps"], a["eu"], a["scale"], a["x"], a["noise"], a["coef"], a["ts"], a["S"], a["temp"],
                      a["step"], a["inc"], a["bad"], a["nin"], a["nts"], a["copies"], a["B"], a["C"], a["H"], a["W"], a["Cp"], None)
    assert rc == code and text in msg and "ddim_step" in msg, (rc, msg)

