"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/ddim_reference.pt from the real reference: its ``DDIMSampler``
(cflearn/modules/multimodal/diffusion/samplers/ddim.py, with ``ISampler.sample`` and ``UncondSamplerMixin`` of schema.py),
imported unmodified through oracle/load_reference.py and run on CPU around a holder module that offers what the sampler reads
of a DDPM: ``t``, ``parameterization``, the float64 ``alphas_cumprod`` of the reference's own ``DDPM._register_noise_schedule``,
``condition_model`` (``nn.Identity``, the reference's "identity" condition model, or None), ``get_cond`` (the reference's
``DDPM.get_cond``), ``denoise`` (oracle/ddim_oracle.py's deterministic stand-in) and one parameter for ``get_device``.

Each case records the seed, z (the first draw after seeding), every step's image, the output, the CPU generator's state after
the call, or -- for a discretisation the reference refuses -- the exception's type.
Needs a carefree-learn checkout (oracle/load_reference.py):  python tools/make_golden_ddim.py"""
from __future__ import annotations

import os
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from load_reference import load_reference_modules  # noqa: E402
import ddim_oracle  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ddim_reference.pt")
SCHEDULES = {1000: dict(linear_start=1e-4, linear_end=2e-2), 37: dict(linear_start=8.5e-4, linear_end=1.2e-2)}
SHAPE = (2, 4, 4, 4)
D = 8  # context width


def _case(name, T, steps, discretize="uniform", eta=0.0, temperature=1.0, scale=1.0, tk=3, tku=3, cond=True, uncond=True,
          condition_model=True):
    return dict(name=name, T=T, num_steps=steps, discretize=discretize, eta=eta, temperature=temperature,
                unconditional_guidance_scale=scale, cond_tokens=tk if cond else None, uncond_tokens=tku if uncond else None,
                condition_model=condition_model)


CASES = [
    _case("t1000-50-uniform-cfg-equal", 1000, 50, scale=7.5),
    _case("t1000-50-quad-eta-temp-cfg-unequal", 1000, 50, "quad", eta=0.7, temperature=0.8, scale=7.5, tku=5),
    _case("t1000-50-uniform-eta-scale1", 1000, 50, eta=0.7),
    _case("t1000-7-uniform-eta-cfg-equal", 1000, 7, eta=0.7, scale=7.5),
    _case("t1000-7-quad-temp-nocond", 1000, 7, "quad", temperature=0.8, scale=7.5, cond=False),
    _case("t1000-7-uniform-cfg-unequal", 1000, 7, scale=7.5, tk=4, tku=2),
    _case("t1000-1-uniform-eta-cfg-equal", 1000, 1, eta=0.7, scale=7.5),
    _case("t1000-1-quad-nouncond", 1000, 1, "quad", uncond=False),
    _case("t37-50-uniform-refused", 37, 50),
    _case("t37-50-quad-eta-cfg-equal", 37, 50, "quad", eta=0.7, scale=7.5),
    _case("t37-7-uniform-eta-temp-cfg-equal", 37, 7, eta=0.7, temperature=0.8, scale=7.5),
    _case("t37-7-quad-cfg-unequal", 37, 7, "quad", scale=7.5, tku=6),
    _case("t37-1-uniform-nocond", 37, 1, cond=False, uncond=False),
    _case("t1000-7-uniform-no-condition-model", 1000, 7, eta=0.7, scale=7.5, condition_model=False),
]


def inputs(case, seed):
    """(z, cond, unconditional_cond) for a case: z first, from the seeded global CPU generator, then the contexts from their own."""
    torch.manual_seed(seed)
    z = torch.randn(SHAPE)
    g = torch.Generator().manual_seed(1000 + seed)
    cond = None if case["cond_tokens"] is None else torch.randn(SHAPE[0], case["cond_tokens"], D, generator=g)
    uncond = None if case["uncond_tokens"] is None else torch.randn(1, case["uncond_tokens"], D, generator=g)
    return z, cond, uncond


def main() -> None:
    load_reference_modules()
    from cflearn.modules.multimodal.diffusion.ddpm import DDPM
    from cflearn.modules.multimodal.diffusion.samplers.ddim import DDIMSampler

    out = {"shape": SHAPE, "context_dim": D, "schedules": SCHEDULES, "cases": []}
    for seed, case in enumerate(CASES):
        holder = nn.Module()
        holder.parameterization, holder.v_posterior = "eps", 0.0
        DDPM._register_noise_schedule(holder, case["T"], None, "linear", SCHEDULES[case["T"]]["linear_start"],
                                      SCHEDULES[case["T"]]["linear_end"], 8e-3)
        holder.condition_model = nn.Identity() if case["condition_model"] else None
        holder.get_cond = lambda c, h=holder: DDPM.get_cond(h, c)
        holder.denoise = lambda image, ts, cond, step, total_step: ddim_oracle.standin_denoise(image, ts, cond)
        holder.dummy = nn.Parameter(torch.zeros(1))
        z, cond, uncond = inputs(case, seed)
        sampler = DDIMSampler(holder, eta=case["eta"], discretize=case["discretize"], unconditional_cond=uncond,
                              unconditional_guidance_scale=case["unconditional_guidance_scale"], temperature=case["temperature"])
        seen = []
        rec = dict(case, seed=seed, z=z.clone(), alphas_cumprod=holder.alphas_cumprod.clone())
        try:
            final = sampler.sample(z, cond=cond, num_steps=case["num_steps"], verbose=False,
                                   step_callback=lambda image: seen.append(image.clone()) or True)
        except Exception as e:  # a discretisation the reference cannot make
            rec["raises"] = type(e).__name__
        else:
            rec["steps"] = torch.stack(seen[1:] + [final])
            rec["rng_state"] = torch.get_rng_state()
        out["cases"].append(rec)
        print(case["name"], rec.get("raises", "ok"))
    torch.save(out, OUT)
    print(f"wrote {OUT}: {len(out['cases'])} cases, {os.path.getsize(OUT) // 1024} KiB")


if __name__ == "__main__":
    main()
