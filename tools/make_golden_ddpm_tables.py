"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/ddpm_noise_tables.pt from the real reference: the noise tables of
``DDPM._register_noise_schedule`` (cflearn/modules/multimodal/diffusion/ddpm.py:599-679, which calls ``make_beta_schedule``,
:51-84), imported unmodified through oracle/load_reference.py, for the four ``beta_schedule``s and for ``given_betas``.  Each
table is rounded to fp32 as ``DDPMQSampler.q_sample``'s ``.to(net)`` does for an fp32 latent (samplers/schema.py:100-101).
Needs a carefree-learn checkout (oracle/load_reference.py):  python tools/make_golden_ddpm_tables.py"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from load_reference import load_reference_modules  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ddpm_noise_tables.pt")
CASES = [(s, T, ls, le, 8e-3) for s in ("linear", "cosine", "sqrt_linear", "sqrt") for T, ls, le in ((1000, 1e-4, 2e-2),
                                                                                                     (37, 8.5e-4, 1.2e-2))]
GIVEN = np.linspace(1e-3, 3e-2, 250, dtype=np.float64)


def tables(ddpm_cls, timesteps, given_betas, schedule, ls, le, cs):
    holder = nn.Module()  # what _register_noise_schedule reads of a DDPM besides its arguments
    holder.parameterization, holder.v_posterior = "eps", 0.0
    ddpm_cls._register_noise_schedule(holder, timesteps, given_betas, schedule, ls, le, cs)
    return {"sqrt_alphas_cumprod": holder.sqrt_alphas_cumprod.to(torch.float32),
            "sqrt_one_minus_alphas_cumprod": holder.sqrt_one_minus_alphas_cumprod.to(torch.float32)}


def main() -> None:
    load_reference_modules()
    from cflearn.modules.multimodal.diffusion.ddpm import DDPM

    out = {"cases": [dict(args=dict(timesteps=T, beta_schedule=s, linear_start=ls, linear_end=le, cosine_s=cs),
                          **tables(DDPM, T, None, s, ls, le, cs)) for s, T, ls, le, cs in CASES]}
    out["cases"].append(dict(args=dict(timesteps=1000, beta_schedule="cosine", linear_start=1e-4, linear_end=2e-2, cosine_s=8e-3,
                                       given_betas=torch.from_numpy(GIVEN)),
                             **tables(DDPM, 1000, GIVEN, "cosine", 1e-4, 2e-2, 8e-3)))
    torch.save(out, OUT)
    print(f"wrote {OUT}: {len(out['cases'])} cases")


if __name__ == "__main__":
    main()
