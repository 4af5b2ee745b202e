"""Plain-PyTorch restatement of the reference's ``DDIMSampler`` (cflearn/modules/multimodal/diffusion/samplers/ddim.py:37-293
and the classifier-free guidance of samplers/schema.py:153-255), with the denoiser passed in: the float64 tables, the per-step
fp32 scalars, the guided model output and the update, each with the reference's dtypes and rounding points, and the loop
with its draws.  Test infrastructure: ``tests/test_ddim_contract.py`` checks it against ``tests/golden/ddim_reference.pt`` (the
reference's own sampler, run by ``tools/make_golden_ddim.py``), and the GPU tests drive it with the native UNet.

``denoise(image, ts, cond)`` returns the model output for an fp32 image [B, C, H, W], int64 timesteps [B] and a context
[B, Tk, D] (or None)."""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional

import numpy as np
import torch
from torch import Tensor

Denoise = Callable[[Tensor, Tensor, Optional[Tensor]], Tensor]


def ddim_timesteps(t: int, discretize: str, total_step: int) -> np.ndarray:
    """DDIMQSampler.reset_buffers (ddim.py:38-53): the DDIM timesteps, possibly more than ``total_step`` of them ("uniform")."""
    if discretize == "uniform":
        span = t // (total_step + int(t % total_step == 0) - 1)
        q = np.array(list(range(0, t, span)) + [t - 1])
    elif discretize == "quad":
        end = math.sqrt(t * 0.8)
        q = (np.linspace(0, end, total_step) ** 2).astype(int)
    else:
        raise ValueError(f"unrecognized discretize method '{discretize}' occurred")
    q += 1
    return np.minimum(q, t - 1)


def tables(alphas_cumprod: Tensor, discretize: str, total_step: int, eta: float) -> Dict[str, object]:
    """DDIMMixin._reset_buffers (ddim.py:241-268) on the model's float64 ``alphas_cumprod``: float64 tables and the timesteps."""
    q = ddim_timesteps(alphas_cumprod.shape[0], discretize, total_step)
    alphas = alphas_cumprod[q]
    alphas_prev = torch.tensor([alphas_cumprod[0]] + alphas_cumprod[q[:-1]].tolist(), dtype=alphas_cumprod.dtype)
    sigmas = eta * torch.sqrt((1.0 - alphas_prev) / (1.0 - alphas) * (1.0 - alphas / alphas_prev))
    return dict(alphas=alphas, alphas_prev=alphas_prev, sigmas=sigmas, sqrt_one_minus_alphas=torch.sqrt(1.0 - alphas),
                timesteps=q.tolist())


def step_scalars(tab: Dict[str, object], t_index: int, b: int, device: torch.device) -> Dict[str, Tensor]:
    """_register_temp_buffers (ddim.py:175-193): torch.full of one float64 entry at the image's dtype (fp32)."""
    def extract(base: Tensor) -> Tensor:
        return torch.full((b, 1, 1, 1), base[t_index], dtype=torch.float32, device=device)

    return dict(at=extract(tab["alphas"]), a_prev=extract(tab["alphas_prev"]), sigma=extract(tab["sigmas"]),
                s1m=extract(tab["sqrt_one_minus_alphas"]))


def coefficients(s: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """The fp32 factors of the update, as ddim.py:207 and :234-238 compute them."""
    return dict(s1m=s["s1m"], sqrt_a=s["at"].sqrt(), sqrt_ap=s["a_prev"].sqrt(), c_dir=(1.0 - s["a_prev"] - s["sigma"] ** 2).sqrt(),
                sigma=s["sigma"])


def guided_output(denoise: Denoise, image: Tensor, ts: Tensor, cond: Optional[Tensor], uncond: Optional[Tensor], scale: float) -> Tensor:
    """UncondSamplerMixin._uncond_denoise (schema.py:215-255) for tensor conditions."""
    if cond is None or uncond is None or scale == 1.0:
        return denoise(image, ts, cond)
    uncond = uncond.repeat_interleave(image.shape[0], dim=0)
    if cond.shape[1] == uncond.shape[1]:
        eps, eps_uncond = denoise(torch.cat([image, image]), torch.cat([ts, ts]), torch.cat([cond, uncond])).chunk(2)
    else:
        eps = denoise(image, ts, cond)
        eps_uncond = denoise(image, ts, uncond)
    return eps_uncond + scale * (eps - eps_uncond)


def update(image: Tensor, eps: Tensor, c: Dict[str, Tensor], noise: Tensor, temperature: float) -> Tensor:
    """_get_pred_x0 + _get_denoised_and_pred_x0 (ddim.py:195-239) for eps parameterization, with the step's draw passed in."""
    pred_x0 = (image - c["s1m"] * eps) / c["sqrt_a"]
    direction = c["c_dir"] * eps
    noise = c["sigma"] * noise * temperature
    return c["sqrt_ap"] * pred_x0 + direction + noise


def sample(denoise: Denoise, alphas_cumprod: Tensor, z: Tensor, *, num_steps: int = 50, cond: Optional[Tensor] = None,
           eta: float = 0.0, discretize: str = "uniform", unconditional_cond: Optional[Tensor] = None,
           unconditional_guidance_scale: float = 1.0, temperature: float = 1.0, has_condition_model: bool = True,
           trace: Optional[List[Tensor]] = None) -> Tensor:
    """ISampler.sample (schema.py:153-194) with DDIMSampler's step: ``num_steps`` steps from z, one ``randn_like`` per step from
    the image's device generator.  The condition model is the identity (``has_condition_model``) or absent, in which case the
    unconditional context is ignored, as _reset_uncond_buffers does.  ``trace`` receives every step's image."""
    tab = tables(alphas_cumprod, discretize, num_steps, eta)
    if unconditional_cond is None or not has_condition_model:
        uncond, scale = None, 0.0
    else:
        uncond, scale = unconditional_cond, unconditional_guidance_scale
    image = z
    B = z.shape[0]
    for step in range(num_steps):
        t_index = num_steps - step - 1
        ts = torch.full((B,), tab["timesteps"][t_index], device=z.device, dtype=torch.long)
        c = coefficients(step_scalars(tab, t_index, B, z.device))
        eps = guided_output(denoise, image, ts, cond, uncond, scale)
        image = update(image, eps, c, torch.randn_like(image), temperature)
        if trace is not None:
            trace.append(image)
    return image


def standin_denoise(image: Tensor, ts: Tensor, cond: Optional[Tensor]) -> Tensor:
    """A deterministic stand-in for the UNet: bf16, a function of the image, the timestep and the context (so the conditional
    and unconditional halves differ), and of the image's position in the batch only through those."""
    t = ts.to(torch.float32).view(-1, 1, 1, 1)
    C = image.shape[1]
    chan = torch.arange(C, dtype=torch.float32, device=image.device).view(1, C, 1, 1)
    out = image * (0.6 + 0.3 * torch.cos(t * 0.013 + chan)) + 0.2 * torch.sin(t * 0.007 - chan * 0.5)
    if cond is not None:
        c = cond.to(torch.float32)
        out = out + c.mean(dim=(1, 2)).view(-1, 1, 1, 1) * 2.0 + c[:, :, :C].mean(dim=1).view(-1, C, 1, 1)
    return out.to(torch.bfloat16)
