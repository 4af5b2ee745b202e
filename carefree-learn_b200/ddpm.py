"""The reference's ``DDPM`` training forward (cflearn/modules/multimodal/diffusion/ddpm.py:250-260) on the native SD-UNet.

``DDPMB200`` wraps a ``UNetDiffuserB200`` (child ``unet``, so its keys are ``unet.*`` as in the reference) and the noise schedule
(``make_beta_schedule`` / ``_register_noise_schedule``, ddpm.py:51-84 and :599-679, computed in float64 and rounded to fp32 once,
as ``q_sample``'s ``.to(net)`` does).  One training step is

    timesteps = randint(0, T, (B,)), noise = randn_like(net)        the current CUDA generator, in the reference's order
    x = bf16(sqrt_ac[t] net + sqrt_1m_ac[t] noise), padded to 64    ops.q_sample_pad (samplers/schema.py:94-108 + the stem's cast)
    pred = unet(x, t, cond); loss = noise_prediction_loss(pred, noise); loss.backward()

with every parameter gradient written into one flat arena (``unet.UNetGradArena``), bucket by bucket in the order backward
completes them, and all-reduced bucket by bucket when a communicator is attached (``dp.attach_native_reducers``).  The arena is
what ``optim.ArenaAdam`` / ``ArenaAdamW``, ``trainer.B200TrainStep`` and ``optim.GraphedTrainStep`` drive, so the whole step --
draws, noising, forward, loss, backward, exchange, clipping and the update -- is one CUDA graph.

Sampling is the reference's default, DDIM with classifier-free guidance (``ddim.DDIMSamplerB200``): ``sample`` / ``decode``
run one CUDA-graph replay per denoising step.

Not implemented, and refused by name: other parameterizations than ``eps``, a learned log-variance, EMA, condition models other
than "identity" (pass the encoded context as ``cond``) and samplers other than "ddim".
"""
from __future__ import annotations

from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch
from torch import Tensor, nn

from . import ops
from .ddim import DDIMSamplerB200
from ._cabi import B200Error
from .unet import PAD_CHANNELS, UNetDiffuserB200, enable_grad_arena, noise_prediction_loss

PREDICTIONS_KEY = "predictions"  # cflearn/constants.py
NOISE_KEY = "noise"  # DDPM.noise_key (ddpm.py:99)
TIMESTEPS_KEY = "timesteps"  # DDPM.timesteps_key (ddpm.py:100)
IDENTITY_CONDITION_MODEL = "identity"  # DDPM.identity_condition_model (ddpm.py:101)


def _check_sampler(sampler: str) -> None:
    if sampler != "ddim":
        raise NotImplementedError(f"DDPMB200: sampler={sampler!r} is not supported (ddim only)")


def make_beta_schedule(schedule: str, timesteps: int, linear_start: float, linear_end: float, cosine_s: float) -> np.ndarray:
    """ddpm.py:51-84, float64."""
    if schedule == "linear":
        return np.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=np.float64) ** 2
    if schedule == "cosine":
        arange = np.arange(timesteps + 1, dtype=np.float64)
        alphas = np.cos((arange / timesteps + cosine_s) / (1 + cosine_s) * np.pi / 2) ** 2
        alphas = alphas / alphas[0]
        return np.clip(1.0 - alphas[1:] / alphas[:-1], 0.0, 0.999)
    lin = np.linspace(linear_start, linear_end, timesteps, dtype=np.float64)
    if schedule == "sqrt_linear":
        return lin
    if schedule == "sqrt":
        return lin ** 0.5
    raise ValueError(f"unrecognized schedule '{schedule}' occurred")


def alphas_cumprod_table(timesteps: int = 1000, given_betas: Optional[np.ndarray] = None, beta_schedule: str = "linear",
                         linear_start: float = 1.0e-4, linear_end: float = 2.0e-2, cosine_s: float = 8.0e-3) -> np.ndarray:
    """alphas_cumprod as _register_noise_schedule (ddpm.py:608-616) computes it: float64 [T]."""
    if given_betas is not None:
        betas = np.asarray(given_betas, dtype=np.float64)
    else:
        betas = make_beta_schedule(beta_schedule, timesteps, linear_start, linear_end, cosine_s)
    return np.cumprod(1.0 - betas, axis=0)


def noise_tables(timesteps: int = 1000, given_betas: Optional[np.ndarray] = None, beta_schedule: str = "linear",
                 linear_start: float = 1.0e-4, linear_end: float = 2.0e-2, cosine_s: float = 8.0e-3) -> Tuple[Tensor, Tensor]:
    """(sqrt(alphas_cumprod), sqrt(1 - alphas_cumprod)) as fp32 [T]: _register_noise_schedule (ddpm.py:599-629) in float64, then
    one rounding to fp32."""
    alphas_cumprod = alphas_cumprod_table(timesteps, given_betas, beta_schedule, linear_start, linear_end, cosine_s)
    a = torch.from_numpy(np.sqrt(alphas_cumprod)).to(torch.float32)
    s = torch.from_numpy(np.sqrt(1.0 - alphas_cumprod)).to(torch.float32)
    return a, s


class DDPMB200(nn.Module):
    """Drop-in for the training forward of cflearn's ``DDPM`` with an SD-style ``UNetDiffuser`` on the native kernels (CUDA only).

    ``forward(net, cond)``: DDPM.forward's dict {predictions, noise, timesteps} for the fp32 latent ``net`` [B, C, H, W] and the
    context ``cond`` [B, Tk, context_dim] (or None).  ``train_step(net, cond, noise=None, timesteps=None)``: noising, forward,
    loss and backward into the gradient arena; returns the loss (fp32 device scalar).  ``noise`` / ``timesteps`` replace the
    draws (parity checks).  A timestep outside [0, T) sets ``last_bad_flag`` (int32 [1] on the device) and makes its image NaN.

    ``state_dict`` holds the UNet's parameters under ``unet.*`` only: the schedule's tables follow from the constructor's
    keywords, so load a reference DDPM's ``unet.state_dict()`` into ``unet`` rather than its whole ``state_dict`` (which also
    carries the schedule buffers)."""

    def __init__(self, img_size: int, in_channels: int, out_channels: int, *, num_heads: Optional[int] = 8,
                 channel_multipliers: Tuple[int, ...] = (1, 2, 4, 4), ema_decay: Optional[float] = None, parameterization: str = "eps",
                 condition_model: Optional[str] = None, timesteps: int = 1000, given_betas: Optional[np.ndarray] = None,
                 beta_schedule: str = "linear", linear_start: float = 1.0e-4, linear_end: float = 2.0e-2, cosine_s: float = 8.0e-3,
                 learn_log_var: bool = False, sampler: str = "ddim", sampler_config: Optional[Dict[str, Any]] = None,
                 **unet_kwargs: Any) -> None:
        super().__init__()
        what = "DDPMB200"
        refused = [(parameterization != "eps", f"parameterization={parameterization!r} (eps only)"),
                   (learn_log_var, "learn_log_var (a learned log-variance)"), (ema_decay is not None, "ema_decay (EMA)"),
                   (condition_model not in (None, IDENTITY_CONDITION_MODEL),
                    "condition_model (pass the encoded context as cond, with condition_model None or \"identity\")")]
        for bad, option in refused:
            if bad:
                raise NotImplementedError(f"{what}: {option} is not supported")
        _check_sampler(sampler)
        self.img_size = img_size
        self.in_channels, self.out_channels = in_channels, out_channels
        self.unet = UNetDiffuserB200(in_channels, out_channels, num_heads=num_heads, channel_multipliers=channel_multipliers,
                                     **unet_kwargs)
        a, s = noise_tables(timesteps, given_betas, beta_schedule, linear_start, linear_end, cosine_s)
        self.t = int(a.shape[0])
        # the reference's float64 buffer, read by the sampler's host tables: a plain attribute, so it stays on the host and out of
        # the state_dict
        self.alphas_cumprod = torch.from_numpy(alphas_cumprod_table(timesteps, given_betas, beta_schedule, linear_start, linear_end,
                                                                    cosine_s))
        # _initialize_condition_model (ddpm.py:573-585): "identity" is nn.Identity, which has no state
        self.condition_model: Optional[nn.Module] = nn.Identity() if condition_model == IDENTITY_CONDITION_MODEL else None
        self.register_buffer("sqrt_alphas_cumprod", a, persistent=False)
        self.register_buffer("sqrt_one_minus_alphas_cumprod", s, persistent=False)
        grads = enable_grad_arena(self.unet)
        self.arena = grads.arena
        self.geo = self.engine = grads  # what dp reads: buckets(), reducer, shrink_next
        self.grad_arena = grads
        self.last_bad_flag: Optional[Tensor] = None
        self.sampler: DDIMSamplerB200
        self.switch_sampler(sampler, sampler_config)

    def _noised(self, net: Tensor, noise: Optional[Tensor], timesteps: Optional[Tensor]) -> Tuple[Tensor, Tensor, Tensor]:
        what = "DDPMB200"
        if net.dim() != 4 or net.shape[1] != self.in_channels or net.dtype != torch.float32 or not net.is_cuda:
            raise B200Error(f"{what}: net must be a CUDA fp32 latent [B, {self.in_channels}, H, W]")
        B = net.shape[0]
        if timesteps is None:
            timesteps = torch.randint(0, self.t, (B,), device=net.device)
        if noise is None:
            noise = torch.randn_like(net)
        x, bad = ops.q_sample_pad(net, noise, timesteps, self.sqrt_alphas_cumprod, self.sqrt_one_minus_alphas_cumprod, PAD_CHANNELS)
        self.last_bad_flag = bad
        return x, noise, timesteps

    def forward(self, net: Tensor, cond: Optional[Tensor] = None) -> Dict[str, Tensor]:
        x, noise, timesteps = self._noised(net, None, None)
        pred = self.unet.forward_padded(x, timesteps, cond)
        return {PREDICTIONS_KEY: pred, NOISE_KEY: noise, TIMESTEPS_KEY: timesteps}

    def train_step(self, net: Tensor, cond: Optional[Tensor] = None, noise: Optional[Tensor] = None,
                   timesteps: Optional[Tensor] = None) -> Tensor:
        x, noise, timesteps = self._noised(net, noise, timesteps)
        loss = noise_prediction_loss(self.unet.forward_padded(x, timesteps, cond), noise)
        loss.backward()  # the gradients land in the arena; buckets start their all-reduce as they complete
        red = self.engine.reducer
        if red is not None:
            red.finish()
        self.grad_arena.end_backward()
        if red is not None:
            self.grad_arena.check()
        return loss.detach()

    # sampling (DDPM.generate_z / decode / sample / get_cond / switch_sampler, ddpm.py:264-356)

    def switch_sampler(self, sampler: str, sampler_config: Optional[Dict[str, Any]] = None) -> None:
        """Replace the sampler: "ddim" with ``DDIMSamplerB200``'s keywords; any other name raises ``NotImplementedError``."""
        _check_sampler(sampler)
        old = getattr(self, "sampler", None)
        if old is not None:
            old.release()
        self.sampler = DDIMSamplerB200(self, **(sampler_config or {}))

    def get_cond(self, cond: Any) -> Any:
        if self.condition_model is None:
            raise ValueError("should not call `get_cond` when `condition_model` is not provided")
        return self.condition_model(cond)

    def decode(self, z: Tensor, *, cond: Optional[Any] = None, num_steps: Optional[int] = None, start_step: Optional[int] = None,
               verbose: bool = False, **kwargs: Any) -> Tensor:
        """The sampler's loop from the fp32 latent z [B, in_channels, H, W] (CUDA, contiguous), conditioned on ``cond`` (an
        encoded context [B, Tk, context_dim], or None).  ``kwargs`` override the sampler's keywords for this call."""
        return self.sampler.sample(z, cond=cond, num_steps=num_steps, start_step=start_step, verbose=verbose, **kwargs)

    def sample(self, num_samples: int, *, cond: Optional[Any] = None, num_steps: Optional[int] = None,
               start_step: Optional[int] = None, clip_output: bool = True, verbose: bool = False,
               kwargs: Optional[Dict[str, Any]] = None, **other_kw: Any) -> Tensor:
        """``num_samples`` latents from ``torch.randn`` [n, in_channels, img_size, img_size] on the parameters' device (the current
        CUDA generator), then ``decode``, then clipped to [-1, 1] unless ``clip_output`` is False."""
        kw = dict(other_kw)
        if kwargs is not None:
            kw.update(kwargs)
        device = next(self.unet.parameters()).device
        z = torch.randn((num_samples, self.in_channels, self.img_size, self.img_size), dtype=torch.float32, device=device)
        sampled = self.decode(z, cond=cond, num_steps=num_steps, start_step=start_step, verbose=verbose, **kw)
        return torch.clip(sampled, -1.0, 1.0) if clip_output else sampled
