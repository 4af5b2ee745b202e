"""The reference DDPM's default sampler, ``DDIMSampler`` (cflearn/modules/multimodal/diffusion/samplers/ddim.py, with the loop of
``ISampler.sample`` and the classifier-free guidance of ``UncondSamplerMixin``, samplers/schema.py:153-255), on the native
SD-UNet.  Each denoising step is one replay of a CUDA graph holding the UNet forward(s) and ``ops.ddim_step``, which advances
the latent, writes the stem's padded input and the timesteps of the next step, and advances the step counter on the device.

The per-step scalars follow the reference's dtypes: its tables are float64 (``alphas_cumprod`` as numpy made it), rounded to
fp32 when ``_register_temp_buffers`` fills them at the image's dtype; the update then runs in fp32 on the bf16 model output
(autocast's), with guidance as eager's bf16 tensor ops.  ``step_tables`` computes those fp32 scalars once per call, on the host,
with the reference's operations in its order, so the sampled bits are eager's.

Each step draws ``randn_like(image)`` from the current CUDA generator, as the reference does even at eta = 0; the draw is made
outside the graph, into a static buffer, so the generator ends each call where the reference's does.
"""
from __future__ import annotations

import math
from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from . import ops
from ._cabi import B200Error
from .unet import PAD_CHANNELS

KEYWORDS = ("eta", "discretize", "unconditional_cond", "unconditional_guidance_scale", "temperature", "noise_dropout",
            "quantize_denoised")


def ddim_timesteps(t: int, discretize: str, num_steps: int) -> np.ndarray:
    """DDIMQSampler.reset_buffers (ddim.py:38-53): the DDIM timesteps for a model with ``t`` timesteps.  "uniform" can give more
    than ``num_steps`` of them (the sampler uses the first ``num_steps``), and raises the reference's ValueError for a step count
    it cannot space over ``t``."""
    if num_steps < 1:
        raise ValueError(f"num_steps must be >= 1, got {num_steps}")
    if discretize == "uniform":
        span = t // (num_steps + int(t % num_steps == 0) - 1)
        q = np.array(list(range(0, t, span)) + [t - 1])
    elif discretize == "quad":
        q = (np.linspace(0, math.sqrt(t * 0.8), num_steps) ** 2).astype(int)
    else:
        raise ValueError(f"unrecognized discretize method '{discretize}' occurred")
    return np.minimum(q + 1, t - 1)


def step_tables(alphas_cumprod: Tensor, discretize: str, num_steps: int, eta: float) -> Tuple[Tensor, Tensor]:
    """The host tables of one sampling call, in step order (step i runs the reference's t_index = num_steps - 1 - i):
    (timesteps int64 [S], coef fp32 [S, 5] = {s1m, sqrt_a, sqrt_ap, c_dir, sigma}).  From the model's float64 ``alphas_cumprod``:
    the float64 tables of DDIMMixin._reset_buffers (ddim.py:241-264), each entry rounded to fp32 (_register_temp_buffers), then
    sqrt_a = sqrt(a), sqrt_ap = sqrt(a_prev) and c_dir = sqrt((1 - a_prev) - sigma^2) in fp32 (ddim.py:207, :234-238)."""
    if alphas_cumprod.dtype != torch.float64 or alphas_cumprod.dim() != 1:
        raise B200Error("step_tables: alphas_cumprod must be the float64 [T] table")
    q = ddim_timesteps(alphas_cumprod.shape[0], discretize, num_steps)
    ac = alphas_cumprod.cpu()
    alphas = ac[q]
    alphas_prev = torch.tensor([ac[0].item()] + ac[q[:-1]].tolist(), dtype=torch.float64)
    sigmas = eta * torch.sqrt((1.0 - alphas_prev) / (1.0 - alphas) * (1.0 - alphas / alphas_prev))
    s1m = torch.sqrt(1.0 - alphas)
    order = torch.arange(num_steps - 1, -1, -1)
    at, ap, sg = (v[order].to(torch.float32) for v in (alphas, alphas_prev, sigmas))
    coef = torch.stack([s1m[order].to(torch.float32), at.sqrt(), ap.sqrt(), (1.0 - ap - sg ** 2).sqrt(), sg], dim=1)
    return torch.from_numpy(q[order.numpy()].astype(np.int64)), coef.contiguous()


class _NoBucketCounts:
    """Hide the UNet's gradient arena from a sampling forward: the arena stays where it is (``ensure`` ran before), and the
    forward leaves the buckets' counts of a training step alone."""

    def __init__(self, unet: Any) -> None:
        self.unet, self.saved = unet, None

    def __enter__(self) -> None:
        self.saved, self.unet._grad_arena = self.unet._grad_arena, None

    def __exit__(self, *exc: Any) -> None:
        self.unet._grad_arena = self.saved


class DDIMSamplerB200:
    """``DDIMSampler`` for ``ddpm.DDPMB200``, with ``DDIMMixin``'s keywords.  ``eta``, ``discretize`` ("uniform" or "quad"),
    ``unconditional_cond`` (an encoded context [1, Tk, context_dim]), ``unconditional_guidance_scale``, ``temperature`` and
    ``default_steps`` are implemented; ``noise_dropout > 0`` and ``quantize_denoised`` raise ``NotImplementedError``.

    ``sample(z, cond=..., num_steps=...)`` runs the loop on the fp32 latent z [B, C, H, W] (CUDA) and returns the result.  The
    captured graph is kept for the next call; it is captured again when the batch, latent size, token counts, guidance, guidance
    scale, temperature or step count change, or when the UNet's parameters move.  ``release()`` drops it."""

    def __init__(self, model: Any, *, eta: float = 0.0, discretize: str = "uniform", unconditional_cond: Optional[Tensor] = None,
                 unconditional_guidance_scale: float = 1.0, temperature: float = 1.0, noise_dropout: float = 0.0,
                 quantize_denoised: bool = False, default_steps: int = 50) -> None:
        _refuse_options(noise_dropout, quantize_denoised)
        self.model = model
        self.eta, self.discretize = eta, discretize
        self.unconditional_cond = unconditional_cond
        self.unconditional_guidance_scale = unconditional_guidance_scale
        self.temperature = temperature
        self.noise_dropout, self.quantize_denoised = noise_dropout, quantize_denoised
        self.default_steps = default_steps
        self.last_bad_flag: Optional[Tensor] = None
        self._graph: Optional[torch.cuda.CUDAGraph] = None
        self._sig: Optional[tuple] = None
        self._buf: Dict[str, Tensor] = {}
        self.captures = 0  # graphs captured so far

    @property
    def sample_kwargs(self) -> Dict[str, Any]:
        return {k: getattr(self, k) for k in KEYWORDS}

    def release(self) -> None:
        """Drop the captured graph and its buffers."""
        self._graph, self._sig, self._buf = None, None, {}

    def sample(self, z: Tensor, *, cond: Optional[Any] = None, num_steps: Optional[int] = None, start_step: Optional[int] = None,
               verbose: bool = False, ref: Optional[Tensor] = None, ref_mask: Optional[Tensor] = None, **kwargs: Any) -> Tensor:
        what = "DDIMSamplerB200"
        if start_step:
            raise NotImplementedError(f"{what}: start_step > 0 is not supported (the reference reads tables left by an earlier call)")
        if ref is not None or ref_mask is not None:
            raise NotImplementedError(f"{what}: ref / ref_mask (inpainting) are not supported")
        if kwargs.get("step_callback") is not None:
            raise NotImplementedError(f"{what}: step_callback is not supported (the steps run as graph replays)")
        unknown = sorted(set(kwargs) - set(KEYWORDS) - {"step_callback", "ref_noise", "use_unified_ref_noise"})
        if unknown:
            raise TypeError(f"{what}: unexpected keyword arguments {unknown}")
        kw = self.sample_kwargs
        kw.update({k: v for k, v in kwargs.items() if k in KEYWORDS})
        _refuse_options(kw["noise_dropout"], kw["quantize_denoised"])
        if isinstance(cond, dict):
            raise NotImplementedError(f"{what}: dict conds are not supported (pass the encoded context as a tensor)")
        if num_steps is None:
            num_steps = self.default_steps
        m = self.model
        unet = m.unet
        C = m.in_channels
        if z.dim() != 4 or z.shape[1] != C or z.dtype != torch.float32 or not z.is_cuda or not z.is_contiguous():
            raise B200Error(f"{what}: z must be a contiguous CUDA fp32 latent [B, {C}, H, W]")
        B, _, H, W = z.shape
        ts, coef = step_tables(m.alphas_cumprod, kw["discretize"], num_steps, kw["eta"])
        if cond is not None and m.condition_model is not None:
            cond = m.get_cond(cond)
        uncond, scale = None, 0.0  # _reset_uncond_buffers: guidance only with a condition model
        if kw["unconditional_cond"] is not None and m.condition_model is not None:
            uncond, scale = m.get_cond(kw["unconditional_cond"]), float(kw["unconditional_guidance_scale"])
        if cond is None or uncond is None or scale == 1.0:
            mode, ctx, ctx_u = "plain", cond, None
        else:
            uncond = uncond.to(z.device).repeat_interleave(B, dim=0)
            if cond.shape[1] == uncond.shape[1]:
                mode, ctx, ctx_u = "equal", torch.cat([cond, uncond]), None
            else:
                mode, ctx, ctx_u = "unequal", cond, uncond
        unet.check_geometry(B * (2 if mode == "equal" else 1), H, W)
        grads = getattr(unet, "_grad_arena", None)
        if grads is not None:
            grads.arena.ensure()
        storage = tuple(p.data_ptr() for p in unet.parameters())
        spec = lambda t: None if t is None else (tuple(t.shape), t.dtype, t.device)  # noqa: E731
        sig = (B, C, H, W, num_steps, mode, spec(ctx), spec(ctx_u), scale, float(kw["temperature"]), z.device, storage)
        if self._graph is None or sig != self._sig:
            self._capture(sig, mode, ctx, ctx_u, scale, float(kw["temperature"]))
        b = self._buf
        b["x"].copy_(z)
        b["coef"].copy_(coef, non_blocking=False)
        b["ts"].copy_(ts, non_blocking=False)
        for name, t in (("ctx", ctx), ("ctx_u", ctx_u)):
            if t is not None:
                b[name].copy_(t)
        b["step"].zero_()
        b["bad"].zero_()
        copies = b["next_in"].shape[0] // B
        for k in range(copies):  # the first step's stem input and timesteps
            ops.pad_channels(b["x"], PAD_CHANNELS, out=b["next_in"][k * B:(k + 1) * B])
        b["next_ts"].fill_(int(ts[0]))
        for _ in range(num_steps):
            b["noise"].normal_()  # randn_like(image)'s draw, from the current generator
            self._graph.replay()
        self.last_bad_flag = b["bad"]
        return b["x"].clone()

    # internal

    def _capture(self, sig: tuple, mode: str, ctx: Optional[Tensor], ctx_u: Optional[Tensor], scale: float, temperature: float) -> None:
        self.release()
        B, C, H, W, S = sig[:5]
        dev = sig[10]
        copies = 2 if mode == "equal" else 1
        f32 = dict(dtype=torch.float32, device=dev)
        b = dict(x=torch.zeros((B, C, H, W), **f32), noise=torch.zeros((B, C, H, W), **f32), coef=torch.zeros((S, 5), **f32),
                 ts=torch.zeros(S, dtype=torch.int64, device=dev), step=torch.zeros(1, dtype=torch.int32, device=dev),
                 bad=torch.zeros(1, dtype=torch.int32, device=dev),
                 next_in=torch.zeros((copies * B, H, W, PAD_CHANNELS), dtype=torch.bfloat16, device=dev),
                 next_ts=torch.zeros(copies * B, dtype=torch.int64, device=dev))
        for name, t in (("ctx", ctx), ("ctx_u", ctx_u)):
            if t is not None:
                b[name] = t.detach().clone().contiguous()
        unet = self.model.unet

        def body() -> None:
            with torch.no_grad(), _NoBucketCounts(unet):
                if mode == "equal":
                    out = unet.forward_padded(b["next_in"], b["next_ts"], b["ctx"])
                    eps, eps_u = out[:B], out[B:]
                elif mode == "unequal":
                    eps = unet.forward_padded(b["next_in"], b["next_ts"], b["ctx"])
                    eps_u = unet.forward_padded(b["next_in"], b["next_ts"], b["ctx_u"])
                else:
                    eps, eps_u = unet.forward_padded(b["next_in"], b["next_ts"], b.get("ctx")), None
                ops.ddim_step(eps, eps_u, scale, b["x"], b["noise"], b["coef"], b["ts"], temperature, b["step"], b["bad"],
                              b["next_in"], b["next_ts"])

        # one eager run first (lazy kernel attributes, the allocator's pools); the buffers are reset by every sample call
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            body()
        torch.cuda.current_stream(dev).wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, capture_error_mode="thread_local"):
            body()
        self._graph, self._sig, self._buf = graph, sig, b
        self.captures += 1


def _refuse_options(noise_dropout: float, quantize_denoised: bool) -> None:
    if noise_dropout > 0:
        raise NotImplementedError("DDIMSamplerB200: noise_dropout > 0 is not supported")
    if quantize_denoised:
        raise NotImplementedError("DDIMSamplerB200: quantize_denoised (a VQ first stage) is not supported")
