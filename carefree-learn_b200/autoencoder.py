"""The first stage of latent diffusion: the decoder of the KL autoencoder (``AttentionAutoEncoderKL``,
cflearn/modules/cv/ae/kl.py:69-124, built by ae/common.py:12-72 with the ``AttentionDecoder`` of cv/decoder/attn.py) on the native
kernels, on CHANNELS-LAST bf16 activations:

    from_embedding      1x1 Conv2d on the latent zero-padded to 64 channels       ops.pad_channels, ops.gemm (bias epilogue)
    decoder.0           Conv2d(latent, C, 3, padding 1)                            unet.stem_conv (padded input)
    ResBlock            ResidualBlockWithTimeEmbedding without a time embedding    unet_blocks.res_block_fwd (eps 1e-6)
    SpatialAttention    GroupNorm(32, eps 1e-6) -> 1x1 q / k / v -> one head of   ``spatial_attention``: ops.groupnorm_silu_fwd,
                        width C over the H * W pixels -> 1x1 to_out, + input       ops.gemm, ops.softmax_rows
    Upsample            nearest 2x, then Conv2d(C, C, 3, padding 1)                ops.conv3x3_up2 (fused, per-image bias)
    head                GroupNorm(32, eps 1e-6) + SiLU, Conv2d(C, out, 3, pad 1)  ops.groupnorm_silu_fwd, unet.head_conv

Rounding points are eager's under bf16 autocast (oracle/ae_oracle.py::decode), with the UNet's one difference (DESIGN.md section
2): the 1x1 convolutions add their bias in fp32 and round once.  The attention rounds where its kernels hand over: S = Q K^T in
fp32, P = bf16(softmax(S / sqrt(C))), O = bf16(P V), then bf16(bf16(O Wo^T + bo) + x).

``AttentionAutoEncoderKLB200`` takes ``AttentionAutoEncoderKL``'s constructor keywords and holds its parameters under its names
(encoder, decoder, ``to_embedding``, ``from_embedding``), so a reference ``state_dict`` loads strictly in both directions.  Only
``decode`` runs: the encoder's asymmetrically padded stride-2 convolution has no kernel, and AE training is out of scope.
"""
from __future__ import annotations

import math
from typing import Any, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor, nn

from . import ops
from ._cabi import B200Error
from .attention import _bf, _check_cuda
from .unet import PAD_CHANNELS, head_conv, stem_conv
from .unet_blocks import MAX_CHANNELS, _bias_rows, res_block_fwd

NORM_EPS = 1.0e-6  # every GroupNorm of the autoencoder (residual.py:175 default, attn.py head, attentions.py:330 default)


# ------------------------------------------------------------------------------------------------------------------------------
# the parameter holders, in the reference's registration order (its state_dict order)
# ------------------------------------------------------------------------------------------------------------------------------
class _ResBlock(nn.Module):
    """``ResidualBlockWithTimeEmbedding(cin, cout, time_embedding_channels=0)``'s parameters (residual.py:154-209)."""

    def __init__(self, cin: int, cout: int) -> None:
        super().__init__()
        self.norm1 = nn.GroupNorm(32, cin, eps=NORM_EPS)
        self.conv1 = nn.Conv2d(cin, cout, 3, 1, 1)
        self.norm2 = nn.GroupNorm(32, cout, eps=NORM_EPS)
        self.conv2 = nn.Conv2d(cout, cout, 3, 1, 1)
        with torch.no_grad():  # zero_module(conv2), as the reference
            self.conv2.weight.zero_()
            self.conv2.bias.zero_()
        self.shortcut = nn.Conv2d(cin, cout, 1, 1, 0) if cin != cout else None

    def params(self) -> List[Optional[Tensor]]:
        """``res_block_fwd``'s P, without the time embedding."""
        s = self.shortcut
        return [self.norm1.weight, self.norm1.bias, self.conv1.weight, self.conv1.bias, None, None, self.norm2.weight, self.norm2.bias,
                self.conv2.weight, self.conv2.bias, None if s is None else s.weight, None if s is None else s.bias]


class _SpatialAttention(nn.Module):
    """``SpatialAttention(c)``'s parameters (core/attentions.py:330-348)."""

    def __init__(self, c: int) -> None:
        super().__init__()
        self.group_norm = nn.GroupNorm(32, c, eps=NORM_EPS)
        self.to_q = nn.Conv2d(c, c, 1, 1, 0)
        self.to_k = nn.Conv2d(c, c, 1, 1, 0)
        self.to_v = nn.Conv2d(c, c, 1, 1, 0)
        self.to_out = nn.Conv2d(c, c, 1, 1, 0)

    def params(self) -> List[Tensor]:
        return [self.group_norm.weight, self.group_norm.bias, self.to_q.weight, self.to_q.bias, self.to_k.weight, self.to_k.bias,
                self.to_v.weight, self.to_v.bias, self.to_out.weight, self.to_out.bias]


class _Resample(nn.Module):
    """The decoder's ``Upsample`` (conv 3x3, padding 1) or the encoder's ``Downsample`` (conv 3x3, stride 2, no padding) with
    ``with_conv=True`` (decoder/attn.py:18-31, encoder/attn.py:14-28)."""

    def __init__(self, c: int, down: bool) -> None:
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, 2, 0) if down else nn.Conv2d(c, c, 3, 1, 1)


def _head(c: int, out: int) -> List[nn.Module]:
    return [nn.GroupNorm(32, c, eps=NORM_EPS), nn.SiLU(), nn.Conv2d(c, out, 3, 1, 1)]


class _Encoder(nn.Module):
    """``AttentionEncoder``'s parameters (encoder/attn.py:31-94); it has no forward here."""

    def __init__(self, in_channels: int, inner: int, latent: int, mults: Sequence[int], num_res_blocks: int) -> None:
        super().__init__()
        blocks: List[nn.Module] = [nn.Conv2d(in_channels, inner, 3, 1, 1)]
        in_mults = (1,) + tuple(mults)
        c = inner
        for i, mult in enumerate(mults):
            c = inner * in_mults[i]
            for _ in range(num_res_blocks):
                blocks.append(_ResBlock(c, inner * mult))
                c = inner * mult
            if i != len(mults) - 1:
                blocks.append(_Resample(c, down=True))
        blocks += [_ResBlock(c, c), _SpatialAttention(c), _ResBlock(c, c)] + _head(c, latent)
        self.encoder = nn.Sequential(*blocks)


class _Decoder(nn.Module):
    """``AttentionDecoder``'s parameters (decoder/attn.py:34-104): ``decoder`` and ``head``."""

    def __init__(self, out_channels: int, inner: int, latent: int, mults: Sequence[int], num_res_blocks: int) -> None:
        super().__init__()
        c = inner * mults[-1]
        blocks: List[nn.Module] = [nn.Conv2d(latent, c, 3, 1, 1), _ResBlock(c, c), _SpatialAttention(c), _ResBlock(c, c)]
        for i in reversed(range(len(mults))):
            for _ in range(num_res_blocks + 1):
                blocks.append(_ResBlock(c, inner * mults[i]))
                c = inner * mults[i]
            if i != 0:
                blocks.append(_Resample(c, down=False))
        self.decoder = nn.Sequential(*blocks)
        self.head = nn.Sequential(*_head(c, out_channels))


class _Generator(nn.Module):
    """``EncoderDecoder`` (cv/common.py:338-349)."""

    def __init__(self, encoder: _Encoder, decoder: _Decoder) -> None:
        super().__init__()
        self.encoder = encoder
        self.decoder = decoder


# ------------------------------------------------------------------------------------------------------------------------------
# the attention
# ------------------------------------------------------------------------------------------------------------------------------
def spatial_attention(x: Tensor, P: Sequence[Tensor], eps: float = NORM_EPS) -> Tensor:
    """``SpatialAttention.forward`` (core/attentions.py:350-370) on x, contiguous bf16 [B, H, W, C] (C % 8 == 0); P: group_norm
    weight / bias, to_q, to_k, to_v, to_out weight / bias (the reference's shapes).  Returns bf16 [B, H, W, C].

    One GEMM makes q, k and v for every pixel ([B H W, 3C]).  Per image, S = Q K^T is a GEMM on transposed copies of q and k
    into an fp32 [T, T] buffer.  The fp32-output epilogue (``EPI_PARTIAL_F32``) is compiled for MN-major operands only, so the
    lda = 3C row views of qkv cannot feed it directly; the copy (2 T C bf16 per image, 8 MiB written and read at T = 4,096 and
    C = 512) is the cost of that restriction, small next to S and P (96 MiB, each written once and read once).
    ``ops.softmax_rows`` makes P with the scale 1 / sqrt(C) of ``F.scaled_dot_product_attention``, and O = P V reads v in place
    as an MN-major operand.  to_out and the residual are one GEMM with the bf16 residual epilogue."""
    gn_w, gn_b, wq, bq, wk, bk, wv, bv, wo, bo = P
    B, H, W, C = x.shape
    T = H * W
    y, _, _ = ops.groupnorm_silu_fwd(x.view(B, T, C), gn_w.float().contiguous(), gn_b.float().contiguous(), eps, silu=False)
    qkv = ops.gemm(y.view(B * T, C), _bf(torch.cat([wq, wk, wv]).reshape(3 * C, C)), bias=_bf(torch.cat([bq, bk, bv])))
    s = torch.empty((1, T, T), dtype=torch.float32, device=x.device)
    p = torch.empty((T, T), dtype=torch.bfloat16, device=x.device)
    o = torch.empty((B * T, C), dtype=torch.bfloat16, device=x.device)
    scale = 1.0 / math.sqrt(C)
    for b in range(B):
        rows = qkv[b * T:(b + 1) * T]
        qk_t = rows[:, :2 * C].t().contiguous()  # [2C, T]: q^T, then k^T (MN-major operands of the fp32-output epilogue)
        ops.gemm(qk_t[:C], qk_t[C:], a_mn_major=True, b_mn_major=True, epilogue=ops.EPI_PARTIAL_F32, out0=s)
        ops.softmax_rows(s[0], scale, out=p)
        ops.gemm(p, rows[:, 2 * C:], b_mn_major=True, out0=o[b * T:(b + 1) * T])
    out = ops.gemm(o, _bf(wo.reshape(C, C)), bias=_bf(bo), epilogue=ops.EPI_BIAS_RESID_BF16, aux=x.view(B * T, C))
    return out.view(B, H, W, C)


# ------------------------------------------------------------------------------------------------------------------------------
# the module
# ------------------------------------------------------------------------------------------------------------------------------
def _conv_grid(h: int, w: int) -> None:
    """The tile rule of the forward 3x3 convolutions (``ops.conv3x3``, and ``ops.conv3x3_up2`` on its input grid):
    128-pixel tiles of whole rows, or of one row when the width is 128 times a power of 2."""
    if w > 128 and w % 128 == 0 and (w // 128) & (w // 128 - 1) == 0:
        return
    if w > 128 or 128 % w != 0:
        raise B200Error(f"the width {w} must divide 128 or be 128 times a power of 2 (conv3x3 tiles of 128 pixels)")
    hb = min(h, 128 // w)
    if h % hb != 0 or 128 % (w * hb) != 0:
        raise B200Error(f"the height {h} must be a multiple of 128 / {w} (conv3x3 tiles of 128 pixels of whole rows)")


class AttentionAutoEncoderKLB200(nn.Module):
    """Drop-in for cflearn's ``AttentionAutoEncoderKL`` that decodes on the native kernels (fp32 parameters, bf16 activations;
    CUDA only).

    ``decode(inputs)``: ``inputs`` is a latent or anything with ``.z`` (and optionally ``.no_head`` / ``.apply_tanh``, as the
    reference's ``DecoderInputs``); the latent is fp32 or bf16 [B, embedding_channels, h, w] on the parameters' CUDA device, in
    either memory format.  Returns bf16 [B, out_channels, H, W] (``no_head``: the pre-head features [B, C, H, W]) with
    channels-last strides, without autograd.  A latent size the kernels cannot tile raises one ``B200Error`` before any launch,
    naming the level (``check_geometry``).  Everything that needs the encoder raises ``NotImplementedError``."""

    def __init__(self, img_size: int, in_channels: int, out_channels: int, inner_channels: int, latent_channels: int,
                 channel_multipliers: Tuple[int, ...], *, embedding_channels: int, num_res_blocks: int,
                 attention_resolutions: Tuple[int, ...] = (), dropout: float = 0.0, resample_with_conv: bool = True,
                 attention_type: str = "spatial", apply_tanh: bool = False) -> None:
        super().__init__()
        what = "AttentionAutoEncoderKLB200"
        refused = [(len(attention_resolutions) > 0, "attention_resolutions (attention outside the middle block)"),
                   (dropout > 0.0, "dropout > 0"), (not resample_with_conv, "resample_with_conv=False"),
                   (attention_type != "spatial", f"attention_type={attention_type!r} (only 'spatial')"), (apply_tanh, "apply_tanh")]
        for bad, option in refused:
            if bad:
                raise NotImplementedError(f"{what}: {option} is not supported")
        mults = tuple(channel_multipliers)
        if latent_channels > PAD_CHANNELS or embedding_channels > PAD_CHANNELS or out_channels > PAD_CHANNELS:
            raise NotImplementedError(f"{what}: latent, embedding and out channels must be at most {PAD_CHANNELS} (the padded "
                                      "convolutions)")
        self.z_size = img_size // 2 ** (len(mults) - 1)
        self.img_size, self.in_channels, self.out_channels = img_size, in_channels, out_channels
        self.inner_channels, self.latent_channels, self.embedding_channels = inner_channels, latent_channels, embedding_channels
        self.channel_multipliers, self.num_res_blocks = mults, num_res_blocks
        self.generator = _Generator(_Encoder(in_channels, inner_channels, 2 * latent_channels, mults, num_res_blocks),
                                    _Decoder(out_channels, inner_channels, latent_channels, mults, num_res_blocks))
        self.to_embedding = nn.Conv2d(2 * latent_channels, 2 * embedding_channels, 1)
        self.from_embedding = nn.Conv2d(embedding_channels, latent_channels, 1)

    # ---- what needs the encoder ----------------------------------------------------------------------------------------------
    def _no_encoder(self, name: str) -> None:
        raise NotImplementedError(f"AttentionAutoEncoderKLB200: {name} is not supported (the encoder's (0, 1, 0, 1)-padded stride-2 "
                                  "convolution has no native kernel; only decode runs)")

    def encode(self, net: Tensor) -> Any:
        self._no_encoder("encode")

    def forward(self, net: Tensor, **kwargs: Any) -> Any:
        self._no_encoder("forward")

    def get_results(self, net: Tensor, **kwargs: Any) -> Any:
        self._no_encoder("get_results")

    def reconstruct(self, net: Tensor, **kwargs: Any) -> Any:
        self._no_encoder("reconstruct")

    # ---- decode --------------------------------------------------------------------------------------------------------------
    def check_geometry(self, B: int, h: int, w: int) -> None:
        """Raise one ``B200Error`` naming the first decoder level (from the latent up) whose grid the kernels cannot tile.  Level
        i is the reference's loop index (decoder/attn.py:76): channel_multipliers[i], at the latent size times 2^(n - 1 - i)."""
        n = len(self.channel_multipliers)
        if B <= 0 or h <= 0 or w <= 0:
            raise B200Error(f"AttentionAutoEncoderKLB200: a {B} x {h} x {w} latent batch is empty")
        for i in reversed(range(n)):
            H, W = h << (n - 1 - i), w << (n - 1 - i)
            try:
                for c in {self.inner_channels * self.channel_multipliers[j] for j in (i, min(i + 1, n - 1))}:
                    if c % 64 != 0 or c > MAX_CHANNELS:
                        raise B200Error(f"{c} channels must be a multiple of 64, at most {MAX_CHANNELS} (conv3x3 / GroupNorm kernels)")
                _conv_grid(H, W)
                if B * H * W * (16 if i != 0 else 1) > 0x7FFFFFFF:  # (the upsampling convolution's four classes of 2H x 2W rows)
                    raise B200Error(f"{B} images of {H} x {W} are too many pixels for one convolution")
            except B200Error as err:
                raise B200Error(f"AttentionAutoEncoderKLB200: level {i} ({H} x {W} of a {h} x {w} latent): {err}") from None

    @torch.no_grad()
    def decode(self, inputs: Any) -> Tensor:
        what = "AttentionAutoEncoderKLB200"
        if isinstance(inputs, Tensor):
            z, no_head, apply_tanh = inputs, False, None
        else:
            z, no_head, apply_tanh = inputs.z, bool(getattr(inputs, "no_head", False)), getattr(inputs, "apply_tanh", None)
        if apply_tanh:
            raise NotImplementedError(f"{what}: apply_tanh is not supported")
        if not isinstance(z, Tensor) or z.dim() != 4 or z.shape[1] != self.embedding_channels or z.dtype not in (torch.float32, torch.bfloat16):
            raise B200Error(f"{what}: the latent must be an fp32 or bf16 tensor [B, {self.embedding_channels}, h, w]")
        B, _, h, w = z.shape
        self.check_geometry(B, h, w)
        _check_cuda(what, z)
        dev = self.from_embedding.weight.device
        if z.device != dev:
            raise B200Error(f"{what}: the latent is on {z.device}, the parameters on {dev}")
        if not (z.is_contiguous() or z.is_contiguous(memory_format=torch.channels_last)):
            z = z.contiguous()
        x = self._from_embedding(z)
        for block in self.generator.decoder.decoder:
            if isinstance(block, nn.Conv2d):  # decoder.0 on the padded latent
                x = stem_conv(x, block.weight, block.bias, padded=True)[0]
            elif isinstance(block, _ResBlock):
                x = res_block_fwd(x, None, block.params(), NORM_EPS)[0]
            elif isinstance(block, _SpatialAttention):
                x = spatial_attention(x, block.params())
            else:
                conv = block.conv
                x = ops.conv3x3_up2(x, ops.pack_conv3x3_weight(conv.weight), epilogue=ops.EPI_BIAS_ADD_PER_IMAGE_BF16,
                                    aux=_bias_rows(conv.bias, B))
        if no_head:
            return x.permute(0, 3, 1, 2)
        gn, conv = self.generator.decoder.head[0], self.generator.decoder.head[2]
        _, H, W, C = x.shape
        y, _, _ = ops.groupnorm_silu_fwd(x.view(B, H * W, C), gn.weight.float().contiguous(), gn.bias.float().contiguous(), gn.eps)
        return head_conv(y.view(B, H, W, C), conv.weight, conv.bias)[0].permute(0, 3, 1, 2)

    def _from_embedding(self, z: Tensor) -> Tensor:
        """The 1x1 ``from_embedding`` of z as one GEMM on its 64-channel-padded bf16 cast: bf16 [B, h, w, 64], channels >=
        latent_channels zero (the padded stem's input)."""
        B, E, h, w = z.shape
        L = self.latent_channels
        x = ops.pad_channels(z, PAD_CHANNELS)
        wt = F.pad(self.from_embedding.weight.reshape(L, E), (0, PAD_CHANNELS - E, 0, PAD_CHANNELS - L))
        out = ops.gemm(x.view(B * h * w, PAD_CHANNELS), _bf(wt), bias=_bf(F.pad(self.from_embedding.bias, (0, PAD_CHANNELS - L))))
        return out.view(B, h, w, PAD_CHANNELS)
