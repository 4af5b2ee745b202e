"""First SD-v1.5 UNet building block on the native kernels (BASELINE.json configs[4]; SURVEY.md 8f row N3): the forward of
``ResidualBlockWithTimeEmbedding`` (cflearn/modules/core/convs/residual.py:154-253) as ``UNetDiffuser`` builds it
(cflearn/modules/multimodal/diffusion/unet.py:151-161), on CHANNELS-LAST bf16 activations:

    GroupNorm(32, eps 1e-5) -> SiLU -> conv3x3          b200_groupnorm_silu_fwd, b200_conv3x3_nhwc_bf16 (implicit GEMM)
    + Linear(SiLU(time_embedding))[b, c]                b200_gemm_bf16 (+ the bf16 elementwise glue eager runs)
    GroupNorm -> SiLU -> Dropout(0) -> conv3x3
    + shortcut (1x1 conv = plain GEMM on [B*H*W, Cin] when the width changes), clamp to the dtype's finite range

Rounding points are eager's under bf16 autocast (oracle/unet_oracle.py::res_block): GroupNorm / SiLU in fp32 with one bf16
rounding at the conv input, every conv / Linear output rounded to bf16, the two residual adds in bf16.  This is the
forward only.  The UNet's attention (``attention.CrossAttentionB200``) and its SpatialTransformer with GEGLU
(``spatial_transformer.SpatialTransformerB200``) train natively; the ResBlock backward, up / down-sampling and the
module / training step are the open part of row N3.
"""
from __future__ import annotations

from typing import Dict

import torch
from torch import Tensor

from . import ops
from ._cabi import B200Error


def res_block_forward(sd: Dict[str, Tensor], prefix: str, net: Tensor, time_net: Tensor) -> Tensor:
    """``net``: bf16 [B, H, W, Cin] channels-last; ``time_net``: bf16 [B, time_dim]; ``sd``: the reference's parameters of the
    block under ``prefix`` (fp32, NCHW conv weights).  Returns bf16 [B, H, W, Cout]."""
    if not net.is_cuda or net.dtype != torch.bfloat16 or net.dim() != 4:
        raise B200Error("res_block_forward: bf16 CUDA activations [B, H, W, C] (there is no CPU fallback)")
    p = prefix
    B, H, W, Cin = net.shape
    w1, w2 = sd[p + "conv1.weight"], sd[p + "conv2.weight"]
    Cout = w1.shape[0]
    bf = lambda t: t.to(torch.bfloat16).contiguous()  # noqa: E731  (autocast's per-op weight casts)
    y, _, _ = ops.groupnorm_silu_fwd(net.reshape(B, H * W, Cin), sd[p + "norm1.weight"].float().contiguous(), sd[p + "norm1.bias"].float().contiguous(), 1e-5)
    h = ops.conv3x3(y.view(B, H, W, Cin), ops.pack_conv3x3_weight(w1), bf(sd[p + "conv1.bias"]))
    # time embedding: F.silu on the bf16 tensor (fp32 maths, bf16 result), then a bf16 Linear
    t_act = torch.nn.functional.silu(time_net)
    t = ops.gemm(t_act.contiguous(), bf(sd[p + "time_embedding.weight"]), bias=bf(sd[p + "time_embedding.bias"]))  # [B, Cout]
    h = h + t[:, None, None, :]                                                                                     # bf16 + bf16 -> bf16
    y2, _, _ = ops.groupnorm_silu_fwd(h.reshape(B, H * W, Cout), sd[p + "norm2.weight"].float().contiguous(), sd[p + "norm2.bias"].float().contiguous(), 1e-5)
    h2 = ops.conv3x3(y2.view(B, H, W, Cout), ops.pack_conv3x3_weight(w2), bf(sd[p + "conv2.bias"]))
    inp = net
    if p + "shortcut.weight" in sd:  # 1x1 convolution on channels-last activations == a plain GEMM over the pixels
        ws = sd[p + "shortcut.weight"]
        inp = ops.gemm(net.reshape(B * H * W, Cin), bf(ws.reshape(ws.shape[0], Cin)), bias=bf(sd[p + "shortcut.bias"])).view(B, H, W, Cout)
    out = inp + h2
    fi = torch.finfo(out.dtype)
    return out.clamp(fi.min, fi.max)
