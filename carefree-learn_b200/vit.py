"""H100-native (sm_90a) drop-in for the reference's ViT encoder / classifier training step.

``ViTEncoderB200`` mirrors ``cflearn.modules.cv.encoder.transformer.ViTEncoder`` (transformer.py:17-100): same
constructor keywords, same ``state_dict`` keys and shapes (SURVEY.md 8b), same forward signature, plus the
``.encode`` method ``cv_clf`` expects (cv/classifier/vanilla.py:57; SURVEY finding 4).  ``VanillaClassifierB200``
mirrors ``VanillaClassifier`` (vanilla.py:16-66) with the ViT encoder and returns ``{"predictions": logits}``.

Everything between the input image and the logits -- and its whole backward -- runs in hand-written sm_90a kernels
through the C-ABI (``ops``); autograd sees ONE ``torch.autograd.Function`` per module.  Numerics follow the
reference under ``torch.autocast(bf16)``: fp32 residual stream / LayerNorm / softmax / loss, bf16 GEMM operands with
fp32 accumulation, bf16 rounding at exactly the points eager rounds (see DESIGN.md "rounding points").

Parameters live in ONE flat fp32 arena (each ``nn.Parameter`` is a view), shadowed by a bf16 arena refreshed once
per step and a flat fp32 gradient arena that the data-parallel reducer (``dp.py``) all-reduces in buckets while
backward is still running.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple, Union

import torch
import torch.nn as nn
from torch import Tensor

from . import ops
from ._cabi import B200Error
from .arena import ArenaModule, ParamArena, register_dotted

PREDICTIONS_KEY = "predictions"  # cflearn/constants.py:6
LATENT_KEY = "latent"


# -----------------------------------------------------------------------------------------------------------------
# geometry / spec
# -----------------------------------------------------------------------------------------------------------------
class ViTGeometry:
    def __init__(self, *, img_size: int, patch_size: int, in_channels: int, latent_dim: int, num_layers: int,
                 ff_ratio: float, eps: float, num_classes: Optional[int], conv_bias: bool = True,
                 embedding_norm_eps: Optional[float] = None, norm_after_head: bool = False,
                 output_dim: Optional[int] = None, activation: str = "GELU",
                 context_length: Optional[int] = None, causal: bool = False):
        if latent_dim % 64 != 0:
            raise NotImplementedError("latent_dim must be a multiple of 64 (head dim 64, transformer.py:61)")
        # token mode (TeTEncoder, nlp/encoder/transformer.py:16-99): the input is an embedded sequence [B, T, D]; no patch
        # stem, no head token; the head is PreNorm(Identity) = LayerNorm over every token
        self.tokens = context_length is not None
        self.causal = causal
        if not self.tokens and (patch_size % 16 != 0 or img_size % patch_size != 0):
            raise NotImplementedError("patch_size must be a multiple of 16 dividing img_size")
        self.img, self.patch, self.cin, self.D, self.L = img_size, patch_size, in_channels, latent_dim, num_layers
        self.H = latent_dim // 64
        self.FF = int(round(latent_dim * ff_ratio))
        self.np = 0 if self.tokens else (img_size // patch_size) ** 2
        self.T = int(context_length) if self.tokens else self.np + 1
        self.eps = eps
        self.C = num_classes
        # the options CLIP's vision tower switches on (multimodal/clip.py:121-135)
        self.conv_bias = conv_bias                    # to_patches_config={"bias": False}
        self.emb_eps = embedding_norm_eps             # embedding_norm=nn.LayerNorm(D, eps): LN right after cls + pos-enc
        self.norm_after_head = norm_after_head        # head_norm applied to the cls token (same maths, other key names)
        self.out_dim = output_dim                     # `net @ output_projection`  [D, out_dim], no bias
        self.quick_gelu = activation == "quick_gelu"  # feedforward_kwargs={"activation": "quick_gelu"}
        if activation not in ("GELU", "quick_gelu"):
            raise NotImplementedError(f"FeedForward activation {activation!r} is outside the fused path (GELU, quick_gelu)")
        if output_dim is not None and (output_dim % 8 != 0 or num_classes is not None):
            raise NotImplementedError("output_dim must be a multiple of 8 and cannot be combined with a classifier head")
        if self.T > ops.ATTENTION_MAX_T:
            raise NotImplementedError(f"sequence length > {ops.ATTENTION_MAX_T} tokens is not supported by the fused attention")

    @property
    def head_norm_key(self) -> str:  # mixed_stacks/api.py:383-395: PreNorm(head) vs head then head_norm
        return "encoder.head_norm." if self.norm_after_head else "encoder.head.norms.0."

    def _groups(self) -> List[Tuple[Union[int, str], List[Tuple[str, Tuple[int, ...]]]]]:
        """The parameters in the reference's state_dict order (a module's own parameters precede its sub-modules'),
        in runs labelled with the point of ``ViTEngine.encoder_backward`` after which their gradients are complete."""
        d, p, c, ff = self.D, self.patch, self.cin, self.FF
        out: List[Tuple[Union[int, str], List[Tuple[str, Tuple[int, ...]]]]] = []
        if self.out_dim is not None:  # a parameter of the encoder itself: first in state_dict order, written with the tail
            out.append(("tail", [("output_projection", (d, self.out_dim))]))
        if self.tokens:
            stem = [("encoder.pos_encoding.pos_encoding", (1, self.T, d))]
        else:
            stem = [("to_patches.projection.weight", (d, c, p, p))]
            if self.conv_bias:
                stem.append(("to_patches.projection.bias", (d,)))
            stem += [("encoder.head_token", (1, 1, d)), ("encoder.pos_encoding.pos_encoding", (1, self.T, d))]
        if self.emb_eps is not None:
            stem += [("encoder.embedding_norm.weight", (d,)), ("encoder.embedding_norm.bias", (d,))]
        out.append(("stem", stem))
        for i in range(self.L):
            b = f"encoder.mixing_blocks.{i}."
            out.append((i, [
                (b + "token_norm.weight", (d,)), (b + "token_norm.bias", (d,)),
                (b + "token_mixing.net.in_w", (3 * d, d)), (b + "token_mixing.net.qkv_bias", (3 * d,)),
                (b + "token_mixing.net.out_linear.linear.weight", (d, d)), (b + "token_mixing.net.out_linear.linear.bias", (d,)),
                (b + "channel_norm.weight", (d,)), (b + "channel_norm.bias", (d,)),
                (b + "channel_mixing.net.0.linear.weight", (ff, d)), (b + "channel_mixing.net.0.linear.bias", (ff,)),
                (b + "channel_mixing.net.3.linear.weight", (d, ff)), (b + "channel_mixing.net.3.linear.bias", (d,)),
            ]))
        tail = [(self.head_norm_key + "weight", (d,)), (self.head_norm_key + "bias", (d,))]
        if self.C is not None:
            tail += [("head.linear.weight", (self.C, d)), ("head.linear.bias", (self.C,))]
        out.append(("tail", tail))
        return out

    def spec(self) -> List[Tuple[str, Tuple[int, ...]]]:
        return [kv for _, run in self._groups() for kv in run]

    def buckets(self) -> Dict[Union[int, str], List[List[str]]]:
        """Gradient all-reduce buckets: for each point where ``encoder_backward`` calls ``reducer.ready``, the keys of
        each contiguous run of the arena that is complete there."""
        out: Dict[Union[int, str], List[List[str]]] = {}
        for point, run in self._groups():
            out.setdefault(point, []).append([k for k, _ in run])
        return out


def _init_param(key: str, shape: Tuple[int, ...]) -> Tensor:
    """Reference initialisation: trunc_normal(0.02) for Linear / in_w / cls / pos (mixed_stacks/api.py:205,405-417;
    attentions.py:108-110), zero biases, LayerNorm 1/0, xavier_normal conv with gain `gain / sqrt 2` where the Conv2d
    default is gain = sqrt 2, i.e. 1.0 (convs/basic.py:56,94-97; pinned live by tests/test_host_logic.py)."""
    if key.endswith("norm.weight") or key.endswith("norms.0.weight"):
        return torch.ones(shape)
    if key == "output_projection":  # cv/encoder/transformer.py:81-82
        return (shape[0] ** -0.5) * torch.randn(shape)
    if key.endswith("bias"):
        return torch.zeros(shape)
    if key == "to_patches.projection.weight":
        t = torch.empty(shape)
        nn.init.xavier_normal_(t, 1.0)
        return t
    return nn.init.trunc_normal_(torch.empty(shape), std=0.02)


# -----------------------------------------------------------------------------------------------------------------
# the engine: forward / backward of the whole stack on raw buffers
# -----------------------------------------------------------------------------------------------------------------
class _Saved:
    __slots__ = ("B", "cols", "blocks", "net_last", "head_mean", "head_rstd", "enc_bf16", "emb_in", "emb_mean", "emb_rstd")


class _Scratch:
    """One block's intermediates, reused by every block of a forward that keeps nothing for backward.  ``mean`` / ``rstd``
    and ``lse`` receive what only backward would read; ``mid`` is the second buffer of the fp32 residual stream."""

    def __init__(self, geo: ViTGeometry, B: int, device: torch.device):
        M, D = B * geo.T, geo.D
        bf16, f32 = dict(dtype=torch.bfloat16, device=device), dict(dtype=torch.float32, device=device)
        self.ln = torch.empty((M, D), **bf16)
        self.mean = torch.empty(M, **f32)
        self.rstd = torch.empty(M, **f32)
        self.qkv = torch.empty((M, 3 * D), **bf16)
        self.attn = torch.empty((M, D), **bf16)
        self.lse = torch.empty((B, geo.H, geo.T), **f32)
        self.mid = torch.empty((M, D), **f32)
        self.h = torch.empty((M, geo.FF), **bf16)
        self.act = torch.empty((M, geo.FF), **bf16)


class ViTEngine:
    def __init__(self, geo: ViTGeometry, arena: ParamArena):
        self.geo = geo
        self.arena = arena
        self.reducer = None  # set by dp.attach_reducer / dp.attach_native_reducers
        # uint8 [B, S, S, C] inputs: {"division": 255.0, "mean": [...], "std": [...]} = the reference's static_normalize +
        # imagenet / affine normalisation blocks (data/blocks/cv/normalize.py); None: division by 255 only
        self.input_pipeline: Optional[Dict[str, Any]] = None
        self.shrink_next = 0  # SMs to leave free for an in-flight bucket all-reduce when launching the next GEMM (dp.py)

    def buckets(self) -> Dict[Union[int, str], List[List[str]]]:
        """The gradient exchange's buckets (``ViTGeometry.buckets``): this engine is an exchange site of its model."""
        return self.geo.buckets()

    # ---- stages (also the units of the teacher-forced parity tests, tests/test_taps_gpu.py) --------------------
    def stem_forward(self, x: Tensor) -> Tuple[Optional[Tensor], Tensor]:
        """image [B, C, S, S] fp32 (or embedded tokens [B, T, D]) -> (im2col matrix or None, fp32 tokens [B*T, D])."""
        g, A = self.geo, self.arena
        B, T, D = x.shape[0], g.T, g.D
        if g.tokens:  # TeTEncoder.forward -> pre_process (api.py:419-438 without head token): x + pos
            return None, ops.add_pos(x, A.p("encoder.pos_encoding.pos_encoding"), B, T, D).view(B * T, D)
        if x.dtype == torch.uint8:  # raw HWC batch: the host-side normalise / transpose / float32 / H2D chain fused into the gather
            pipe = self.input_pipeline or {}
            cols = ops.patch_im2col_u8(x, g.patch, pipe.get("division", 255.0), pipe.get("mean"), pipe.get("std"))
        else:
            cols = ops.patch_im2col(x, g.patch)
        # F.conv2d with a bias on CUDA is TWO roundings in eager: ATen's cuDNN path produces the bf16 convolution output and
        # then runs `output.add_(bias)` on the bf16 tensor (aten/native/Convolution.cpp) -- unlike F.linear, whose bias is
        # fused before the single rounding (tools/probe_conv_bias.py).  So the bias is added after the GEMM's rounding.
        patch = ops.gemm(cols, A.w("to_patches.projection.weight").view(D, -1))
        net = ops.assemble_tokens(patch, A.p("encoder.head_token"), A.p("encoder.pos_encoding.pos_encoding"), B, g.np, D,
                                  conv_bias=A.w("to_patches.projection.bias") if g.conv_bias else None).view(B * T, D)
        return cols, net

    def block_forward(self, i: int, net: Tensor, B: int, scratch: Optional[_Scratch] = None) -> Tuple[Tensor, Tuple[Tensor, ...]]:
        """MixingBlock._pre_norm_forward (mixed_stacks/api.py:130-158) on the fp32 residual stream [B*T, D].  ``scratch``: every
        intermediate goes to its buffers and the block's output overwrites ``net`` (the same kernels, so the same bits); the
        returned tuple then aliases buffers the next block overwrites."""
        g, A = self.geo, self.arena
        T, D, M = g.T, g.D, B * g.T
        b = f"encoder.mixing_blocks.{i}."
        s = scratch
        epi_act = ops.EPI_BIAS_QGELU_BF16 if g.quick_gelu else ops.EPI_BIAS_GELU_BF16
        ln1, mean1, rstd1 = ops.layernorm_fwd(net, A.p(b + "token_norm.weight"), A.p(b + "token_norm.bias"), g.eps, rows=M, dim=D, ld_x=D,
                                              y=s and s.ln, mean=s and s.mean, rstd=s and s.rstd)
        qkv = ops.gemm(ln1, A.w(b + "token_mixing.net.in_w"), bias=A.w(b + "token_mixing.net.qkv_bias"), out0=s and s.qkv)
        attn, lse = ops.attention_fwd(qkv, B, T, g.H, causal=g.causal, out=s and s.attn, lse=s and s.lse)
        mid = ops.gemm(attn, A.w(b + "token_mixing.net.out_linear.linear.weight"), bias=A.w(b + "token_mixing.net.out_linear.linear.bias"),
                       epilogue=ops.EPI_BIAS_RESID_F32, aux=net, out0=s and s.mid)
        ln2, mean2, rstd2 = ops.layernorm_fwd(mid, A.p(b + "channel_norm.weight"), A.p(b + "channel_norm.bias"), g.eps, rows=M, dim=D, ld_x=D,
                                              y=s and s.ln, mean=s and s.mean, rstd=s and s.rstd)
        act = s.act if s else torch.empty((M, g.FF), dtype=torch.bfloat16, device=net.device)
        h = ops.gemm(ln2, A.w(b + "channel_mixing.net.0.linear.weight"), bias=A.w(b + "channel_mixing.net.0.linear.bias"),
                     epilogue=epi_act, out1=act, out0=s and s.h)
        out = ops.gemm(act, A.w(b + "channel_mixing.net.3.linear.weight"), bias=A.w(b + "channel_mixing.net.3.linear.bias"),
                       epilogue=ops.EPI_BIAS_RESID_F32, aux=mid, out0=s and net)
        return out, (net, mean1, rstd1, ln1, qkv, attn, lse, mid, mean2, rstd2, ln2, h, act)

    def block_backward(self, i: int, saved: Tuple[Tensor, ...], dnet: Tensor, dnet_bf: Tensor, G: Tensor, B: int,
                       *, ff2_bias_done: bool = True, next_ff2_bias: bool = True, accumulate: bool = False) -> None:
        """Backward of block ``i``.  ``dnet`` (fp32) / ``dnet_bf`` (its bf16 rounding) hold the gradient of the block's
        output and are OVERWRITTEN with the gradient of its input.  ``ff2_bias_done``: this block's FF2 bias gradient was
        already emitted by the producer of ``dnet_bf``; ``next_ff2_bias``: emit block ``i-1``'s from the last LayerNorm
        backward here (both fusions remove a pass over the [M, D] gradient).  ``accumulate``: the parameter gradients are
        added to ``G`` instead of overwriting it."""
        g, A = self.geo, self.arena
        T, D, M = g.T, g.D, B * g.T
        dev = dnet.device
        b = f"encoder.mixing_blocks.{i}."
        net, mean1, rstd1, ln1, qkv, attn, lse, mid, mean2, rstd2, ln2, h, act = saved
        if not ff2_bias_done:
            ops.colsum(dnet_bf, A.g(b + "channel_mixing.net.3.linear.bias", G), accumulate=accumulate)
        # FeedForward: net_out = mid + W2 gelu(W1 ln2 + b1) + b2
        ff1_bias = A.g(b + "channel_mixing.net.0.linear.bias", G)
        shrink, self.shrink_next = self.shrink_next, 0  # the previous block's bucket is being all-reduced right now
        dh = ops.gemm(dnet_bf, A.w(b + "channel_mixing.net.3.linear.weight"), b_mn_major=True,
                      epilogue=ops.EPI_DQGELU_BF16 if g.quick_gelu else ops.EPI_DGELU_BF16, aux=h,
                      max_ctas=(ops.num_sms() - shrink) if shrink else 0)
        ops.wgrad(dnet_bf, act, A.g(b + "channel_mixing.net.3.linear.weight", G), accumulate=accumulate)
        dln2 = ops.gemm(dh, A.w(b + "channel_mixing.net.0.linear.weight"), b_mn_major=True)
        ops.wgrad(dh, ln2, A.g(b + "channel_mixing.net.0.linear.weight", G), accumulate=accumulate)
        ops.colsum(dh, ff1_bias, accumulate=accumulate)
        dmid = torch.empty((M, D), dtype=torch.float32, device=dev)
        dmid_bf = torch.empty((M, D), dtype=torch.bfloat16, device=dev)
        ops.layernorm_bwd(dln2, mid, A.p(b + "channel_norm.weight"), mean2, rstd2, rows=M, dim=D, ld_x=D, dres=dnet,
                          dx_out=dmid, ld_dx=D, dx_bf16=dmid_bf,
                          dgamma=A.g(b + "channel_norm.weight", G), dbeta=A.g(b + "channel_norm.bias", G),
                          dx_colsum=A.g(b + "token_mixing.net.out_linear.linear.bias", G), accumulate=accumulate)
        # attention: mid = net + Wo attn + bo
        dattn = ops.gemm(dmid_bf, A.w(b + "token_mixing.net.out_linear.linear.weight"), b_mn_major=True)
        ops.wgrad(dmid_bf, attn, A.g(b + "token_mixing.net.out_linear.linear.weight", G), accumulate=accumulate)
        dqkv = ops.attention_bwd(qkv, attn, dattn, lse, B, T, g.H, causal=g.causal, dbias=A.g(b + "token_mixing.net.qkv_bias", G),
                                 accumulate=accumulate)
        dln1 = ops.gemm(dqkv, A.w(b + "token_mixing.net.in_w"), b_mn_major=True)
        ops.wgrad(dqkv, ln1, A.g(b + "token_mixing.net.in_w", G), accumulate=accumulate)
        ops.layernorm_bwd(dln1, net, A.p(b + "token_norm.weight"), mean1, rstd1, rows=M, dim=D, ld_x=D, dres=dmid,
                          dx_out=dnet, ld_dx=D, dx_bf16=dnet_bf,
                          dgamma=A.g(b + "token_norm.weight", G), dbeta=A.g(b + "token_norm.bias", G),
                          dx_colsum=A.g(f"encoder.mixing_blocks.{i - 1}.channel_mixing.net.3.linear.bias", G) if (i > 0 and next_ff2_bias) else None,
                          accumulate=accumulate)

    def stem_backward(self, sv: "_Saved", dnet: Tensor, G: Tensor, *, accumulate: bool = False) -> None:
        """tokens = cat(cls, patches) + pos ; patches = conv(x): pos / cls / conv weight (+ bias) gradients."""
        g, A = self.geo, self.arena
        dpatch = ops.assemble_tokens_bwd(dnet, A.g("encoder.pos_encoding.pos_encoding", G), A.g("encoder.head_token", G), sv.B, g.np, g.D,
                                         accumulate=accumulate)
        ops.wgrad(dpatch, sv.cols, A.g("to_patches.projection.weight", G).view(g.D, -1), accumulate=accumulate)
        if g.conv_bias:
            ops.colsum(dpatch, A.g("to_patches.projection.bias", G), accumulate=accumulate)

    # ---- forward ------------------------------------------------------------------------------------------
    def encoder_forward(self, x: Tensor, want_f32: bool, save: bool = True) -> Tuple[Tensor, Optional[Tensor], Optional[_Saved]]:
        """``save=False``: the same kernels in the same order, but nothing is kept for backward (the returned ``_Saved`` is
        None): the residual stream lives in two buffers and every block reuses one ``_Scratch``."""
        g, A = self.geo, self.arena
        if not x.is_cuda:
            raise B200Error("ViTEncoderB200 runs on CUDA only: there is no CPU fallback")
        if g.tokens:
            if x.dim() != 3 or x.shape[1] != g.T or x.shape[2] != g.D:
                raise ValueError(f"expected embedded tokens [B, {g.T}, {g.D}], got {tuple(x.shape)}")
        elif x.dtype == torch.uint8:
            if x.dim() != 4 or x.shape[3] != g.cin or x.shape[1] != g.img or x.shape[2] != g.img:
                raise ValueError(f"expected raw uint8 input [B, {g.img}, {g.img}, {g.cin}] (HWC), got {tuple(x.shape)}")
        elif x.dim() != 4 or x.shape[1] != g.cin or x.shape[2] != g.img or x.shape[3] != g.img:
            raise ValueError(f"expected input [B, {g.cin}, {g.img}, {g.img}], got {tuple(x.shape)}")
        x = x.contiguous() if x.dtype == torch.uint8 else x.contiguous().float()
        A.refresh_bf16()
        B, T, D, M = x.shape[0], g.T, g.D, x.shape[0] * g.T
        cols, net = self.stem_forward(x)
        sv, s = None, None
        if save:
            sv = _Saved()
            sv.B, sv.cols, sv.emb_in, sv.blocks = B, cols, None, []
        else:
            cols, s = None, _Scratch(g, B, x.device)  # (the im2col matrix is only kept for the weight gradient)
        if g.emb_eps is not None:  # embedding_norm (api.py:433-434): its fp32 output IS the residual stream
            normed = torch.empty_like(net)
            _, mean, rstd = ops.layernorm_fwd(net, A.p("encoder.embedding_norm.weight"), A.p("encoder.embedding_norm.bias"),
                                              g.emb_eps, rows=M, dim=D, ld_x=D, y_f32=normed, y=s and s.ln, mean=s and s.mean,
                                              rstd=s and s.rstd)
            if save:
                sv.emb_in, sv.emb_mean, sv.emb_rstd = net, mean, rstd
            net = normed
        for i in range(g.L):
            net, saved = self.block_forward(i, net, B, s)
            if save:
                sv.blocks.append(saved)
        hrows, hld = (M, D) if g.tokens else (B, T * D)
        enc_f32 = torch.empty((hrows, D), dtype=torch.float32, device=x.device) if want_f32 else None
        # head = LayerNorm over all tokens then token 0 (api.py:365,397-402): only row 0 of each image is needed;
        # token mode: head = PreNorm(Identity), every token is an output row
        enc_bf16, hm, hr = ops.layernorm_fwd(net, A.p(g.head_norm_key + "weight"), A.p(g.head_norm_key + "bias"), g.eps,
                                             rows=hrows, dim=D, ld_x=hld, y_f32=enc_f32,
                                             mean=s and s.mean[:hrows], rstd=s and s.rstd[:hrows])
        if save:
            sv.net_last, sv.head_mean, sv.head_rstd, sv.enc_bf16 = net, hm, hr, enc_bf16
        return enc_bf16, enc_f32, sv

    def head_forward(self, enc_bf16: Tensor) -> Tensor:
        A = self.arena
        return ops.gemm(enc_bf16, A.w("head.linear.weight"), bias=A.w("head.linear.bias"))

    # ---- `net @ output_projection` (cv/encoder/transformer.py:93-94): a bf16 matmul under autocast ----------------
    def projection_forward(self, enc_bf16: Tensor) -> Tensor:
        return ops.gemm(enc_bf16, self.arena.w("output_projection"), b_mn_major=True)  # [B, D] . [D, out] -> bf16 [B, out]

    def projection_backward(self, sv: _Saved, d_out: Tensor, G: Tensor, *, accumulate: bool = False) -> Tensor:
        A = self.arena
        d_enc = ops.gemm(d_out, A.w("output_projection"))                      # [B, out] . [D, out]^T -> bf16 [B, D]
        ops.wgrad(sv.enc_bf16, d_out, A.g("output_projection", G), accumulate=accumulate)  # enc^T . d_out -> [D, out]
        return d_enc

    # ---- backward -----------------------------------------------------------------------------------------
    def head_backward(self, sv: _Saved, dlogits: Tensor, G: Tensor, *, accumulate: bool = False) -> Tensor:
        A = self.arena
        d_enc = ops.gemm(dlogits, A.w("head.linear.weight"), b_mn_major=True)  # [B, D] bf16
        ops.wgrad(dlogits, sv.enc_bf16, A.g("head.linear.weight", G), accumulate=accumulate)
        ops.colsum(dlogits, A.g("head.linear.bias", G), accumulate=accumulate)
        return d_enc

    def encoder_backward(self, sv: _Saved, d_enc_bf16: Tensor, G: Tensor, *, accumulate: bool = False) -> Optional[Tensor]:
        """Writes every encoder parameter gradient into the flat arena ``G`` (overwriting it, or adding to it with
        ``accumulate``; activation gradients are never accumulated).  ``d_enc_bf16``: the
        gradient of the head LayerNorm's output -- bf16 [B, D] (vision: it feeds a bf16 matmul) or, in token mode,
        fp32 [B*T, D] (the LayerNorm output itself is what the module returns).  Token mode returns the gradient of the
        embedded input [B, T, D]."""
        g, A = self.geo, self.arena
        B, T, D, M = sv.B, g.T, g.D, sv.B * g.T
        dev = d_enc_bf16.device
        red = self.reducer
        dnet = torch.empty((M, D), dtype=torch.float32, device=dev)
        if g.tokens:
            dnet_bf = torch.empty((M, D), dtype=torch.bfloat16, device=dev)
            ops.layernorm_bwd(d_enc_bf16, sv.net_last, A.p(g.head_norm_key + "weight"), sv.head_mean, sv.head_rstd,
                              rows=M, dim=D, ld_x=D, dres=None, dx_out=dnet, ld_dx=D, dx_bf16=dnet_bf,
                              dgamma=A.g(g.head_norm_key + "weight", G), dbeta=A.g(g.head_norm_key + "bias", G), accumulate=accumulate)
        else:
            ops.fill_f32(dnet, 0.0)
            ops.layernorm_bwd(d_enc_bf16, sv.net_last, A.p(g.head_norm_key + "weight"), sv.head_mean, sv.head_rstd,
                              rows=B, dim=D, ld_x=T * D, dres=None, dx_out=dnet, ld_dx=T * D, dx_bf16=None,
                              dgamma=A.g(g.head_norm_key + "weight", G), dbeta=A.g(g.head_norm_key + "bias", G), accumulate=accumulate)
            dnet_bf = ops.cast_bf16(dnet)
        # bias gradient of the last block's FF2 (dY = dnet_bf); every other Linear whose dY comes out of a LayerNorm
        # backward gets its bias gradient from that kernel (dx_colsum)
        ops.colsum(dnet_bf, A.g(f"encoder.mixing_blocks.{g.L - 1}.channel_mixing.net.3.linear.bias", G), accumulate=accumulate)
        if red is not None:
            red.ready("tail", G)
        for i in reversed(range(g.L)):
            self.block_backward(i, sv.blocks[i], dnet, dnet_bf, G, B, accumulate=accumulate)
            sv.blocks[i] = None  # release this block's activations
            if red is not None:
                red.ready(i, G)
        if sv.emb_in is not None:  # embedding_norm backward: dy is the fp32 residual-stream gradient
            dpre = torch.empty_like(dnet)
            ops.layernorm_bwd(dnet, sv.emb_in, A.p("encoder.embedding_norm.weight"), sv.emb_mean, sv.emb_rstd, rows=M, dim=D, ld_x=D,
                              dres=None, dx_out=dpre, ld_dx=D, dx_bf16=None,
                              dgamma=A.g("encoder.embedding_norm.weight", G), dbeta=A.g("encoder.embedding_norm.bias", G),
                              accumulate=accumulate)
            dnet = dpre
        if g.tokens:  # net = x + pos: the input gradient is dnet itself
            ops.add_pos_bwd(dnet, A.g("encoder.pos_encoding.pos_encoding", G), B, T, D, accumulate=accumulate)
        else:
            self.stem_backward(sv, dnet, G, accumulate=accumulate)
        if red is not None:
            red.ready("stem", G)
        return dnet.view(B, T, D) if g.tokens else None

    # ---- the whole stack: the encoder, then what the geometry puts after it ----------------------------------------
    def stack_forward(self, x: Tensor, head: bool, save: bool = True) -> Tuple[Tensor, Optional[_Saved]]:
        """The module output: the classifier's bf16 logits (``head``), the bf16 ``net @ output_projection``, or the fp32
        head LayerNorm output (vision: [B, D] of the cls token; token mode: [B, T, D]).  ``save=False``: the forward-only
        stack of ``encoder_forward``, bit-identical output, no ``_Saved``."""
        g = self.geo
        bf16_tail = head or g.out_dim is not None
        enc_bf16, enc_f32, sv = self.encoder_forward(x, want_f32=not bf16_tail, save=save)
        if head:
            return self.head_forward(enc_bf16), sv
        if g.out_dim is not None:
            return self.projection_forward(enc_bf16), sv
        return (enc_f32.view(x.shape[0], g.T, g.D) if g.tokens else enc_f32), sv

    def stack_backward(self, sv: _Saved, d_out: Tensor, G: Tensor, head: bool, *, accumulate: bool = False) -> Optional[Tensor]:
        """Backward of ``stack_forward`` from the gradient of its output (``accumulate``: added to ``G``); returns the input
        gradient in token mode."""
        g = self.geo
        if head:
            if d_out.dtype != torch.bfloat16:
                raise B200Error("classifier backward expects a bf16 gradient for the bf16 logits")
            d_enc = self.head_backward(sv, ops.tma_aligned(d_out), G, accumulate=accumulate)
        elif g.tokens:  # fp32: the LayerNorm output is the module output
            d_enc = d_out.contiguous().float().view(-1, g.D)
        else:  # under autocast the encoder output feeds a bf16 matmul, so its gradient is bf16-representable
            d_enc = d_out.contiguous() if d_out.dtype == torch.bfloat16 else ops.cast_bf16(d_out.contiguous().float())
            if g.out_dim is not None:
                d_enc = self.projection_backward(sv, d_enc, G, accumulate=accumulate)
        return self.encoder_backward(sv, d_enc, G, accumulate=accumulate)


# -----------------------------------------------------------------------------------------------------------------
# autograd glue
# -----------------------------------------------------------------------------------------------------------------
class _StackFn(torch.autograd.Function):
    """The whole native stack of one module as ONE autograd node (``ViTEngine.stack_forward``).  Its backward writes every
    parameter gradient into the gradient arena -- overwriting it, or adding to it in place while the parameters hold
    gradients (``ParamArena.claim_grads``) -- and publishes them as ``p.grad`` views, so autograd receives ``None`` for the
    parameters; only token mode returns an input gradient."""

    @staticmethod
    def forward(ctx: Any, engine: ViTEngine, keys: List[str], head: bool, x: Tensor, *params: Tensor) -> Tensor:
        out, sv = engine.stack_forward(x, head)
        ctx.engine, ctx.keys, ctx.head, ctx.sv = engine, keys, head, sv
        return out

    @staticmethod
    def backward(ctx: Any, d_out: Tensor) -> Tuple[Any, ...]:
        eng, keys = ctx.engine, ctx.keys
        accumulate = eng.arena.claim_grads(keys)
        d_in = eng.stack_backward(ctx.sv, d_out, eng.arena.grad, ctx.head, accumulate=accumulate)
        if eng.reducer is not None:
            eng.reducer.finish()
        eng.arena.publish_grads(keys)
        ctx.sv = None
        return (None, None, None, d_in) + (None,) * len(keys)


class _SoftmaxXentFn(torch.autograd.Function):
    """CrossEntropyLoss (losses/basic.py:137-141) + mean reduction (schema.py:767-775) on bf16 logits."""

    last_bad: Optional[Tensor] = None

    @staticmethod
    def forward(ctx: Any, logits: Tensor, labels: Tensor) -> Tensor:
        lab = labels.reshape(-1).contiguous()
        loss_mean, _, _, bad = ops.softmax_xent(logits, lab, need_grad=False)
        ctx.save_for_backward(logits, lab)
        _SoftmaxXentFn.last_bad = bad  # int32[1] on the device: non-zero if a label was outside [0, C)
        return loss_mean.reshape(())

    @staticmethod
    def backward(ctx: Any, grad_out: Tensor) -> Tuple[Any, ...]:
        logits, lab = ctx.saved_tensors
        go = grad_out.reshape(1).contiguous().float()
        _, _, dlogits, _ = ops.softmax_xent(logits, lab, need_grad=True, grad_scale_dev=go)
        return dlogits, None


def cross_entropy(logits: Tensor, labels: Tensor) -> Tensor:
    """Mean softmax cross-entropy of bf16 ``logits`` [B, C] against int64 ``labels`` [B] or [B, 1].  Labels outside
    [0, C) contribute nothing and set a device flag (``bad_label_flag()``); ``VanillaClassifierB200`` raises for it."""
    if logits.dtype != torch.bfloat16:
        raise B200Error("cross_entropy expects the bf16 logits produced by VanillaClassifierB200")
    return _SoftmaxXentFn.apply(logits, labels)  # keeps the logits' padded row stride (see ops.gemm)


def bad_label_flag() -> Optional[Tensor]:
    """int32[1] device tensor written by the most recent ``cross_entropy`` forward (non-zero: a label was out of range)."""
    return _SoftmaxXentFn.last_bad


# -----------------------------------------------------------------------------------------------------------------
# modules (the plug-in surface)
# -----------------------------------------------------------------------------------------------------------------
def _check_supported(**kw: Any) -> None:
    expected = dict(to_patches_type="vanilla", dropout=0.0, drop_path_rate=0.0, norm_type="layer",
                    residual_after_norm=False, use_head_token=True, use_positional_encoding=True)
    for k, v in expected.items():
        if k in kw and kw[k] != v and not (kw[k] is None and v is None):
            raise NotImplementedError(
                f"ViTEncoderB200: {k}={kw[k]!r} is outside the fused B200 path (supported: {v!r}); "
                f"use the reference module for this configuration"
            )


def _check_common(name: str, latent_dim: int, *, default_heads: int, norm_kwargs: Optional[Dict[str, Any]],
                  embedding_norm: Optional[nn.Module], attention_kwargs: Optional[Dict[str, Any]],
                  feedforward_kwargs: Optional[Dict[str, Any]]) -> Dict[str, Any]:
    """The keywords both encoders read alike; returns the ``ViTGeometry`` keywords they determine."""
    fk = dict(feedforward_kwargs or {})
    if set(fk) - {"activation"}:
        raise NotImplementedError(f"unsupported feedforward_kwargs: {sorted(set(fk) - {'activation'})}")
    emb_eps: Optional[float] = None
    if embedding_norm is not None:  # clip.py:131: nn.LayerNorm(latent_dim, eps)
        if not isinstance(embedding_norm, nn.LayerNorm) or tuple(embedding_norm.normalized_shape) != (latent_dim,) \
                or not embedding_norm.elementwise_affine or embedding_norm.bias is None:
            raise NotImplementedError("embedding_norm must be an affine nn.LayerNorm(latent_dim)")
        emb_eps = float(embedding_norm.eps)
    ak = dict(attention_kwargs or {})
    if ak.get("num_heads", default_heads) != latent_dim // 64 or not ak.get("bias", True) or set(ak) - {"num_heads", "bias"}:
        raise NotImplementedError(f"{name} needs attention_kwargs num_heads = latent_dim // 64 (head dim 64) and bias=True, "
                                  f"got {ak}")
    eps = float((norm_kwargs or {}).get("eps", 1e-6))  # norms.py:118-119 default, clip.py:128 overrides to 1e-5
    return dict(eps=eps, embedding_norm_eps=emb_eps, activation=fk.get("activation", "GELU"))


class _FusedStack(ArenaModule):
    """What ``ViTEncoderB200`` and ``TeTEncoderB200`` share: parameters in one arena, one engine, one autograd node."""

    def _build(self, geo: ViTGeometry, embedding_norm: Optional[nn.Module], defer_head: bool = False) -> None:
        """Parameters with the reference initialisation (an ``embedding_norm`` instance handed in is adopted), registered
        under the reference's names, then the arena and the engine.  ``defer_head``: the classifier registers
        ``head.linear.*`` itself, after its ``encoder`` sub-module (the reference's key order)."""
        spec = geo.spec()
        params: Dict[str, nn.Parameter] = {}
        for key, shape in spec:
            p = nn.Parameter(_init_param(key, shape))
            if embedding_norm is not None and key.startswith("encoder.embedding_norm."):
                p.data.copy_(getattr(embedding_norm, key.rsplit(".", 1)[1]).data)
            params[key] = p
            if not (defer_head and key.startswith("head.linear")):
                register_dotted(self, key, p)
        self.geo = geo
        self.arena = ParamArena(spec)
        self.arena.attach(params)
        self.engine = ViTEngine(geo, self.arena)
        self.all_keys = [k for k, _ in spec]
        self.encoder_keys = [k for k in self.all_keys if not k.startswith("head.linear")]

    def _run(self, net: Tensor, head: bool = False) -> Tensor:
        """The stack on ``net`` as one autograd node; ``head``: through the classifier head.  With gradients disabled
        (``torch.no_grad``, evaluation) the forward-only stack runs instead: the same output, bit for bit, without holding
        any block's activations."""
        keys = self.all_keys if head else self.encoder_keys
        self.arena.ensure()
        if not torch.is_grad_enabled():
            return self.engine.stack_forward(net, head, save=False)[0]
        return _StackFn.apply(self.engine, keys, head, net, *[self.arena.params[k] for k in keys])


class ViTEncoderB200(_FusedStack):
    """Drop-in for ``ViTEncoder`` (registered as ``encoders.vit`` in the reference, transformer.py:16-17)."""

    def __init__(
        self,
        *,
        img_size: int,
        patch_size: int,
        in_channels: int,
        latent_dim: int = 384,
        to_patches_type: str = "vanilla",
        to_patches_config: Optional[Dict[str, Any]] = None,
        num_layers: int = 12,
        dropout: float = 0.0,
        drop_path_rate: float = 0.0,
        norm_type: Optional[str] = "layer",
        norm_kwargs: Optional[Dict[str, Any]] = None,
        embedding_norm: Optional[nn.Module] = None,
        residual_after_norm: bool = False,
        feedforward_dim_ratio: float = 4.0,
        attention_kwargs: Optional[Dict[str, Any]] = None,
        feedforward_kwargs: Optional[Dict[str, Any]] = None,
        use_head_token: bool = True,
        head_pooler: Optional[str] = "mean",
        use_positional_encoding: bool = True,
        norm_after_head: bool = False,
        output_dim: Optional[int] = None,
        _num_classes: Optional[int] = None,
        _defer_head: bool = False,
    ):
        super().__init__()
        _check_supported(to_patches_type=to_patches_type, dropout=dropout, drop_path_rate=drop_path_rate, norm_type=norm_type,
                         residual_after_norm=residual_after_norm, use_head_token=use_head_token,
                         use_positional_encoding=use_positional_encoding)
        common = _check_common("ViTEncoderB200", latent_dim, default_heads=latent_dim // 64, norm_kwargs=norm_kwargs,
                               embedding_norm=embedding_norm, attention_kwargs=attention_kwargs,
                               feedforward_kwargs=feedforward_kwargs)
        tpc = dict(to_patches_config or {})
        if set(tpc) - {"bias"}:
            raise NotImplementedError(f"unsupported to_patches_config: {sorted(set(tpc) - {'bias'})}")
        self._build(ViTGeometry(img_size=img_size, patch_size=patch_size, in_channels=in_channels, latent_dim=latent_dim,
                                num_layers=num_layers, ff_ratio=feedforward_dim_ratio, num_classes=_num_classes,
                                conv_bias=bool(tpc.get("bias", True)), norm_after_head=bool(norm_after_head),
                                output_dim=output_dim, **common),
                    embedding_norm, defer_head=_defer_head)
        self.latent_dim = latent_dim

    def named_arena_parameters(self):
        """(arena key, parameter) pairs: the reference ``ViTEncoder`` state_dict names (+ ``head.linear.*``)."""
        return [(k, self.arena.params[k]) for k in self.all_keys]

    def forward(self, net: Tensor, *, hw: Any = None, hwp: Any = None, deterministic: bool = False) -> Tensor:
        if hwp is not None:
            raise NotImplementedError("positional-encoding interpolation (hwp) is outside the fused path")
        return self._run(net)

    def encode(self, net: Tensor) -> Tensor:  # IEncoder.encode, cv/common.py:42-50
        return self.forward(net)

    def set_input_pipeline(self, *, division: float = 255.0, mean: Any = None, std: Any = None) -> None:
        """Accept RAW uint8 [B, S, S, C] batches: ``((x / division) - mean) / std`` (float64 -> float32 -> bf16, the reference's
        static_normalize + imagenet_normalize / affine_normalize + hwc_to_chw runtime blocks) is evaluated inside the
        patch gather on the GPU.  Float [B, C, S, S] inputs keep working unchanged."""
        self.engine.input_pipeline = dict(division=float(division), mean=None if mean is None else [float(v) for v in mean],
                                          std=None if std is None else [float(v) for v in std])


class TeTEncoderB200(_FusedStack):
    """Drop-in for ``TeTEncoder`` (registered as ``tet``, cflearn/modules/nlp/encoder/transformer.py:16-99): the text
    tower's transformer stack on an already embedded sequence [B, T, D] -> LayerNorm-ed tokens [B, T, D] (fp32).
    Same kernels as the ViT blocks with the causal flag of the attention kernels (``use_triu_attn_mask``); the
    ``attention_mask`` buffer is kept so that ``state_dict`` keys match the reference's."""

    def __init__(self, latent_dim: int = 384, context_length: int = 77, *, use_triu_attn_mask: bool = False, num_layers: int = 12,
                 dropout: float = 0.0, drop_path_rate: float = 0.0, norm_position: str = "pre_norm",
                 norm_type: Optional[str] = "layer", norm_kwargs: Optional[Dict[str, Any]] = None,
                 embedding_norm: Optional[nn.Module] = None, embedding_dropout: Optional[float] = None,
                 residual_after_norm: bool = False, feedforward_dim_ratio: float = 4.0,
                 attention_kwargs: Optional[Dict[str, Any]] = None, feedforward_kwargs: Optional[Dict[str, Any]] = None,
                 use_positional_encoding: bool = True, head_pooler: Optional[str] = None, no_head_norm: Optional[bool] = None,
                 norm_after_head: bool = False):
        super().__init__()
        if dropout != 0.0 or drop_path_rate != 0.0 or norm_position != "pre_norm" or norm_type != "layer" or residual_after_norm \
                or embedding_dropout not in (None, 0.0) or not use_positional_encoding or head_pooler is not None \
                or no_head_norm not in (None, False) or norm_after_head:
            raise NotImplementedError("TeTEncoderB200 implements the configuration CLIP's text tower uses (pre-norm LayerNorm, "
                                      "no dropout / drop-path, learned positions, head_pooler=None)")
        # the reference TeTEncoder's num_heads defaults to 6, whatever latent_dim is
        common = _check_common("TeTEncoderB200", latent_dim, default_heads=6, norm_kwargs=norm_kwargs, embedding_norm=embedding_norm,
                               attention_kwargs=attention_kwargs, feedforward_kwargs=feedforward_kwargs)
        if use_triu_attn_mask:  # transformer.py:42-48
            self.register_buffer("attention_mask", torch.ones(context_length, context_length, dtype=torch.bool).triu_(1))
        else:
            self.attention_mask = None
        self._build(ViTGeometry(img_size=0, patch_size=16, in_channels=0, latent_dim=latent_dim, num_layers=num_layers,
                                ff_ratio=feedforward_dim_ratio, num_classes=None, context_length=context_length,
                                causal=bool(use_triu_attn_mask), **common),
                    embedding_norm)
        self.latent_dim = latent_dim

    def forward(self, net: Tensor, mask: Optional[Tensor] = None, *, apply_head: bool = True, clip_skip: int = 0, **kwargs: Any) -> Tensor:
        if mask is not None or not apply_head or clip_skip != 0:
            raise NotImplementedError("TeTEncoderB200: custom masks, apply_head=False and clip_skip are outside the fused path")
        return self._run(net)


class VanillaClassifierB200(ArenaModule):
    """Drop-in for ``cv_clf`` with ``encoder="vit"`` (cv/classifier/vanilla.py:16-66): ``{"predictions": logits}``.

    Module tree and ``state_dict`` layout are the reference's: the encoder is the sub-module ``encoder``
    (``encoder.to_patches.*``, ``encoder.encoder.mixing_blocks.*`` ...) followed by ``head.linear.{weight,bias}``, so
    checkpoints move between the reference ``cv_clf`` and this class with a plain ``load_state_dict(strict=True)``.
    The head's parameters live in the same flat arena as the encoder's (one cast, one all-reduce, one Adam launch).
    For convenience ``load_state_dict`` also accepts the encoder's keys WITHOUT the ``encoder.`` prefix (the layout of a
    bare ``ViTEncoder`` checkpoint + head, which is what ``oracle/vit_oracle.py`` emits)."""

    def __init__(self, in_channels: int, num_classes: int, img_size: Optional[int] = None, latent_dim: int = 128,
                 aux_num_classes: Optional[Dict[str, int]] = None, *, encoder: str = "vit",
                 encoder_config: Optional[Dict[str, Any]] = None):
        super().__init__()
        if aux_num_classes is not None:
            raise NotImplementedError("aux heads are outside the fused path")
        if encoder not in ("vit", "vit_b200"):
            raise NotImplementedError(f"VanillaClassifierB200 only fuses the ViT encoder, got encoder={encoder!r}")
        cfg = dict(encoder_config or {})
        cfg.setdefault("img_size", img_size)
        cfg.setdefault("in_channels", in_channels)
        cfg.setdefault("latent_dim", latent_dim)
        self.img_size = img_size
        self.encoder = ViTEncoderB200(**cfg, _num_classes=num_classes, _defer_head=True)
        for key in ("head.linear.weight", "head.linear.bias"):  # registered after `encoder`: the reference's key order
            register_dotted(self, key, self.encoder.arena.params[key])
        self.num_classes = num_classes
        self._bad_host: Optional[Tensor] = None
        self._bad_event: Optional[torch.cuda.Event] = None
        self._register_load_state_dict_pre_hook(self._accept_bare_encoder_keys)

    # the engine, arena and geometry are the encoder's (they include the head's parameters)
    @property
    def arena(self) -> ParamArena:
        return self.encoder.arena

    @property
    def engine(self) -> ViTEngine:
        return self.encoder.engine

    @property
    def geo(self) -> ViTGeometry:
        return self.encoder.geo

    @property
    def all_keys(self) -> List[str]:
        return self.encoder.all_keys

    @property
    def encoder_keys(self) -> List[str]:
        return self.encoder.encoder_keys

    def named_arena_parameters(self):
        """(arena key, parameter): ``ViTEncoder`` keys + ``head.linear.*`` -- the names ``oracle/vit_oracle.py`` uses."""
        return self.encoder.named_arena_parameters()

    def set_input_pipeline(self, **kw: Any) -> None:
        self.encoder.set_input_pipeline(**kw)

    def _accept_bare_encoder_keys(self, state_dict: Dict[str, Tensor], prefix: str, *args: Any) -> None:
        enc = set(self.encoder_keys)
        for k in list(state_dict.keys()):
            if k.startswith(prefix) and k[len(prefix):] in enc and (prefix + "encoder." + k[len(prefix):]) not in state_dict:
                state_dict[prefix + "encoder." + k[len(prefix):]] = state_dict.pop(k)

    def forward(self, net: Tensor, *, return_latent: bool = False) -> Dict[str, Tensor]:
        self.check_labels()
        if return_latent:
            return {LATENT_KEY: self.encoder._run(net)}
        return {PREDICTIONS_KEY: self.encoder._run(net, head=True)}

    def train_step(self, net: Tensor, labels: Tensor) -> Tensor:
        """forward + CrossEntropyLoss + backward (IDLModel.train, schema.py:1266-1276,:980); returns the loss.
        An out-of-range label raises ``ValueError`` from a later call (see ``check_labels``): the flag travels to pinned
        host memory asynchronously, so no step ever waits on the device for it."""
        logits = self.forward(net)[PREDICTIONS_KEY]
        loss = cross_entropy(logits, labels)
        bad = _SoftmaxXentFn.last_bad
        self.last_bad_flag = bad
        if bad is not None and not torch.cuda.is_current_stream_capturing():
            if self._bad_host is None:
                self._bad_host = torch.zeros(1, dtype=torch.int32).pin_memory()
            elif self._bad_event is not None:
                self._bad_event.synchronize()  # the previous copy must have landed before its buffer is reused
                self._raise_if_bad()
            self._bad_host.copy_(bad, non_blocking=True)
            self._bad_event = torch.cuda.Event()
            self._bad_event.record()
        loss.backward()
        return loss.detach()

    def _raise_if_bad(self) -> None:
        if self._bad_host is not None and int(self._bad_host[0]) != 0:
            self._bad_host.zero_()
            self._bad_event = None
            raise ValueError("cross_entropy: a label of an earlier train_step was outside [0, num_classes)")

    def check_labels(self, sync: bool = False) -> None:
        """Eager raises a device-side assert on an out-of-range class index (``gather`` in losses/basic.py:139); the fused
        loss records a flag on the device instead.  This raises ``ValueError`` for it once the flag has reached the host
        (``sync=True`` waits for it); ``forward`` calls it without waiting."""
        ev = self._bad_event
        if ev is None or torch.cuda.is_current_stream_capturing():  # (querying an event is not allowed while capturing)
            return
        if sync:
            ev.synchronize()
        if ev.query():
            self._bad_event = None
            self._raise_if_bad()

    def load_reference_state_dict(self, sd: Dict[str, Tensor]) -> None:
        """Reference ``cv_clf`` checkpoint (``encoder.<ViTEncoder keys>`` + ``head.linear.*``): same as ``load_state_dict``."""
        self.load_state_dict(sd, strict=True)
