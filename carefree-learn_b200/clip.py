"""Drop-in for the reference's ``CLIP`` (cflearn/modules/multimodal/clip.py:21-275, registry name ``"clip"``) on sm_90a.

Both towers run on the native kernels (``ViTEncoderB200`` with CLIP's options, ``TeTEncoderB200``); the text glue's integer
ops (embedding gather / scatter-add, arg-max token pooling) and the two small matmuls (``text_projection``, the logits
product) are C-ABI kernels as well.  What remains PyTorch are the elementwise bf16 ops on [B, latent_dim] tensors that
the reference itself runs eagerly -- ``l2_normalize`` (cftool.array, restated as ``t / t.norm(dim=-1, keepdim=True)``)
and ``logit_scale.exp() * image_features`` -- executed in fp32 exactly as CUDA autocast would (``norm`` and ``exp`` are on its
fp32 list), so their rounding points are eager's by construction; the logits matmul casts its operands to bf16.  Constructor keywords, ``state_dict`` keys / order (incl. the ``attention_mask`` buffer) and
the ``forward(image, text) -> logits_per_image`` / ``encode_image`` / ``encode_text`` signatures are the reference's.
The reference defines no CLIP loss or training step (SURVEY.md 8d); gradients flow through autograd.
"""
from __future__ import annotations

import math
from typing import Any, List, Optional, Tuple

import torch
import torch.nn as nn
from torch import Tensor

from . import ops
from ._cabi import B200Error
from .arena import ArenaModule, ParamArena
from .vit import TeTEncoderB200, ViTEncoderB200


def l2_normalize(t: Tensor) -> Tensor:
    """``t / t.norm(dim=-1, keepdim=True)`` as CUDA autocast runs it: ``norm`` is on autocast's fp32 list, so the norm is taken
    of the up-cast features and the division promotes to fp32 -- the bf16 rounding only happens at the next matmul."""
    tf = t.float()
    return tf / tf.norm(dim=-1, keepdim=True)


class _EmbeddingFn(torch.autograd.Function):
    """nn.Embedding(vocab, dim, padding_idx) (clip.py:157-161): gather forward, scatter-add backward, both bit-exact row moves."""

    @staticmethod
    def forward(ctx: Any, ids: Tensor, weight: Tensor, padding_idx: int) -> Tensor:
        ids = ids.contiguous()
        out, _ = ops.embedding_fwd(ids, weight)
        ctx.save_for_backward(ids)
        ctx.shape, ctx.padding_idx = weight.shape, padding_idx
        return out

    @staticmethod
    def backward(ctx: Any, dnet: Tensor) -> Tuple[Any, ...]:
        (ids,) = ctx.saved_tensors
        return None, ops.embedding_bwd(ids, dnet.contiguous().float(), *ctx.shape, ctx.padding_idx), None


class _ArgmaxPoolFn(torch.autograd.Function):
    """``net[arange(B), indices.argmax(-1)]`` (clip.py:248-250)."""

    @staticmethod
    def forward(ctx: Any, net: Tensor, ids: Tensor) -> Tensor:
        out, pos = ops.argmax_gather_rows(net.contiguous().float(), ids.contiguous())
        ctx.save_for_backward(pos)
        ctx.T = net.shape[1]
        return out

    @staticmethod
    def backward(ctx: Any, dout: Tensor) -> Tuple[Any, ...]:
        (pos,) = ctx.saved_tensors
        return ops.scatter_rows(dout.contiguous().float(), pos, ctx.T), None


class _LinearBf16Fn(torch.autograd.Function):
    """``F.linear`` under autocast (HijackLinear text_projection, clip.py:188,253): bf16 operands, fp32 accumulate, bf16 out;
    gradients: bf16 dgrad, weight / bias gradients rounded to bf16 then widened (what autocast's backward produces)."""

    @staticmethod
    def forward(ctx: Any, x: Tensor, weight: Tensor, bias: Optional[Tensor]) -> Tensor:
        xb = ops.cast_bf16(x.contiguous().float()) if x.dtype != torch.bfloat16 else x.contiguous()
        wb = ops.cast_bf16(weight.contiguous().float())
        bb = ops.cast_bf16(bias.contiguous().float()) if bias is not None else None
        ctx.save_for_backward(xb, wb)
        ctx.has_bias, ctx.x_dtype = bias is not None, x.dtype
        return ops.gemm(xb, wb, bias=bb)

    @staticmethod
    def backward(ctx: Any, dy: Tensor) -> Tuple[Any, ...]:
        xb, wb = ctx.saved_tensors
        dy = dy.contiguous()
        dy = ops.tma_aligned(dy if dy.dtype == torch.bfloat16 else ops.cast_bf16(dy.float()))
        dx = ops.gemm(dy, wb, b_mn_major=True)                       # [B, out] . [out, in] -> bf16 [B, in]
        dw = torch.empty(wb.shape, dtype=torch.float32, device=dy.device)
        ops.wgrad(dy, xb, dw)                                        # dy^T . x -> [out, in]
        db = None
        if ctx.has_bias:
            db = torch.empty(wb.shape[0], dtype=torch.float32, device=dy.device)
            ops.colsum(dy, db)
        return (dx if ctx.x_dtype == torch.bfloat16 else dx.float()), dw, db


class _MatmulNTFn(torch.autograd.Function):
    """``a @ b.t()`` on bf16 [B, L] features (schema.py:29): the logits product and its two gradients on the wgmma GEMM."""

    @staticmethod
    def forward(ctx: Any, a: Tensor, b: Tensor) -> Tensor:
        if not a.is_cuda or not b.is_cuda:
            raise B200Error("the logits product runs on CUDA only: there is no CPU fallback")
        ctx.dtypes = (a.dtype, b.dtype)
        a = a.contiguous() if a.dtype == torch.bfloat16 else ops.cast_bf16(a.contiguous().float())  # autocast's operand casts
        b = b.contiguous() if b.dtype == torch.bfloat16 else ops.cast_bf16(b.contiguous().float())
        ctx.save_for_backward(a, b)
        return ops.gemm(a, b)                                        # [Ba, L] . [Bb, L]^T -> bf16 [Ba, Bb]

    @staticmethod
    def backward(ctx: Any, dy: Tensor) -> Tuple[Any, ...]:
        a, b = ctx.saved_tensors
        dy = dy.contiguous()
        dy = ops.tma_aligned(dy if dy.dtype == torch.bfloat16 else ops.cast_bf16(dy.float()))
        da = ops.gemm(dy, b, b_mn_major=True)                        # dy . b        -> [Ba, L]
        db = ops.gemm(dy, a, a_mn_major=True, b_mn_major=True)       # dy^T . a      -> [Bb, L]
        return (da if ctx.dtypes[0] == torch.bfloat16 else da.float()), (db if ctx.dtypes[1] == torch.bfloat16 else db.float())


class _SymmetricXentFn(torch.autograd.Function):
    """``(CE(L, arange) + CE(L^T, arange)) / 2`` on the bf16 logits [B, B] (fp32 maths, like autocast's cross_entropy)."""

    @staticmethod
    def forward(ctx: Any, logits: Tensor) -> Tensor:
        loss = ops.symmetric_xent(logits)
        ctx.save_for_backward(logits)
        return loss.reshape(())

    @staticmethod
    def backward(ctx: Any, grad_out: Tensor) -> Tuple[Any, ...]:
        (logits,) = ctx.saved_tensors
        dlogits = torch.empty_strided(logits.shape, logits.stride(), dtype=torch.bfloat16, device=logits.device)
        ops.symmetric_xent(logits, dlogits=dlogits, grad_scale_dev=grad_out.reshape(1).contiguous().float())
        return (dlogits,)


def symmetric_cross_entropy(logits_per_image: Tensor) -> Tensor:
    """The contrastive objective of CLIP on ``logits_per_image`` [B, B] (targets ``arange(B)`` in both directions).  The
    reference ships no loss for its CLIP module (SURVEY.md 8d: none in ``models/`` or ``losses/``); this is the standard
    definition, restated for the parity tests in ``oracle/clip_oracle.py::symmetric_cross_entropy``."""
    return _SymmetricXentFn.apply(logits_per_image)


class CLIPB200(ArenaModule):
    def __init__(self, img_size: int = 224, latent_dim: int = 512, *, use_vision: bool = True, in_channels: int = 3,
                 vision_latent_dim: int = 768, vision_patch_size: int = 32, vision_num_heads: int = 12, vision_num_layers: int = 12,
                 vision_norm_eps: float = 1.0e-5, vision_feedforward_activation: str = "quick_gelu", use_text: bool = True,
                 vocab_size: int = 49408, context_length: int = 77, use_text_triu_attn_mask: bool = True,
                 token_type_size: Optional[int] = None, text_latent_dim: int = 512, text_padding_idx: int = 0,
                 use_text_embedding_norm: bool = False, text_embedding_dropout: Optional[bool] = None, text_dropout: float = 0.0,
                 text_num_heads: int = 8, text_num_layers: int = 12, text_norm_position: str = "pre_norm",
                 text_norm_eps: float = 1.0e-5, text_feedforward_activation: str = "quick_gelu",
                 text_head_pooler: Optional[str] = None):
        super().__init__()
        if not use_vision or not use_text or token_type_size is not None or text_dropout != 0.0 or text_embedding_dropout \
                or text_head_pooler is not None:
            raise NotImplementedError("CLIPB200 implements the reference defaults: both towers, no token types, no dropout, "
                                      "arg-max token pooling")
        self.img_size, self.context_length = img_size, context_length
        self.logit_scale = nn.Parameter(torch.tensor(math.log(1 / 0.07)))  # multimodal/schema.py:15
        # clip.py:121-135
        self.vit = ViTEncoderB200(
            img_size=img_size, patch_size=vision_patch_size, in_channels=in_channels, latent_dim=vision_latent_dim,
            to_patches_config={"bias": False}, num_layers=vision_num_layers, norm_kwargs={"eps": vision_norm_eps},
            embedding_norm=nn.LayerNorm(vision_latent_dim, vision_norm_eps), attention_kwargs={"num_heads": vision_num_heads},
            feedforward_kwargs={"activation": vision_feedforward_activation}, norm_after_head=True, output_dim=latent_dim)
        # clip.py:157-188
        self.token_embedding = nn.Embedding(vocab_size, text_latent_dim, padding_idx=text_padding_idx)
        self.text_transformer = TeTEncoderB200(
            text_latent_dim, context_length, use_triu_attn_mask=use_text_triu_attn_mask, num_layers=text_num_layers,
            norm_position=text_norm_position, norm_kwargs={"eps": text_norm_eps},
            embedding_norm=nn.LayerNorm(text_latent_dim, text_norm_eps) if use_text_embedding_norm else None,
            attention_kwargs={"num_heads": text_num_heads}, feedforward_kwargs={"activation": text_feedforward_activation},
            head_pooler=text_head_pooler)
        self.text_projection = nn.Linear(text_latent_dim, latent_dim)
        self.text_latent_dim, self.text_num_layers = text_latent_dim, text_num_layers
        self.reset_parameters()
        # the parameters outside the towers live in a third flat arena (same machinery: one Adam launch, one all-reduce)
        self._glue_keys = ["logit_scale", "token_embedding.weight", "text_projection.weight", "text_projection.bias"]
        glue = {"logit_scale": self.logit_scale, "token_embedding.weight": self.token_embedding.weight,
                "text_projection.weight": self.text_projection.weight, "text_projection.bias": self.text_projection.bias}
        self.glue = ParamArena([(k, tuple(p.shape)) for k, p in glue.items()])
        self.glue.attach(glue)

    # ---- the trainer seam's contract (arena.ArenaModule): the glue arena is exchanged through ``comm`` by train_step ----
    def arenas(self) -> List[ParamArena]:
        return [self.vit.arena, self.text_transformer.arena, self.glue]

    def exchanges(self) -> List[Any]:
        return [self.vit.engine, self.text_transformer.engine]

    def _collect_glue_grads(self) -> None:
        """autograd hands the loose parameters' gradients over as separate tensors: move them into the glue arena.  Once they
        are its views, autograd accumulates the next backward's gradients into them in place."""
        with torch.no_grad():
            for k in self._glue_keys:
                p = self.glue.params[k]
                v = self.glue.g(k)
                if p.grad is None:
                    v.zero_()
                elif p.grad.data_ptr() != v.data_ptr():
                    v.copy_(p.grad)
                p.grad = v

    def train_step(self, image: Tensor, text: Tensor) -> Tensor:
        """forward + symmetric cross-entropy + backward (+ data parallel: the towers' bucket reducers run inside their
        backward, the loose parameters are all-reduced here); returns the loss (fp32 scalar on the device).  Under
        gradient accumulation the trainer runs every micro-batch but a window's last in ``dp.no_sync``, so both exchanges
        happen once per window, on the accumulated gradients."""
        loss = symmetric_cross_entropy(self.forward(image, text))
        loss.backward()
        self._collect_glue_grads()
        if self.comm is not None and self.comm.world > 1:
            self.comm.allreduce_(self.glue.grad, average=True)
        return loss.detach()

    def reset_parameters(self) -> None:
        """clip.py:188-207: the text tower is re-initialised with CLIP's own standard deviations (the vision tower keeps the
        encoder's trunc_normal(0.02) initialisation, as in the reference)."""
        tld = self.text_latent_dim
        proj_std = (tld ** -0.5) * ((2 * self.text_num_layers) ** -0.5)
        attn_std = tld ** -0.5
        fc_std = (2 * tld) ** -0.5
        P = self.text_transformer.arena.params
        with torch.no_grad():
            nn.init.normal_(self.token_embedding.weight, std=0.02)
            nn.init.normal_(P["encoder.pos_encoding.pos_encoding"], std=0.01)
            for i in range(self.text_num_layers):
                b = f"encoder.mixing_blocks.{i}."
                nn.init.normal_(P[b + "token_mixing.net.in_w"], std=attn_std)
                nn.init.normal_(P[b + "token_mixing.net.out_linear.linear.weight"], std=proj_std)
                nn.init.normal_(P[b + "channel_mixing.net.0.linear.weight"], std=fc_std)
                nn.init.normal_(P[b + "channel_mixing.net.3.linear.weight"], std=proj_std)
            nn.init.normal_(self.text_projection.weight, std=tld ** -0.5)
            nn.init.zeros_(self.text_projection.bias)

    def encode_image(self, image: Tensor) -> Tensor:  # clip.py:209-216
        self.glue.ensure()
        return l2_normalize(self.vit(image))

    def encode_text(self, indices: Tensor, *, apply_pooling: bool = True, deterministic: bool = True, clip_skip: int = 0) -> Tensor:
        if clip_skip != 0:
            raise NotImplementedError("clip_skip is outside the fused path")
        net = _EmbeddingFn.apply(indices, self.token_embedding.weight, self.token_embedding.padding_idx)
        net = self.text_transformer(net)
        if not apply_pooling:
            return net
        net = _ArgmaxPoolFn.apply(net, indices)
        net = _LinearBf16Fn.apply(net, self.text_projection.weight, self.text_projection.bias)
        return l2_normalize(net)

    def forward(self, image: Tensor, text: Tensor) -> Tensor:  # multimodal/schema.py:25-30
        image_features = self.encode_image(image)
        text_features = self.encode_text(text)
        return _MatmulNTFn.apply(self.logit_scale.exp() * image_features, text_features)
