"""Tensor-level wrappers over the C-ABI: PyTorch supplies device memory and the current stream, nothing else.

Every function launches hand-written sm_90a kernels from ``libb200_cflearn.so`` on the *current* CUDA stream
(autograd's backward thread included) and raises ``B200Error`` on any failure.  No function here has a CPU or
ATen fallback.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Tuple

import torch
from torch import Tensor

from . import _cabi
from ._cabi import B200Error, call

EPI_BIAS_BF16 = 0
EPI_BIAS_GELU_BF16 = 1
EPI_BIAS_RESID_F32 = 2
EPI_DGELU_BF16 = 3
EPI_PARTIAL_F32 = 4
EPI_BIAS_QGELU_BF16 = 5  # QuickGELU (CLIP towers) flavours of 1 and 3
EPI_DQGELU_BF16 = 6
EPI_BIAS_GEGLU_BF16 = 7   # GEGLU: out0 = hg [M, 2F], out1 = a = h * gelu(gate) [M, F]  (b = W1 [2F, K])
EPI_DGEGLU_BF16 = 8       # its backward through the FF2 dgrad: out0 = dhg [M, 2F] from aux = hg  (b = W2 MN-major [K, F])
EPI_BIAS_RESID_BF16 = 9   # out0 = bf16(bf16(acc + bias) + aux), the bf16 residual stream (aux may alias out0)
EPI_BIAS_ADD_PER_IMAGE_BF16 = 10  # conv3x3 only: out0 = bf16(bf16(acc + bias) + aux[image, c]), aux bf16 [B, Cout]
EPI_BIAS_RESID_CLAMP_BF16 = 11    # conv3x3 only: 9, then +-inf -> +-bf16 max (NaN kept)

# What the torch-level checks need per epilogue (dtypes and shapes, which the C side cannot see): (out0 dtype, aux, out1).
# aux has out0's dtype: "rows" = [M, N] with out0's leading dim (conv3x3: contiguous [B*H*W, Cout]), "image" = contiguous
# [B, Cout], one row per image (conv3x3).  out1 is bf16: "rows" as for aux, "dense" = contiguous [M, N / 2] (GEGLU's a).
_BF16, _F32 = torch.bfloat16, torch.float32
EPILOGUES: Dict[int, Tuple[torch.dtype, Optional[str], Optional[str]]] = {
    EPI_BIAS_BF16: (_BF16, None, None),
    EPI_BIAS_GELU_BF16: (_BF16, None, "rows"),
    EPI_BIAS_RESID_F32: (_F32, "rows", None),
    EPI_DGELU_BF16: (_BF16, "rows", None),
    EPI_PARTIAL_F32: (_F32, None, None),
    EPI_BIAS_QGELU_BF16: (_BF16, None, "rows"),
    EPI_DQGELU_BF16: (_BF16, "rows", None),
    EPI_BIAS_GEGLU_BF16: (_BF16, None, "dense"),
    EPI_DGEGLU_BF16: (_BF16, "rows", None),
    EPI_BIAS_RESID_BF16: (_BF16, "rows", None),
    EPI_BIAS_ADD_PER_IMAGE_BF16: (_BF16, "image", None),
    EPI_BIAS_RESID_CLAMP_BF16: (_BF16, "rows", None),
}

_MAX_PARTS = 1024


def _ptr(t: Optional[Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _need_cuda(*ts: Optional[Tensor]) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise B200Error("b200 kernels need CUDA tensors (there is no CPU fallback)")


class Workspace:
    """Per-device scratch for split-K partials and column-sum partials (grown on demand, never freed)."""

    def __init__(self) -> None:
        self._bufs = {}

    def get(self, device: torch.device, nfloats: int, tag: str = "ws") -> Tensor:
        key = (device.index, tag)
        buf = self._bufs.get(key)
        if buf is None or buf.numel() < nfloats:
            buf = torch.empty(max(nfloats, 1 << 20), dtype=torch.float32, device=device)
            self._bufs[key] = buf
        return buf


WORKSPACE = Workspace()


# ----------------------------------------------------------------------------------------------------------------
# GEMM
# ----------------------------------------------------------------------------------------------------------------
def gemm(
    a: Tensor,
    b: Tensor,
    *,
    a_mn_major: bool = False,
    b_mn_major: bool = False,
    epilogue: int = EPI_BIAS_BF16,
    bias: Optional[Tensor] = None,
    out0: Optional[Tensor] = None,
    out1: Optional[Tensor] = None,
    aux: Optional[Tensor] = None,
    splits: int = 1,
    max_ctas: int = 0,
) -> Tensor:
    """C[M,N] = A . B^T on wgmma (sm_90a).  ``a``: [M,K] (or [K,M] if a_mn_major); ``b``: [N,K] (or [K,N])."""
    _need_cuda(a, b, bias, out0, out1, aux)
    if a.dtype != torch.bfloat16 or b.dtype != torch.bfloat16:
        raise B200Error("gemm operands must be bf16")
    if a.dim() != 2 or b.dim() != 2 or a.stride(1) != 1 or b.stride(1) != 1:
        raise B200Error("gemm operands must be 2-D with unit inner stride")
    if a_mn_major:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_mn_major:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    if K != Kb:
        raise B200Error(f"gemm reduction mismatch: {K} vs {Kb}")
    dtype, aux_kind, out1_kind = EPILOGUES.get(epilogue, (_BF16, None, None))  # the C side refuses unknown epilogues
    # dGEGLU: the product da is F wide, its input hg and output dhg 2F wide -- the C-ABI's N is 2F for both GEGLU epilogues
    if epilogue == EPI_DGEGLU_BF16:
        N = 2 * N
    if out0 is None:
        if epilogue == EPI_PARTIAL_F32:
            out0 = torch.empty((splits, M, N), dtype=dtype, device=a.device)
        else:  # rows stay 16-byte aligned for TMA: pad the leading dimension, hand back the [M, N] view
            npad = (N + 7) // 8 * 8
            out0 = torch.empty((M, npad), dtype=dtype, device=a.device)[:, :N]
    if out0.dtype != dtype:
        raise B200Error("gemm: out0 dtype does not match the epilogue")
    ldo = out0.stride(-2)
    if (aux_kind or out1_kind) and (tuple(out0.shape) != (M, N) or out0.stride(1) != 1):
        raise B200Error("gemm: out0 must be an [M, N] view with unit inner stride")
    for t, kind, dt, name in ((aux, aux_kind, dtype, "aux"), (out1, out1_kind, _BF16, "out1")):
        if kind == "rows" and (t is None or t.dtype != dt or tuple(t.shape) != (M, N) or t.stride() != (ldo, 1)):
            raise B200Error(f"gemm: this epilogue needs a {dt} {name} [M, N] with out0's leading dim")
    if out1_kind == "dense" and (out1 is None or out1.dtype != _BF16 or tuple(out1.shape) != (M, N // 2) or not out1.is_contiguous()):
        raise B200Error("gemm: the GEGLU epilogue needs out1 = contiguous bf16 [M, F]")
    call(
        "b200_gemm_bf16",
        a.data_ptr(), a.stride(0), int(a_mn_major),
        b.data_ptr(), b.stride(0), int(b_mn_major),
        M, N, K, epilogue, _ptr(bias), out0.data_ptr(), _ptr(out1), _ptr(aux), ldo, splits, max_ctas, _stream(),
    )
    return out0


def geglu(x: Tensor, w1: Tensor, b1: Tensor, *, max_ctas: int = 0) -> Tuple[Tensor, Tensor]:
    """GEGLU's projection and gate in one GEMM: x [M, K] bf16, w1 [2F, K] bf16 (h rows, then gate rows), b1 [2F] bf16.
    Returns (hg [M, 2F] = bf16(x w1^T + b1), a [M, F] = bf16(h * bf16(gelu(gate))))."""
    _need_cuda(x, w1, b1)
    F2 = w1.shape[0]
    if F2 % 16 != 0:
        raise B200Error("geglu: need F % 8 == 0")
    a = torch.empty((x.shape[0], F2 // 2), dtype=torch.bfloat16, device=x.device)
    hg = gemm(x, w1, bias=b1, epilogue=EPI_BIAS_GEGLU_BF16, out1=a, max_ctas=max_ctas)
    return hg, a


_NUM_SMS: Dict[int, int] = {}


def num_sms() -> int:
    dev = torch.cuda.current_device()
    if dev not in _NUM_SMS:
        _NUM_SMS[dev] = torch.cuda.get_device_properties(dev).multi_processor_count
    return _NUM_SMS[dev]


def pick_splits(M: int, N: int, K: int) -> int:
    return int(_cabi.lib().b200_gemm_pick_splits(M, N, K))


def wgrad(dy: Tensor, x: Tensor, out: Tensor, *, round_bf16: bool = True, accumulate: bool = False) -> Tensor:
    """out[N_out, K_in] (fp32) (+)= dy[M, N_out]^T . x[M, K_in]   (split-K over the M tokens, then reduce)."""
    _need_cuda(dy, x, out)
    if dy.dtype != _BF16 or x.dtype != _BF16 or dy.dim() != 2 or x.dim() != 2 or dy.shape[0] != x.shape[0]:
        raise B200Error("wgrad: need bf16 dy [M, N_out] and x [M, K_in]")
    M, n_out = dy.shape
    if out.dtype != _F32 or tuple(out.shape) != (n_out, x.shape[1]) or not out.is_contiguous():
        raise B200Error("wgrad: out must be a contiguous fp32 [N_out, K_in] tensor")
    k_in = x.shape[1]
    splits = pick_splits(n_out, k_in, M)
    part = WORKSPACE.get(dy.device, splits * n_out * k_in, "splitk")[: splits * n_out * k_in].view(splits, n_out, k_in)
    gemm(dy, x, a_mn_major=True, b_mn_major=True, epilogue=EPI_PARTIAL_F32, out0=part, splits=splits)
    call("b200_splitk_reduce", part.data_ptr(), splits, n_out * k_in, out.data_ptr(), int(round_bf16), int(accumulate), _stream())
    return out


def colsum(x: Tensor, out: Tensor, *, round_bf16: bool = True, accumulate: bool = False) -> Tensor:
    """out[cols] (fp32) (+)= sum over rows of x[rows, cols] (bf16): bias gradients."""
    _need_cuda(x, out)
    if x.dtype != _BF16 or x.dim() != 2 or x.stride(1) != 1:
        raise B200Error("colsum: x must be a 2-D bf16 view with unit inner stride")
    rows, cols = x.shape
    _dense_f32(out, cols, "out", "colsum")
    part = WORKSPACE.get(x.device, _MAX_PARTS * cols, "colsum")
    nparts = ctypes.c_int(0)
    call("b200_colsum_bf16", x.data_ptr(), x.stride(0), rows, cols, part.data_ptr(), _MAX_PARTS, ctypes.byref(nparts), _stream())
    call("b200_colsum_finish", part.data_ptr(), cols, nparts.value, cols, out.data_ptr(), int(round_bf16), int(accumulate), _stream())
    return out


def colsum_per_image(x: Tensor) -> Tuple[Tensor, Tensor]:
    """x: contiguous bf16 [B, ..., C] (the pixels of each image in between).  One pass over x returns (per_image bf16 [B, C] =
    bf16(sum over image b's rows), total fp32 [C] = float(bf16(sum over all rows))): the gradients of a per-image [B, C] table
    added to every pixel, and of the bias of the conv that wrote x."""
    _need_cuda(x)
    if x.dtype != torch.bfloat16 or x.dim() < 2 or not x.is_contiguous():
        raise B200Error("colsum_per_image: need contiguous bf16 [B, ..., C]")
    B, C = x.shape[0], x.shape[-1]
    HW = x.numel() // max(B * C, 1)
    per_image = torch.empty((B, C), dtype=torch.bfloat16, device=x.device)
    total = torch.empty(C, dtype=torch.float32, device=x.device)
    ws = WORKSPACE.get(x.device, int(_cabi.lib().b200_colsum_per_image_workspace_floats(B, HW, C)), "colsum_per_image")
    call("b200_colsum_per_image_bf16", x.data_ptr(), B, HW, C, per_image.data_ptr(), total.data_ptr(), ws.data_ptr(), _stream())
    return per_image, total


# ----------------------------------------------------------------------------------------------------------------
# LayerNorm
# ----------------------------------------------------------------------------------------------------------------
def _strided_f32(t: Tensor, rows: int, dim: int, ld: int, msg: str) -> None:
    """t: contiguous fp32 holding `rows` rows of `dim` elements `ld` apart (ld > dim: e.g. token 0 of each image)."""
    if t.dtype != _F32 or not t.is_contiguous() or ld < dim or t.numel() < (rows - 1) * ld + dim:
        raise B200Error(msg)


def layernorm_fwd(x: Tensor, gamma: Tensor, beta: Tensor, eps: float, *, rows: int, dim: int, ld_x: int,
                  y_f32: Optional[Tensor] = None) -> Tuple[Tensor, Tensor, Tensor]:
    _need_cuda(x, gamma, beta, y_f32)
    _strided_f32(x, rows, dim, ld_x, "layernorm_fwd: x must be contiguous fp32 holding rows of dim elements ld_x apart")
    _dense_f32(gamma, dim, "gamma", "layernorm_fwd")
    _dense_f32(beta, dim, "beta", "layernorm_fwd")
    if y_f32 is not None:
        _packed_rows(y_f32, rows, dim, "layernorm_fwd: y_f32 must be contiguous fp32 [rows, dim]", _F32)
    y = torch.empty((rows, dim), dtype=torch.bfloat16, device=x.device)
    mean = torch.empty(rows, dtype=torch.float32, device=x.device)
    rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
    call("b200_layernorm_fwd", x.data_ptr(), ld_x, gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), _ptr(y_f32),
         mean.data_ptr(), rstd.data_ptr(), rows, dim, float(eps), _stream())
    return y, mean, rstd


def layernorm_bwd(
    dy: Tensor, x: Tensor, gamma: Tensor, mean: Tensor, rstd: Tensor, *, rows: int, dim: int, ld_x: int,
    dres: Optional[Tensor], dx_out: Tensor, ld_dx: int, dx_bf16: Optional[Tensor],
    dgamma: Tensor, dbeta: Tensor, accumulate: bool = False, dx_colsum: Optional[Tensor] = None,
) -> None:
    """LayerNorm backward.  ``dx_colsum`` (fp32 [dim]): also receives the bf16-rounded column sums of ``dx_bf16``,
    i.e. the bias gradient of the Linear layer whose dY this dx is -- fused, no extra pass over dx."""
    _need_cuda(dy, x, gamma, mean, rstd, dres, dx_out, dx_bf16, dgamma, dbeta, dx_colsum)
    if dy.dtype not in (_BF16, _F32):
        raise B200Error("layernorm_bwd: dy must be bf16 or fp32")
    _packed_rows(dy, rows, dim, "layernorm_bwd: dy must be contiguous [rows, dim]", dy.dtype)
    _strided_f32(x, rows, dim, ld_x, "layernorm_bwd: x must be contiguous fp32 holding rows of dim elements ld_x apart")
    _strided_f32(dx_out, rows, dim, ld_dx, "layernorm_bwd: dx_out must be contiguous fp32 holding rows of dim elements ld_dx apart")
    if dres is not None:
        _strided_f32(dres, rows, dim, ld_dx, "layernorm_bwd: dres must be contiguous fp32 holding rows of dim elements ld_dx apart")
    if dx_bf16 is not None:
        _packed_rows(dx_bf16, rows, dim, "layernorm_bwd: dx_bf16 must be contiguous bf16 [rows, dim]")
    for t, n, name in ((gamma, dim, "gamma"), (mean, rows, "mean"), (rstd, rows, "rstd"), (dgamma, dim, "dgamma"), (dbeta, dim, "dbeta")):
        _dense_f32(t, n, name, "layernorm_bwd")
    if dx_colsum is not None:
        _dense_f32(dx_colsum, dim, "dx_colsum", "layernorm_bwd")
    nw = 3 if dx_colsum is not None else 2
    part = WORKSPACE.get(x.device, 3 * _MAX_PARTS * dim, "lnbwd")
    nparts = ctypes.c_int(0)
    call(
        "b200_layernorm_bwd", dy.data_ptr(), int(dy.dtype == torch.float32), x.data_ptr(), ld_x, gamma.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
        _ptr(dres), dx_out.data_ptr(), ld_dx, _ptr(dx_bf16), part.data_ptr(), _MAX_PARTS,
        ctypes.byref(nparts), rows, dim, int(dx_colsum is not None), _stream(),
    )
    adjacent = dbeta.data_ptr() == dgamma.data_ptr() + 4 * dim  # adjacent in the gradient arena: one reduction for both
    if adjacent and dx_colsum is not None:
        call("b200_colsum_finish2", part.data_ptr(), nw * dim, nparts.value, 2 * dim, dgamma.data_ptr(), 0,
             dim, dx_colsum.data_ptr(), 1, int(accumulate), _stream())
        return
    if adjacent:
        call("b200_colsum_finish", part.data_ptr(), nw * dim, nparts.value, 2 * dim, dgamma.data_ptr(), 0, int(accumulate), _stream())
    else:
        call("b200_colsum_finish", part.data_ptr(), nw * dim, nparts.value, dim, dgamma.data_ptr(), 0, int(accumulate), _stream())
        call("b200_colsum_finish", part.data_ptr() + 4 * dim, nw * dim, nparts.value, dim, dbeta.data_ptr(), 0, int(accumulate), _stream())
    if dx_colsum is not None:
        call("b200_colsum_finish", part.data_ptr() + 8 * dim, nw * dim, nparts.value, dim, dx_colsum.data_ptr(), 1, int(accumulate), _stream())


def _dense_bf16(t: Tensor, name: str) -> None:
    if t.dtype != torch.bfloat16 or t.dim() != 2 or not t.is_contiguous():
        raise B200Error(f"layernorm_bf16: {name} must be a contiguous bf16 [rows, dim] tensor")


def _dense_f32(t: Tensor, n: int, name: str, what: str = "layernorm_bf16") -> None:
    if t.dtype != torch.float32 or tuple(t.shape) != (n,) or not t.is_contiguous():
        raise B200Error(f"{what}: {name} must be a contiguous fp32 [{n}] tensor")


def layernorm_bf16_fwd(x: Tensor, gamma: Tensor, beta: Tensor, eps: float) -> Tuple[Tensor, Tensor, Tensor]:
    """LayerNorm of bf16 rows x [rows, dim] with fp32 statistics: (y = bf16(LN(x)), mean f32 [rows], rstd f32 [rows]).
    gamma / beta: contiguous fp32 [dim]."""
    _need_cuda(x, gamma, beta)
    _dense_bf16(x, "x")
    rows, dim = x.shape
    _dense_f32(gamma, dim, "gamma")
    _dense_f32(beta, dim, "beta")
    y = torch.empty_like(x)
    mean = torch.empty(rows, dtype=torch.float32, device=x.device)
    rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
    call("b200_layernorm_bf16_fwd", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
         rows, dim, float(eps), _stream())
    return y, mean, rstd


def layernorm_bf16_bwd(dy: Tensor, x: Tensor, gamma: Tensor, mean: Tensor, rstd: Tensor, *, dres: Optional[Tensor] = None,
                       dgamma: Optional[Tensor] = None, dbeta: Optional[Tensor] = None, accumulate: bool = False) -> Tuple[Tensor, Tensor, Tensor]:
    """(dx, dgamma, dbeta): dx = bf16(dres + bf16(LN'(dy))) bf16 [rows, dim]; dgamma / dbeta fp32 [dim] (``accumulate``: added)."""
    _need_cuda(dy, x, gamma, mean, rstd, dres)
    _dense_bf16(dy, "dy")
    _dense_bf16(x, "x")
    if dres is not None:
        _dense_bf16(dres, "dres")
    rows, dim = x.shape
    if dy.shape != x.shape or (dres is not None and dres.shape != x.shape):
        raise B200Error("layernorm_bf16_bwd: dy / dres must have x's shape")
    _dense_f32(gamma, dim, "gamma")
    _dense_f32(mean, rows, "mean")
    _dense_f32(rstd, rows, "rstd")
    dx = torch.empty_like(x)
    if dgamma is None:
        dgamma = torch.empty(dim, dtype=torch.float32, device=x.device)
        dbeta = torch.empty(dim, dtype=torch.float32, device=x.device)
        accumulate = False
    _need_cuda(dgamma, dbeta)
    _dense_f32(dgamma, dim, "dgamma")
    _dense_f32(dbeta, dim, "dbeta")
    part = WORKSPACE.get(x.device, 2 * _MAX_PARTS * dim, "lnbwd")
    nparts = ctypes.c_int(0)
    call("b200_layernorm_bf16_bwd", dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mean.data_ptr(), rstd.data_ptr(), _ptr(dres),
         dx.data_ptr(), part.data_ptr(), _MAX_PARTS, ctypes.byref(nparts), rows, dim, _stream())
    call("b200_colsum_finish", part.data_ptr(), 2 * dim, nparts.value, dim, dgamma.data_ptr(), 0, int(accumulate), _stream())
    call("b200_colsum_finish", part.data_ptr() + 4 * dim, 2 * dim, nparts.value, dim, dbeta.data_ptr(), 0, int(accumulate), _stream())
    return dx, dgamma, dbeta


# ----------------------------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------------------------
ATTENTION_MAX_T = 16384   # longest sequence the attention kernels accept
ATTENTION_RESIDENT_MAX_T = 256  # up to here a whole head fits in shared memory; longer sequences use the streamed kernels


def _packed_rows(t: Tensor, rows: int, width: int, msg: str, dtype: torch.dtype = _BF16) -> None:
    """t: contiguous `dtype` holding `rows` rows of `width` elements ([rows, width], or [B, T, width] with B * T = rows)."""
    if t.dtype != dtype or not t.is_contiguous() or t.dim() < 2 or t.shape[-1] != width or t.numel() != rows * width:
        raise B200Error(msg)


def _lse(lse: Tensor, B: int, H: int, T: int, what: str) -> None:
    if lse.dtype != torch.float32 or tuple(lse.shape) != (B, H, T) or not lse.is_contiguous():
        raise B200Error(f"{what}: lse must be a contiguous fp32 [B, H, T] tensor")


def attention_fwd(qkv: Tensor, B: int, T: int, H: int, *, scale: Optional[float] = None, causal: bool = False) -> Tuple[Tensor, Tensor]:
    _need_cuda(qkv)
    D = H * 64
    _packed_rows(qkv, B * T, 3 * D, "attention_fwd: qkv must be contiguous bf16 [B, T, 3*H*64]")
    out = torch.empty((B * T, D), dtype=torch.bfloat16, device=qkv.device)
    lse = torch.empty((B, H, T), dtype=torch.float32, device=qkv.device)
    sc = float(scale) if scale is not None else 0.125
    name = "b200_attention_fwd" if T <= ATTENTION_RESIDENT_MAX_T else "b200_attention_long_fwd"
    call(name, qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, T, H, 64, sc, int(causal), _stream())
    return out, lse


def attention_bwd(qkv: Tensor, out: Tensor, dout: Tensor, lse: Tensor, B: int, T: int, H: int, *, scale: Optional[float] = None, causal: bool = False, dqkv: Optional[Tensor] = None,
                  dbias: Optional[Tensor] = None) -> Tensor:
    """dqkv (bf16 [B*T, 3*H*64]).  ``dbias`` (fp32 [3*H*64]): also receives the bf16-rounded column sums of dqkv -- the
    gradient of the packed qkv bias -- accumulated inside the kernel (no separate pass over dqkv)."""
    _need_cuda(qkv, out, dout, lse, dqkv, dbias)
    D = H * 64
    _packed_rows(qkv, B * T, 3 * D, "attention_bwd: qkv must be contiguous bf16 [B, T, 3*H*64]")
    _packed_rows(out, B * T, D, "attention_bwd: out must be contiguous bf16 [B*T, H*64]")
    _packed_rows(dout, B * T, D, "attention_bwd: dout must be contiguous bf16 [B*T, H*64]")
    _lse(lse, B, H, T, "attention_bwd")
    if dqkv is None:
        dqkv = torch.empty((B * T, 3 * D), dtype=torch.bfloat16, device=qkv.device)
    _packed_rows(dqkv, B * T, 3 * D, "attention_bwd: dqkv must be contiguous bf16 [B*T, 3*H*64]")
    if dbias is not None:
        _dense_f32(dbias, 3 * D, "dbias", "attention_bwd")
    sc = float(scale) if scale is not None else 0.125
    part = WORKSPACE.get(qkv.device, B * 3 * D, "attn_dbias") if dbias is not None else None
    if T <= ATTENTION_RESIDENT_MAX_T:
        call("b200_attention_bwd", qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), B, T, H, 64, sc, int(causal),
             _ptr(part), _stream())
    else:
        ws = WORKSPACE.get(qkv.device, int(_cabi.lib().b200_attention_long_bwd_workspace_floats(B, T, H)), "attn_long")
        call("b200_attention_long_bwd", qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), B, T, H, 64, sc,
             int(causal), _ptr(part), ws.data_ptr(), _stream())
    if dbias is not None:
        call("b200_colsum_finish", part.data_ptr(), 3 * D, B, 3 * D, dbias.data_ptr(), 1, 0, _stream())
    return dqkv


def _rows_view(t: Tensor, name: str) -> int:
    if t.dtype != torch.bfloat16 or t.dim() != 2 or t.stride(1) != 1:
        raise B200Error(f"cross_attention: {name} must be a 2-D bf16 view with unit inner stride")
    return t.stride(0)


def _cross_operands(q: Tensor, k: Tensor, v: Tensor, B: int, H: int) -> Tuple[int, int, int, int, int]:
    """(ldq, ldk, Tq, Tk, Dh) of the q / k / v views."""
    ldq, ldk, ldv = _rows_view(q, "q"), _rows_view(k, "k"), _rows_view(v, "v")
    if ldk != ldv or k.shape != v.shape:
        raise B200Error("cross_attention: k and v must share shape and leading dim")
    L = q.shape[1]
    if L % H != 0 or k.shape[1] != L or q.shape[0] % B != 0 or k.shape[0] % B != 0:
        raise B200Error("cross_attention: q / k / v widths must be H * Dh and rows a multiple of B")
    return ldq, ldk, q.shape[0] // B, k.shape[0] // B, L // H


def cross_attention_fwd(q: Tensor, k: Tensor, v: Tensor, B: int, H: int, *, scale: Optional[float] = None,
                        causal: bool = False) -> Tuple[Tensor, Tensor]:
    """Attention with separate operands: q [B*Tq, >= H*Dh], k / v [B*Tk, >= H*Dh] (bf16 2-D views with unit inner stride, e.g.
    column slices of one packed projection), head h at columns [h*Dh, (h+1)*Dh).  Returns (out bf16 [B*Tq, H*Dh], lse f32 [B, H, Tq])."""
    _need_cuda(q, k, v)
    ldq, ldk, Tq, Tk, Dh = _cross_operands(q, k, v, B, H)
    out = torch.empty((B * Tq, H * Dh), dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((B, H, Tq), dtype=torch.float32, device=q.device)
    sc = float(scale) if scale is not None else Dh ** -0.5
    call("b200_cross_attention_fwd", q.data_ptr(), ldq, k.data_ptr(), v.data_ptr(), ldk, out.data_ptr(), out.stride(0), lse.data_ptr(),
         B, Tq, Tk, H, Dh, sc, int(causal), _stream())
    return out, lse


def cross_attention_bwd(q: Tensor, k: Tensor, v: Tensor, out: Tensor, dout: Tensor, lse: Tensor, B: int, H: int, *,
                        scale: Optional[float] = None, causal: bool = False, dq: Optional[Tensor] = None, dk: Optional[Tensor] = None,
                        dv: Optional[Tensor] = None) -> Tuple[Tensor, Tensor, Tensor]:
    """(dq, dk, dv) of ``cross_attention_fwd``.  dq / dk / dv may be given as views (dq with q's leading dim, dk / dv with k's), e.g.
    column slices of one packed [M, 3L] gradient for self-attention; otherwise they are allocated contiguous."""
    _need_cuda(q, k, v, out, dout, lse, dq, dk, dv)
    ldq, ldk, Tq, Tk, Dh = _cross_operands(q, k, v, B, H)
    L = q.shape[1]
    if _rows_view(dout, "dout") != _rows_view(out, "out"):
        raise B200Error("cross_attention_bwd: dout must share out's leading dim")
    if tuple(out.shape) != (B * Tq, L) or dout.shape != out.shape:
        raise B200Error("cross_attention_bwd: out / dout must have q's rows and width")
    _lse(lse, B, H, Tq, "cross_attention_bwd")
    if dq is None and dk is None and dv is None and ldq == L and ldk == L:
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    if dq is None or dk is None or dv is None:
        raise B200Error("cross_attention_bwd: give all of dq, dk, dv or none (with contiguous q / k / v)")
    if _rows_view(dq, "dq") != ldq or _rows_view(dk, "dk") != ldk or _rows_view(dv, "dv") != ldk:
        raise B200Error("cross_attention_bwd: dq must share q's leading dim, dk / dv k's")
    if dq.shape != q.shape or dk.shape != k.shape or dv.shape != k.shape:
        raise B200Error("cross_attention_bwd: dq must have q's shape, dk / dv k's")
    sc = float(scale) if scale is not None else Dh ** -0.5
    ws = WORKSPACE.get(q.device, int(_cabi.lib().b200_cross_attention_bwd_workspace_floats(B, Tq, Tk, H, Dh)), "cross_attn")
    call("b200_cross_attention_bwd", q.data_ptr(), ldq, k.data_ptr(), v.data_ptr(), ldk, out.data_ptr(), out.stride(0), dout.data_ptr(),
         lse.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, Tq, Tk, H, Dh, sc, int(causal), ws.data_ptr(), _stream())
    return dq, dk, dv


# ----------------------------------------------------------------------------------------------------------------
# patch embedding glue, loss, casts
# ----------------------------------------------------------------------------------------------------------------
def patch_im2col(x: Tensor, patch: int) -> Tensor:
    _need_cuda(x)
    B, C, Hh, Ww = x.shape
    if Hh != Ww or x.dtype != torch.float32 or not x.is_contiguous():
        raise B200Error("patch_im2col: need contiguous fp32 [B, C, S, S]")
    side = Hh // patch
    cols = torch.empty((B * side * side, C * patch * patch), dtype=torch.bfloat16, device=x.device)
    call("b200_patch_im2col", x.data_ptr(), cols.data_ptr(), B, C, Hh, patch, _stream())
    return cols


def patch_im2col_u8(x: Tensor, patch: int, division: float = 255.0, mean=None, std=None) -> Tensor:
    """uint8 [B, S, S, C] (HWC) -> normalised bf16 im2col matrix: the reference's host-side input pipeline fused into the stem."""
    _need_cuda(x)
    if x.dtype != torch.uint8 or x.dim() != 4 or not x.is_contiguous() or x.shape[1] != x.shape[2]:
        raise B200Error("patch_im2col_u8: need contiguous uint8 [B, S, S, C]")
    B, S, _, C = x.shape
    side = S // patch
    cols = torch.empty((B * side * side, C * patch * patch), dtype=torch.bfloat16, device=x.device)
    dbl = ctypes.c_double * C
    m = dbl(*[float(v) for v in mean]) if mean is not None else None
    sd = dbl(*[float(v) for v in std]) if std is not None else None
    call("b200_patch_im2col_u8", x.data_ptr(), cols.data_ptr(), B, C, S, patch, float(division), m, sd, _stream())
    return cols


def add_pos(x: Tensor, pos: Tensor, B: int, T: int, D: int) -> Tensor:
    """net[b, t, :] = x[b, t, :] + pos[t, :] (fp32): the text tower's input stage."""
    _need_cuda(x, pos)
    _packed_rows(x, B * T, D, "add_pos: x must be contiguous fp32 [B, T, D]", _F32)
    _packed_rows(pos, T, D, "add_pos: pos must be contiguous fp32 [T, D]", _F32)
    net = torch.empty((B, T, D), dtype=torch.float32, device=x.device)
    call("b200_add_pos", x.data_ptr(), pos.data_ptr(), net.data_ptr(), B, T, D, _stream())
    return net


def add_pos_bwd(dnet: Tensor, dpos: Tensor, B: int, T: int, D: int, accumulate: bool = False) -> None:
    _need_cuda(dnet, dpos)
    _packed_rows(dnet, B * T, D, "add_pos_bwd: dnet must be contiguous fp32 [B, T, D]", _F32)
    _packed_rows(dpos, T, D, "add_pos_bwd: dpos must be contiguous fp32 [T, D]", _F32)
    call("b200_add_pos_bwd", dnet.data_ptr(), dpos.data_ptr(), B, T, D, int(accumulate), _stream())


def assemble_tokens(patch: Tensor, cls: Tensor, pos: Tensor, B: int, np_: int, D: int, conv_bias: Optional[Tensor] = None) -> Tensor:
    """net[b, 0] = cls + pos[0]; net[b, t] = float(patch[b, t-1]) + pos[t].  ``conv_bias`` (bf16 [D]): the patch rows first become
    bf16(patch + bias) -- the separate bf16 bias add eager's convolution performs."""
    _need_cuda(patch, cls, pos, conv_bias)
    _packed_rows(patch, B * np_, D, "assemble_tokens: patch must be contiguous bf16 [B * np, D]")
    _packed_rows(pos, np_ + 1, D, "assemble_tokens: pos must be contiguous fp32 [np + 1, D]", _F32)
    if cls.dtype != _F32 or not cls.is_contiguous() or cls.numel() != D:
        raise B200Error("assemble_tokens: cls must be contiguous fp32 with D elements")
    if conv_bias is not None and (conv_bias.dtype != _BF16 or not conv_bias.is_contiguous() or conv_bias.numel() != D):
        raise B200Error("assemble_tokens: conv_bias must be contiguous bf16 with D elements")
    net = torch.empty((B, np_ + 1, D), dtype=torch.float32, device=patch.device)
    call("b200_assemble_tokens", patch.data_ptr(), cls.data_ptr(), pos.data_ptr(), net.data_ptr(), B, np_, D, _ptr(conv_bias), _stream())
    return net


def assemble_tokens_bwd(dnet: Tensor, dpos: Tensor, dcls: Tensor, B: int, np_: int, D: int, accumulate: bool = False) -> Tensor:
    _need_cuda(dnet, dpos, dcls)
    _packed_rows(dnet, B * (np_ + 1), D, "assemble_tokens_bwd: dnet must be contiguous fp32 [B, np + 1, D]", _F32)
    _packed_rows(dpos, np_ + 1, D, "assemble_tokens_bwd: dpos must be contiguous fp32 [np + 1, D]", _F32)
    if dcls.dtype != _F32 or not dcls.is_contiguous() or dcls.numel() != D:
        raise B200Error("assemble_tokens_bwd: dcls must be contiguous fp32 with D elements")
    dpatch = torch.empty((B * np_, D), dtype=torch.bfloat16, device=dnet.device)
    call("b200_assemble_tokens_bwd", dnet.data_ptr(), dpatch.data_ptr(), dpos.data_ptr(), dcls.data_ptr(), B, np_, D, int(accumulate), _stream())
    return dpatch


def softmax_xent(logits: Tensor, labels: Tensor, *, grad_scale: float = 1.0, need_grad: bool = True,
                 grad_scale_dev: Optional[Tensor] = None) -> Tuple[Tensor, Tensor, Optional[Tensor], Tensor]:
    """Returns (loss_mean[1], loss_rows[B], dlogits bf16 [B,C] or None, bad_label_flag int32[1])."""
    _need_cuda(logits, labels)
    Bn, C = logits.shape
    if logits.dtype != torch.bfloat16 or logits.stride(1) != 1:
        raise B200Error("softmax_xent: logits must be bf16 with unit inner stride")
    if labels.dtype != torch.int64 or labels.numel() != Bn or not labels.is_contiguous():
        raise B200Error("softmax_xent: labels must be contiguous int64 with one entry per row")
    loss_rows = torch.empty(Bn, dtype=torch.float32, device=logits.device)
    loss_mean = torch.empty(1, dtype=torch.float32, device=logits.device)
    # dlogits shares the logits' row stride (a multiple of 8 elements so the head dgrad / wgrad can TMA it)
    dlogits = torch.empty_strided((Bn, C), (logits.stride(0), 1), dtype=torch.bfloat16, device=logits.device) if need_grad else None
    bad = torch.zeros(1, dtype=torch.int32, device=logits.device)
    call(
        "b200_softmax_xent_fwd_bwd", logits.data_ptr(), logits.stride(0), labels.data_ptr(), loss_rows.data_ptr(),
        loss_mean.data_ptr(), _ptr(dlogits), bad.data_ptr(), Bn, C, float(grad_scale), _ptr(grad_scale_dev), _stream(),
    )
    return loss_mean, loss_rows, dlogits, bad


def cast_bf16(src: Tensor, dst: Optional[Tensor] = None) -> Tensor:
    _need_cuda(src)
    if src.dtype != torch.float32 or not src.is_contiguous():
        raise B200Error("cast_bf16: need contiguous fp32")
    if dst is None:
        dst = torch.empty(src.shape, dtype=torch.bfloat16, device=src.device)
    call("b200_cast_f32_to_bf16", src.data_ptr(), dst.data_ptr(), src.numel(), _stream())
    return dst


def fill_f32(dst: Tensor, value: float) -> Tensor:
    _need_cuda(dst)
    if dst.dtype != _F32 or not dst.is_contiguous():
        raise B200Error("fill_f32: need contiguous fp32")
    call("b200_fill_f32", dst.data_ptr(), float(value), dst.numel(), _stream())
    return dst


# ----------------------------------------------------------------------------------------------------------------
# GroupNorm(32) + SiLU on channels-last activations (SD-v1.5 UNet, SURVEY.md 8f N3)
# ----------------------------------------------------------------------------------------------------------------
def groupnorm_silu_fwd(x: Tensor, gamma: Tensor, beta: Tensor, eps: float, *, silu: bool = True) -> Tuple[Tensor, Tensor, Tensor]:
    """x: bf16 [B, HW, C] (channels last).  Returns (y bf16 [B, HW, C], mean f32 [B, 32], rstd f32 [B, 32])."""
    _need_cuda(x, gamma, beta)
    if x.dtype != torch.bfloat16 or x.dim() != 3 or not x.is_contiguous():
        raise B200Error("groupnorm_silu_fwd: need contiguous bf16 [B, HW, C]")
    B, HW, C = x.shape
    _dense_f32(gamma, C, "gamma", "groupnorm_silu_fwd")
    _dense_f32(beta, C, "beta", "groupnorm_silu_fwd")
    y = torch.empty_like(x)
    mean = torch.empty((B, 32), dtype=torch.float32, device=x.device)
    rstd = torch.empty((B, 32), dtype=torch.float32, device=x.device)
    ws = WORKSPACE.get(x.device, int(_cabi.lib().b200_groupnorm_workspace_floats(B, HW, C)), "groupnorm")
    call("b200_groupnorm_silu_fwd", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
         ws.data_ptr(), B, HW, C, float(eps), int(silu), _stream())
    return y, mean, rstd


def groupnorm_silu_bwd(x: Tensor, dy: Tensor, gamma: Tensor, beta: Tensor, mean: Tensor, rstd: Tensor, *, silu: bool = True,
                       dgamma: Optional[Tensor] = None, dbeta: Optional[Tensor] = None, accumulate: bool = False) -> Tuple[Tensor, Tensor, Tensor]:
    _need_cuda(x, dy, gamma, beta, mean, rstd, dgamma, dbeta)
    if x.dtype != torch.bfloat16 or x.dim() != 3 or not x.is_contiguous():
        raise B200Error("groupnorm_silu_bwd: need contiguous bf16 x [B, HW, C]")
    B, HW, C = x.shape
    for t, name in ((mean, "mean"), (rstd, "rstd")):
        if t.dtype != _F32 or tuple(t.shape) != (B, 32) or not t.is_contiguous():
            raise B200Error(f"groupnorm_silu_bwd: {name} must be a contiguous fp32 [B, 32] tensor")
    _dense_f32(gamma, C, "gamma", "groupnorm_silu_bwd")
    _dense_f32(beta, C, "beta", "groupnorm_silu_bwd")
    if dy.dtype != torch.bfloat16 or dy.shape != x.shape or not dy.is_contiguous():
        raise B200Error("groupnorm_silu_bwd: dy must be contiguous bf16 with x's shape")
    dx = torch.empty_like(x)
    if dgamma is None:
        dgamma = torch.empty(C, dtype=torch.float32, device=x.device)
        dbeta = torch.empty(C, dtype=torch.float32, device=x.device)
        accumulate = False
    _dense_f32(dgamma, C, "dgamma", "groupnorm_silu_bwd")
    _dense_f32(dbeta, C, "dbeta", "groupnorm_silu_bwd")
    ws = WORKSPACE.get(x.device, int(_cabi.lib().b200_groupnorm_workspace_floats(B, HW, C)), "groupnorm")
    call("b200_groupnorm_silu_bwd", x.data_ptr(), dy.data_ptr(), gamma.data_ptr(), beta.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
         dx.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), ws.data_ptr(), B, HW, C, int(silu), int(accumulate), _stream())
    return dx, dgamma, dbeta


def pack_conv3x3_weight(w: Tensor) -> Tensor:
    """[Cout, Cin, 3, 3] (the reference's Conv2d.weight) -> bf16 [Cout, 9 * Cin], tap-major (k = (ky * 3 + kx) * Cin + ci)."""
    co, ci, kh, kw = w.shape
    if kh != 3 or kw != 3:
        raise B200Error("pack_conv3x3_weight: 3x3 kernels only")
    return w.permute(0, 2, 3, 1).reshape(co, 9 * ci).to(torch.bfloat16).contiguous()


def pack_conv3x3_weight_dgrad(w: Tensor) -> Tensor:
    """Weights of the INPUT-gradient convolution: [Cin, 9 * Cout] with the taps flipped (dx = conv3x3(dy, flip(w)^T))."""
    return pack_conv3x3_weight(w.flip(2, 3).transpose(0, 1))


def conv3x3_wgrad(dy: Tensor, x: Tensor, out: Optional[Tensor] = None, *, round_bf16: bool = True, accumulate: bool = False) -> Tensor:
    """Weight gradient of ``conv3x3``: dy bf16 [B, H, W, Cout], x bf16 [B, H, W, Cin] -> fp32 [Cout, 9 * Cin] in the PACKED layout
    of ``pack_conv3x3_weight`` (``unpack_conv3x3_weight`` gives the reference's [Cout, Cin, 3, 3]).  One split-K implicit GEMM over
    the B * H * W pixels plus the split-K reduction; ``round_bf16`` rounds like eager's bf16 conv backward does."""
    _need_cuda(dy, x, out)
    if dy.dtype != torch.bfloat16 or x.dtype != torch.bfloat16 or dy.dim() != 4 or x.dim() != 4 or not dy.is_contiguous() or not x.is_contiguous():
        raise B200Error("conv3x3_wgrad: need contiguous bf16 dy [B, H, W, Cout] and x [B, H, W, Cin]")
    B, H, W, Cin = x.shape
    Cout = dy.shape[3]
    if tuple(dy.shape[:3]) != (B, H, W):
        raise B200Error("conv3x3_wgrad: dy and x disagree on [B, H, W]")
    if out is None:
        out = torch.empty((Cout, 9 * Cin), dtype=torch.float32, device=x.device)
        accumulate = False
    n = Cout * 9 * Cin
    splits = pick_splits(Cout, 9 * Cin, B * H * W)
    part = WORKSPACE.get(x.device, splits * n, "splitk")[: splits * n]
    call("b200_conv3x3_wgrad_nhwc_bf16", dy.data_ptr(), Cout, x.data_ptr(), part.data_ptr(), B, H, W, Cin, Cout, splits, _stream())
    call("b200_splitk_reduce", part.data_ptr(), splits, n, out.data_ptr(), int(round_bf16), int(accumulate), _stream())
    return out


def unpack_conv3x3_weight(w_packed: Tensor, cin: int) -> Tensor:
    """[Cout, 9 * Cin] (tap-major) -> [Cout, Cin, 3, 3], the reference's Conv2d.weight layout."""
    co = w_packed.shape[0]
    return w_packed.view(co, 3, 3, cin).permute(0, 3, 1, 2).contiguous()


def conv3x3(x: Tensor, w_packed: Tensor, bias: Optional[Tensor] = None, *, epilogue: int = EPI_BIAS_BF16, aux: Optional[Tensor] = None) -> Tensor:
    """x: bf16 [B, H, W, Cin] channels-last; w_packed: bf16 [Cout, 9 * Cin] -> bf16 (or fp32 with the residual epilogue) [B, H, W, Cout].
    ``EPI_BIAS_ADD_PER_IMAGE_BF16``: aux = contiguous bf16 [B, Cout], added to every pixel of its image;
    ``EPI_BIAS_RESID_CLAMP_BF16``: aux = contiguous bf16 [B, H, W, Cout] (or [B * H * W, Cout]), the sum clamped to bf16's finite range."""
    _need_cuda(x, w_packed, bias, aux)
    if x.dtype != torch.bfloat16 or x.dim() != 4 or not x.is_contiguous() or w_packed.dtype != torch.bfloat16 or not w_packed.is_contiguous():
        raise B200Error("conv3x3: need contiguous bf16 x [B, H, W, Cin] and w_packed [Cout, 9 * Cin]")
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    if w_packed.shape[1] != 9 * Cin or Cout % 8 != 0:
        raise B200Error("conv3x3: weight shape does not match (need [Cout, 9 * Cin], Cout % 8 == 0)")
    dtype, aux_kind, _ = EPILOGUES.get(epilogue, (_BF16, None, None))  # the C side refuses the others
    if aux_kind:
        rows = B if aux_kind == "image" else B * H * W
        if aux is None or aux.dtype != dtype or not aux.is_contiguous() or aux.numel() != rows * Cout or aux.shape[-1] != Cout:
            raise B200Error(f"conv3x3: this epilogue needs a contiguous {dtype} aux with {rows} rows of {Cout}")
    out = torch.empty((B, H, W, Cout), dtype=dtype, device=x.device)
    call("b200_conv3x3_nhwc_bf16", x.data_ptr(), w_packed.data_ptr(), _ptr(bias), out.data_ptr(), _ptr(aux), Cout, B, H, W, Cin, Cout, epilogue, _stream())
    return out
