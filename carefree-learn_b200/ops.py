"""Tensor-level wrappers over the C-ABI: PyTorch supplies device memory and the current stream, nothing else.

Every function launches hand-written sm_90a kernels from ``libb200_cflearn.so`` on the *current* CUDA stream
(autograd's backward thread included) and raises ``B200Error`` on any failure.  No function here has a CPU or
ATen fallback.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Sequence, Tuple

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


def _check(what: str, name: str, t: Optional[Tensor], dtype: Optional[torch.dtype], shape: Optional[Tuple[Optional[int], ...]] = None,
           *, numel: Optional[int] = None, rows: Optional[int] = None, width: int = 0, ld: Optional[int] = None, view: bool = False,
           contiguous: bool = True, optional: bool = False) -> int:
    """Refuses, with ``B200Error("<what>: <name> must be ...")``, a tensor the library cannot take as ``name``.  ``t`` must be a
    CUDA tensor of ``dtype`` (None: any), contiguous unless ``contiguous=False``, and where given
      - ``shape``: exactly this shape (None entries: any size); ``numel``: this many elements;
      - ``rows`` / ``width``: ``rows`` rows of ``width`` elements, [rows, width] or any [..., width] whose leading sizes multiply
        to ``rows``; with ``ld``, rows ``ld >= width`` elements apart inside ``t`` (e.g. token 0 of each image);
      - ``view``: instead of contiguous, 2-D with unit inner stride; the row stride is returned (the leading dim the library takes).
    ``optional``: None passes."""
    if t is None and optional:
        return 0
    ok = t is not None and t.is_cuda and (dtype is None or t.dtype == dtype)
    if ok and view:
        ok = t.dim() == 2 and t.stride(1) == 1
    elif ok and contiguous:
        ok = t.is_contiguous()
    if ok and shape is not None:
        ok = t.dim() == len(shape) and all(s is None or s == n for s, n in zip(shape, t.shape))
    if ok and numel is not None:
        ok = t.numel() == numel
    if ok and rows is not None and ld is not None:
        ok = width <= ld and t.numel() >= (rows - 1) * ld + width
    elif ok and rows is not None:
        ok = t.dim() >= 2 and t.shape[-1] == width and t.numel() == rows * width
    if not ok:
        need = ["a 2-D view with unit inner stride" if view else "contiguous" if contiguous else "",
                "[" + ", ".join("*" if s is None else str(s) for s in shape) + "]" if shape is not None else "",
                f"{numel} elements" if numel is not None else "",
                f"{rows} rows of {width}" + (f" elements {ld} apart" if ld is not None else "") if rows is not None else ""]
        got = "None" if t is None else f"{t.dtype} {list(t.shape)} with strides {list(t.stride())} on {t.device}"
        kind = f"a CUDA {dtype} tensor" if dtype is not None else "a CUDA tensor"
        raise B200Error(f"{what}: {name} must be {kind}: " + ", ".join(n for n in need if n) + f" (got {got})")
    return t.stride(0) if view else 0


def _colsum_finish(part: Tensor, part_ld: int, nparts: int, col0: int, cols: int, out: Tensor, *, round_bf16: bool = False,
                   accumulate: bool = False) -> None:
    """out[:cols] (+)= the column sums of part[:nparts, col0 : col0 + cols] (fp32 partials, rows part_ld apart): the second pass
    of every split reduction (bias, LayerNorm and FCNN parameter gradients)."""
    call("b200_colsum_finish", part.data_ptr() + 4 * col0, part_ld, nparts, cols, out.data_ptr(), int(round_bf16), int(accumulate),
         _stream())


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
    _check("gemm", "a", a, _BF16, view=True)
    _check("gemm", "b", b, _BF16, view=True)
    _check("gemm", "bias", bias, None, contiguous=False, optional=True)
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
    if aux_kind or out1_kind:
        _check("gemm", "out0", out0, dtype, (M, N), view=True)
    else:
        _check("gemm", "out0", out0, dtype, contiguous=False)
    ldo = out0.stride(-2)
    for t, kind, dt, name in ((aux, aux_kind, dtype, "aux"), (out1, out1_kind, _BF16, "out1")):
        if kind == "rows" and _check("gemm", name, t, dt, (M, N), view=True) != ldo:
            raise B200Error(f"gemm: {name} must have out0's leading dim {ldo}")
        if kind == "dense":
            _check("gemm", name, t, _BF16, (M, N // 2))
        if kind is None:
            _check("gemm", name, t, None, contiguous=False, optional=True)
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
    F2 = w1.shape[0]
    if F2 % 16 != 0:
        raise B200Error("geglu: need F % 8 == 0")
    a = torch.empty((x.shape[0], F2 // 2), dtype=torch.bfloat16, device=x.device)
    hg = gemm(x, w1, bias=b1, epilogue=EPI_BIAS_GEGLU_BF16, out1=a, max_ctas=max_ctas)
    return hg, a


def tma_aligned(t: Tensor) -> Tensor:
    """``t`` (bf16 [rows, cols]) with rows TMA can load: itself if its inner stride is 1 and its row stride a multiple of 8
    elements (16 bytes), else a copy in zero-padded rows (e.g. a gradient produced by a foreign loss)."""
    if t.stride(1) == 1 and t.stride(0) % 8 == 0:
        return t
    padded = torch.zeros((t.shape[0], (t.shape[1] + 7) // 8 * 8), dtype=torch.bfloat16, device=t.device)
    padded[:, : t.shape[1]].copy_(t)
    return padded[:, : t.shape[1]]


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
    _check("wgrad", "dy", dy, _BF16, view=True)
    M, n_out = dy.shape
    _check("wgrad", "x", x, _BF16, (M, None), view=True)
    k_in = x.shape[1]
    _check("wgrad", "out", out, _F32, (n_out, k_in))
    splits = pick_splits(n_out, k_in, M)
    part = WORKSPACE.get(dy.device, splits * n_out * k_in, "splitk")[: splits * n_out * k_in].view(splits, n_out, k_in)
    gemm(dy, x, a_mn_major=True, b_mn_major=True, epilogue=EPI_PARTIAL_F32, out0=part, splits=splits)
    call("b200_splitk_reduce", part.data_ptr(), splits, n_out * k_in, out.data_ptr(), int(round_bf16), int(accumulate), _stream())
    return out


def colsum(x: Tensor, out: Tensor, *, round_bf16: bool = True, accumulate: bool = False) -> Tensor:
    """out[cols] (fp32) (+)= sum over rows of x[rows, cols] (bf16): bias gradients."""
    ldx = _check("colsum", "x", x, _BF16, view=True)
    rows, cols = x.shape
    _check("colsum", "out", out, _F32, (cols,))
    part = WORKSPACE.get(x.device, _MAX_PARTS * cols, "colsum")
    nparts = ctypes.c_int(0)
    call("b200_colsum_bf16", x.data_ptr(), ldx, rows, cols, part.data_ptr(), _MAX_PARTS, ctypes.byref(nparts), _stream())
    _colsum_finish(part, cols, nparts.value, 0, cols, out, round_bf16=round_bf16, accumulate=accumulate)
    return out


def colsum_per_image(x: Tensor) -> Tuple[Tensor, Tensor]:
    """x: contiguous bf16 [B, ..., C] (the pixels of each image in between).  One pass over x returns (per_image bf16 [B, C] =
    bf16(sum over image b's rows), total fp32 [C] = float(bf16(sum over all rows))): the gradients of a per-image [B, C] table
    added to every pixel, and of the bias of the conv that wrote x."""
    C = x.shape[-1]
    _check("colsum_per_image", "x", x, _BF16, rows=x.numel() // max(C, 1), width=C)
    B = x.shape[0]
    HW = x.numel() // max(B * C, 1)
    per_image = torch.empty((B, C), dtype=torch.bfloat16, device=x.device)
    total = torch.empty(C, dtype=torch.float32, device=x.device)
    ws = WORKSPACE.get(x.device, int(_cabi.lib().b200_colsum_per_image_workspace_floats(B, HW, C)), "colsum_per_image")
    call("b200_colsum_per_image_bf16", x.data_ptr(), B, HW, C, per_image.data_ptr(), total.data_ptr(), ws.data_ptr(), _stream())
    return per_image, total


# ----------------------------------------------------------------------------------------------------------------
# LayerNorm
# ----------------------------------------------------------------------------------------------------------------
def layernorm_fwd(x: Tensor, gamma: Tensor, beta: Tensor, eps: float, *, rows: int, dim: int, ld_x: int,
                  y_f32: Optional[Tensor] = None) -> Tuple[Tensor, Tensor, Tensor]:
    _check("layernorm_fwd", "x", x, _F32, rows=rows, width=dim, ld=ld_x)
    _check("layernorm_fwd", "gamma", gamma, _F32, (dim,))
    _check("layernorm_fwd", "beta", beta, _F32, (dim,))
    _check("layernorm_fwd", "y_f32", y_f32, _F32, rows=rows, width=dim, optional=True)
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
    what = "layernorm_bwd"
    _check(what, "dy", dy, _F32 if dy.dtype == _F32 else _BF16, rows=rows, width=dim)  # bf16, or fp32 (an fp32 residual stream)
    _check(what, "x", x, _F32, rows=rows, width=dim, ld=ld_x)
    _check(what, "dx_out", dx_out, _F32, rows=rows, width=dim, ld=ld_dx)
    _check(what, "dres", dres, _F32, rows=rows, width=dim, ld=ld_dx, optional=True)
    _check(what, "dx_bf16", dx_bf16, _BF16, rows=rows, width=dim, optional=True)
    for t, n, name in ((gamma, dim, "gamma"), (mean, rows, "mean"), (rstd, rows, "rstd"), (dgamma, dim, "dgamma"), (dbeta, dim, "dbeta")):
        _check(what, name, t, _F32, (n,))
    _check(what, "dx_colsum", dx_colsum, _F32, (dim,), optional=True)
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
        _colsum_finish(part, nw * dim, nparts.value, 0, 2 * dim, dgamma, accumulate=accumulate)
    else:
        _colsum_finish(part, nw * dim, nparts.value, 0, dim, dgamma, accumulate=accumulate)
        _colsum_finish(part, nw * dim, nparts.value, dim, dim, dbeta, accumulate=accumulate)
    if dx_colsum is not None:
        _colsum_finish(part, nw * dim, nparts.value, 2 * dim, dim, dx_colsum, round_bf16=True, accumulate=accumulate)


def layernorm_bf16_fwd(x: Tensor, gamma: Tensor, beta: Tensor, eps: float) -> Tuple[Tensor, Tensor, Tensor]:
    """LayerNorm of bf16 rows x [rows, dim] with fp32 statistics: (y = bf16(LN(x)), mean f32 [rows], rstd f32 [rows]).
    gamma / beta: contiguous fp32 [dim]."""
    _check("layernorm_bf16_fwd", "x", x, _BF16, (None, None))
    rows, dim = x.shape
    _check("layernorm_bf16_fwd", "gamma", gamma, _F32, (dim,))
    _check("layernorm_bf16_fwd", "beta", beta, _F32, (dim,))
    y = torch.empty_like(x)
    mean = torch.empty(rows, dtype=torch.float32, device=x.device)
    rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
    call("b200_layernorm_bf16_fwd", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
         rows, dim, float(eps), _stream())
    return y, mean, rstd


def layernorm_bf16_bwd(dy: Tensor, x: Tensor, gamma: Tensor, mean: Tensor, rstd: Tensor, *, dres: Optional[Tensor] = None,
                       dgamma: Optional[Tensor] = None, dbeta: Optional[Tensor] = None, accumulate: bool = False) -> Tuple[Tensor, Tensor, Tensor]:
    """(dx, dgamma, dbeta): dx = bf16(dres + bf16(LN'(dy))) bf16 [rows, dim]; dgamma / dbeta fp32 [dim] (``accumulate``: added)."""
    what = "layernorm_bf16_bwd"
    _check(what, "x", x, _BF16, (None, None))
    rows, dim = x.shape
    _check(what, "dy", dy, _BF16, (rows, dim))
    _check(what, "dres", dres, _BF16, (rows, dim), optional=True)
    for t, n, name in ((gamma, dim, "gamma"), (mean, rows, "mean"), (rstd, rows, "rstd")):
        _check(what, name, t, _F32, (n,))
    dx = torch.empty_like(x)
    if dgamma is None:
        dgamma = torch.empty(dim, dtype=torch.float32, device=x.device)
        dbeta = torch.empty(dim, dtype=torch.float32, device=x.device)
        accumulate = False
    _check(what, "dgamma", dgamma, _F32, (dim,))
    _check(what, "dbeta", dbeta, _F32, (dim,))
    part = WORKSPACE.get(x.device, 2 * _MAX_PARTS * dim, "lnbwd")
    nparts = ctypes.c_int(0)
    call("b200_layernorm_bf16_bwd", dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mean.data_ptr(), rstd.data_ptr(), _ptr(dres),
         dx.data_ptr(), part.data_ptr(), _MAX_PARTS, ctypes.byref(nparts), rows, dim, _stream())
    _colsum_finish(part, 2 * dim, nparts.value, 0, dim, dgamma, accumulate=accumulate)
    _colsum_finish(part, 2 * dim, nparts.value, dim, dim, dbeta, accumulate=accumulate)
    return dx, dgamma, dbeta


# ----------------------------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------------------------
ATTENTION_MAX_T = 16384   # longest sequence the attention kernels accept
ATTENTION_RESIDENT_MAX_T = 256  # up to here a whole head fits in shared memory; longer sequences use the streamed kernels


def attention_fwd(qkv: Tensor, B: int, T: int, H: int, *, scale: Optional[float] = None, causal: bool = False) -> Tuple[Tensor, Tensor]:
    D = H * 64
    _check("attention_fwd", "qkv", qkv, _BF16, rows=B * T, width=3 * D)
    out = torch.empty((B * T, D), dtype=torch.bfloat16, device=qkv.device)
    lse = torch.empty((B, H, T), dtype=torch.float32, device=qkv.device)
    sc = float(scale) if scale is not None else 0.125
    name = "b200_attention_fwd" if T <= ATTENTION_RESIDENT_MAX_T else "b200_attention_long_fwd"
    call(name, qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, T, H, 64, sc, int(causal), _stream())
    return out, lse


def attention_bwd(qkv: Tensor, out: Tensor, dout: Tensor, lse: Tensor, B: int, T: int, H: int, *, scale: Optional[float] = None, causal: bool = False, dqkv: Optional[Tensor] = None,
                  dbias: Optional[Tensor] = None, accumulate: bool = False) -> Tensor:
    """dqkv (bf16 [B*T, 3*H*64]).  ``dbias`` (fp32 [3*H*64]): also receives the bf16-rounded column sums of dqkv -- the
    gradient of the packed qkv bias -- accumulated inside the kernel (no separate pass over dqkv); ``accumulate``: added to
    ``dbias`` instead of overwriting it."""
    what, D = "attention_bwd", H * 64
    _check(what, "qkv", qkv, _BF16, rows=B * T, width=3 * D)
    _check(what, "out", out, _BF16, rows=B * T, width=D)
    _check(what, "dout", dout, _BF16, rows=B * T, width=D)
    _check(what, "lse", lse, _F32, (B, H, T))
    if dqkv is None:
        dqkv = torch.empty((B * T, 3 * D), dtype=torch.bfloat16, device=qkv.device)
    _check(what, "dqkv", dqkv, _BF16, rows=B * T, width=3 * D)
    _check(what, "dbias", dbias, _F32, (3 * D,), optional=True)
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
        _colsum_finish(part, 3 * D, B, 0, 3 * D, dbias, round_bf16=True, accumulate=accumulate)
    return dqkv


def _cross_operands(q: Tensor, k: Tensor, v: Tensor, B: int, H: int) -> Tuple[int, int, int, int, int]:
    """(ldq, ldk, Tq, Tk, Dh) of the q / k / v views."""
    ldq, ldk, ldv = (_check("cross_attention", name, t, _BF16, view=True) for name, t in (("q", q), ("k", k), ("v", v)))
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
    what = "cross_attention_bwd"
    ldq, ldk, Tq, Tk, Dh = _cross_operands(q, k, v, B, H)
    L = q.shape[1]
    ldo = _check(what, "out", out, _BF16, (B * Tq, L), view=True)
    if _check(what, "dout", dout, _BF16, (B * Tq, L), view=True) != ldo:
        raise B200Error(f"{what}: dout must share out's leading dim")
    _check(what, "lse", lse, _F32, (B, H, Tq))
    if dq is None and dk is None and dv is None and ldq == L and ldk == L:
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    if dq is None or dk is None or dv is None:
        raise B200Error(f"{what}: give all of dq, dk, dv or none (with contiguous q / k / v)")
    for name, t, like, ld in (("dq", dq, q, ldq), ("dk", dk, k, ldk), ("dv", dv, k, ldk)):
        if _check(what, name, t, _BF16, tuple(like.shape), view=True) != ld:
            raise B200Error(f"{what}: dq must share q's leading dim, dk / dv k's")
    sc = float(scale) if scale is not None else Dh ** -0.5
    ws = WORKSPACE.get(q.device, int(_cabi.lib().b200_cross_attention_bwd_workspace_floats(B, Tq, Tk, H, Dh)), "cross_attn")
    call("b200_cross_attention_bwd", q.data_ptr(), ldq, k.data_ptr(), v.data_ptr(), ldk, out.data_ptr(), ldo, dout.data_ptr(),
         lse.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, Tq, Tk, H, Dh, sc, int(causal), ws.data_ptr(), _stream())
    return dq, dk, dv


# ----------------------------------------------------------------------------------------------------------------
# glue (patch embedding, CLIP text: integer-indexed row moves, bit-exact), losses, casts
# ----------------------------------------------------------------------------------------------------------------
def patch_im2col(x: Tensor, patch: int) -> Tensor:
    _check("patch_im2col", "x", x, _F32, (None, None, None, None))
    B, C, Hh, Ww = x.shape
    if Hh != Ww:
        raise B200Error("patch_im2col: x must be square images [B, C, S, S]")
    side = Hh // patch
    cols = torch.empty((B * side * side, C * patch * patch), dtype=torch.bfloat16, device=x.device)
    call("b200_patch_im2col", x.data_ptr(), cols.data_ptr(), B, C, Hh, patch, _stream())
    return cols


def patch_im2col_u8(x: Tensor, patch: int, division: float = 255.0, mean=None, std=None) -> Tensor:
    """uint8 [B, S, S, C] (HWC) -> normalised bf16 im2col matrix: the reference's host-side input pipeline fused into the stem."""
    _check("patch_im2col_u8", "x", x, torch.uint8, (None, None, None, None))
    B, S, Ww, C = x.shape
    if S != Ww:
        raise B200Error("patch_im2col_u8: x must be square images [B, S, S, C]")
    side = S // patch
    cols = torch.empty((B * side * side, C * patch * patch), dtype=torch.bfloat16, device=x.device)
    dbl = ctypes.c_double * C
    m = dbl(*[float(v) for v in mean]) if mean is not None else None
    sd = dbl(*[float(v) for v in std]) if std is not None else None
    call("b200_patch_im2col_u8", x.data_ptr(), cols.data_ptr(), B, C, S, patch, float(division), m, sd, _stream())
    return cols


def add_pos(x: Tensor, pos: Tensor, B: int, T: int, D: int) -> Tensor:
    """net[b, t, :] = x[b, t, :] + pos[t, :] (fp32): the text tower's input stage."""
    _check("add_pos", "x", x, _F32, rows=B * T, width=D)
    _check("add_pos", "pos", pos, _F32, rows=T, width=D)
    net = torch.empty((B, T, D), dtype=torch.float32, device=x.device)
    call("b200_add_pos", x.data_ptr(), pos.data_ptr(), net.data_ptr(), B, T, D, _stream())
    return net


def add_pos_bwd(dnet: Tensor, dpos: Tensor, B: int, T: int, D: int, accumulate: bool = False) -> None:
    _check("add_pos_bwd", "dnet", dnet, _F32, rows=B * T, width=D)
    _check("add_pos_bwd", "dpos", dpos, _F32, rows=T, width=D)
    call("b200_add_pos_bwd", dnet.data_ptr(), dpos.data_ptr(), B, T, D, int(accumulate), _stream())


def assemble_tokens(patch: Tensor, cls: Tensor, pos: Tensor, B: int, np_: int, D: int, conv_bias: Optional[Tensor] = None) -> Tensor:
    """net[b, 0] = cls + pos[0]; net[b, t] = float(patch[b, t-1]) + pos[t].  ``conv_bias`` (bf16 [D]): the patch rows first become
    bf16(patch + bias) -- the separate bf16 bias add eager's convolution performs."""
    _check("assemble_tokens", "patch", patch, _BF16, rows=B * np_, width=D)
    _check("assemble_tokens", "pos", pos, _F32, rows=np_ + 1, width=D)
    _check("assemble_tokens", "cls", cls, _F32, numel=D)
    _check("assemble_tokens", "conv_bias", conv_bias, _BF16, numel=D, optional=True)
    net = torch.empty((B, np_ + 1, D), dtype=torch.float32, device=patch.device)
    call("b200_assemble_tokens", patch.data_ptr(), cls.data_ptr(), pos.data_ptr(), net.data_ptr(), B, np_, D, _ptr(conv_bias), _stream())
    return net


def assemble_tokens_bwd(dnet: Tensor, dpos: Tensor, dcls: Tensor, B: int, np_: int, D: int, accumulate: bool = False) -> Tensor:
    _check("assemble_tokens_bwd", "dnet", dnet, _F32, rows=B * (np_ + 1), width=D)
    _check("assemble_tokens_bwd", "dpos", dpos, _F32, rows=np_ + 1, width=D)
    _check("assemble_tokens_bwd", "dcls", dcls, _F32, numel=D)
    dpatch = torch.empty((B * np_, D), dtype=torch.bfloat16, device=dnet.device)
    call("b200_assemble_tokens_bwd", dnet.data_ptr(), dpatch.data_ptr(), dpos.data_ptr(), dcls.data_ptr(), B, np_, D, int(accumulate), _stream())
    return dpatch


def softmax_xent(logits: Tensor, labels: Tensor, *, grad_scale: float = 1.0, need_grad: bool = True,
                 grad_scale_dev: Optional[Tensor] = None) -> Tuple[Tensor, Tensor, Optional[Tensor], Tensor]:
    """Returns (loss_mean[1], loss_rows[B], dlogits bf16 [B,C] or None, bad_label_flag int32[1])."""
    ldl = _check("softmax_xent", "logits", logits, _BF16, view=True)
    Bn, C = logits.shape
    _check("softmax_xent", "labels", labels, torch.int64, numel=Bn)
    loss_rows = torch.empty(Bn, dtype=torch.float32, device=logits.device)
    loss_mean = torch.empty(1, dtype=torch.float32, device=logits.device)
    # dlogits shares the logits' row stride (a multiple of 8 elements so the head dgrad / wgrad can TMA it)
    dlogits = torch.empty_strided((Bn, C), (ldl, 1), dtype=torch.bfloat16, device=logits.device) if need_grad else None
    bad = torch.zeros(1, dtype=torch.int32, device=logits.device)
    call(
        "b200_softmax_xent_fwd_bwd", logits.data_ptr(), ldl, labels.data_ptr(), loss_rows.data_ptr(),
        loss_mean.data_ptr(), _ptr(dlogits), bad.data_ptr(), Bn, C, float(grad_scale), _ptr(grad_scale_dev), _stream(),
    )
    return loss_mean, loss_rows, dlogits, bad


def symmetric_xent(logits: Tensor, *, dlogits: Optional[Tensor] = None, grad_scale: float = 1.0,
                   grad_scale_dev: Optional[Tensor] = None) -> Tensor:
    """CLIP's contrastive loss (CE(L, arange) + CE(L^T, arange)) / 2 of the square bf16 logits L [B, B] (unit inner stride), fp32
    [1].  ``dlogits`` (a bf16 [B, B] view with L's row stride) also receives the gradient, scaled by ``grad_scale`` (and by the
    device fp32 [1] ``grad_scale_dev``)."""
    what = "symmetric_xent"
    ldl = _check(what, "logits", logits, _BF16, view=True)
    Bn = logits.shape[0]
    if logits.shape[1] != Bn:
        raise B200Error(f"{what}: logits must be square, got {list(logits.shape)}")
    if dlogits is not None and _check(what, "dlogits", dlogits, _BF16, (Bn, Bn), view=True) != ldl:
        raise B200Error(f"{what}: dlogits must share logits' row stride")
    _check(what, "grad_scale_dev", grad_scale_dev, _F32, (1,), optional=True)
    loss = torch.empty(1, dtype=torch.float32, device=logits.device)
    ws = torch.empty(2 * Bn, dtype=torch.float32, device=logits.device)
    call("b200_symmetric_xent_fwd_bwd", logits.data_ptr(), ldl, loss.data_ptr(), _ptr(dlogits), ws.data_ptr(), Bn, float(grad_scale),
         _ptr(grad_scale_dev), _stream())
    return loss


def cast_bf16(src: Tensor, dst: Optional[Tensor] = None) -> Tensor:
    _check("cast_bf16", "src", src, _F32)
    if dst is None:
        dst = torch.empty(src.shape, dtype=torch.bfloat16, device=src.device)
    call("b200_cast_f32_to_bf16", src.data_ptr(), dst.data_ptr(), src.numel(), _stream())
    return dst


def fill_f32(dst: Tensor, value: float) -> Tensor:
    _check("fill_f32", "dst", dst, _F32)
    call("b200_fill_f32", dst.data_ptr(), float(value), dst.numel(), _stream())
    return dst


def embedding_fwd(ids: Tensor, weight: Tensor) -> Tuple[Tensor, Tensor]:
    """(out fp32 [*ids.shape, D] = weight[ids], bad int32 [1]: non-zero if an id was outside [0, V)).  ids: contiguous int64;
    weight: contiguous fp32 [V, D]."""
    _check("embedding_fwd", "ids", ids, torch.int64)
    _check("embedding_fwd", "weight", weight, _F32, (None, None))
    V, D = weight.shape
    out = torch.empty(ids.shape + (D,), dtype=torch.float32, device=weight.device)
    bad = torch.zeros(1, dtype=torch.int32, device=weight.device)
    call("b200_embedding_fwd", ids.data_ptr(), weight.data_ptr(), out.data_ptr(), ids.numel(), D, V, bad.data_ptr(), _stream())
    return out, bad


def embedding_bwd(ids: Tensor, dnet: Tensor, V: int, D: int, padding_idx: int) -> Tensor:
    """dweight fp32 [V, D]: the rows of dnet (contiguous fp32, one row of D per id) summed into the rows their ids name, except
    ``padding_idx``'s."""
    _check("embedding_bwd", "ids", ids, torch.int64)
    _check("embedding_bwd", "dnet", dnet, _F32, numel=ids.numel() * D)
    dw = fill_f32(torch.empty((V, D), dtype=torch.float32, device=dnet.device), 0.0)
    call("b200_embedding_bwd", ids.data_ptr(), dnet.data_ptr(), dw.data_ptr(), ids.numel(), D, V, int(padding_idx), _stream())
    return dw


def argmax_gather_rows(net: Tensor, ids: Tensor) -> Tuple[Tensor, Tensor]:
    """(out fp32 [B, D] = net[b, pos[b]], pos int32 [B] = the first arg-max of ids[b]).  net: contiguous fp32 [B, T, D]; ids:
    contiguous int64 [B, T]."""
    _check("argmax_gather_rows", "net", net, _F32, (None, None, None))
    B, T, D = net.shape
    _check("argmax_gather_rows", "ids", ids, torch.int64, (B, T))
    out = torch.empty((B, D), dtype=torch.float32, device=net.device)
    pos = torch.empty(B, dtype=torch.int32, device=net.device)
    call("b200_argmax_gather_rows", ids.data_ptr(), net.data_ptr(), out.data_ptr(), pos.data_ptr(), B, T, D, _stream())
    return out, pos


def scatter_rows(dout: Tensor, pos: Tensor, T: int) -> Tensor:
    """The backward of ``argmax_gather_rows``: dx fp32 [B, T, D], zero but for dx[b, pos[b]] = dout[b].  dout: contiguous fp32
    [B, D]; pos: contiguous int32 [B]."""
    _check("scatter_rows", "dout", dout, _F32, (None, None))
    B, D = dout.shape
    _check("scatter_rows", "pos", pos, torch.int32, (B,))
    dx = fill_f32(torch.empty((B, T, D), dtype=torch.float32, device=dout.device), 0.0)
    call("b200_scatter_rows", dout.data_ptr(), pos.data_ptr(), dx.data_ptr(), B, T, D, _stream())
    return dx


# ----------------------------------------------------------------------------------------------------------------
# optimizer, fused FCNN
# ----------------------------------------------------------------------------------------------------------------
def adam_step(params: Tensor, grads: Tensor, exp_avg: Tensor, exp_avg_sq: Tensor, *, hyper: Sequence[float] = (), step: int = 0,
              hyper_dev: Optional[Tensor] = None, step_dev: Optional[Tensor] = None, increment: bool = True,
              decoupled: bool = False) -> None:
    """One Adam update (torch.optim.Adam without amsgrad) of contiguous fp32 tensors of equal numel, in place.  Either with host
    ``hyper`` = (lr, beta1, beta2, eps, weight_decay) at step count ``step`` >= 1, or with every hyper-parameter on the device:
    ``hyper_dev`` fp32 [6] = (lr, beta1, beta2, eps, weight_decay, grad_scale) and the step counter ``step_dev`` int32 [1],
    incremented first when ``increment`` (so the update can be replayed from a CUDA graph).  ``decoupled``: AdamW
    (torch.optim.AdamW's order, p (1 - lr weight_decay) first, then the update with no L2 term)."""
    what = "adamw_step" if decoupled else "adam_step"
    _check(what, "params", params, _F32)
    n = params.numel()
    for name, t in (("grads", grads), ("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
        _check(what, name, t, _F32, numel=n)
    if hyper_dev is None:
        call("b200_adamw_step" if decoupled else "b200_adam_step", params.data_ptr(), grads.data_ptr(), exp_avg.data_ptr(),
             exp_avg_sq.data_ptr(), n, *hyper, step, None, _stream())
        return
    _check(what, "hyper_dev", hyper_dev, _F32, (6,))
    _check(what, "step_dev", step_dev, torch.int32, (1,))
    call("b200_adamw_step_dev" if decoupled else "b200_adam_step_dev", params.data_ptr(), grads.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(), n, hyper_dev.data_ptr(),
         step_dev.data_ptr(), int(increment), _stream())


def fcnn_step(x: Tensor, params: Tensor, dims: Sequence[int], w_offsets: Sequence[int], b_offsets: Sequence[int], *,
              y: Optional[Tensor] = None, dpred: Optional[Tensor] = None, grads: Optional[Tensor] = None,
              loss_weights: Tuple[float, float] = (1.0, 1.0)) -> Tuple[Tensor, Optional[Tensor]]:
    """The fused ReLU MLP dims[0] -> ... -> dims[-1] (csrc/mlp.cu) on x fp32 [M, dims[0]], its weights and biases in the flat fp32
    arena ``params`` at ``w_offsets`` / ``b_offsets`` (-1: no bias).  Returns (pred fp32 [M, dims[-1]], loss).  With ``grads`` (an
    arena like ``params``) it also writes the parameter gradients of either the multi_task[mae, mse] loss against ``y``
    (weighted ``loss_weights``; ``loss`` is its fp32 scalar) or of ``dpred`` = d(pred), with ``loss`` None."""
    what = "fcnn_step"
    _check(what, "x", x, _F32, (None, dims[0]))
    _check(what, "params", params, _F32, (None,))
    M, P = x.shape[0], params.numel()
    _check(what, "y", y, _F32, (M, dims[-1]), optional=True)
    _check(what, "dpred", dpred, _F32, (M, dims[-1]), optional=True)
    _check(what, "grads", grads, _F32, (P,), optional=True)
    pred = torch.empty((M, dims[-1]), dtype=torch.float32, device=x.device)
    part = WORKSPACE.get(x.device, ((M + 127) // 128) * (P + 1), "fcnn") if grads is not None else None
    nblk = ctypes.c_int(0)
    host_arrays = ((ctypes.c_int * len(v))(*v) for v in (dims, w_offsets, b_offsets))
    call("b200_fcnn_step", x.data_ptr(), _ptr(y), _ptr(dpred), params.data_ptr(), pred.data_ptr(), _ptr(part), M, len(dims) - 1,
         *host_arrays, P, int(y is not None), float(loss_weights[0]), float(loss_weights[1]), ctypes.byref(nblk), _stream())
    loss = None
    if grads is not None:
        _colsum_finish(part, P + 1, nblk.value, 0, P, grads)
        if y is not None:  # column P of the partials: the loss
            loss = torch.empty((), dtype=torch.float32, device=x.device)
            _colsum_finish(part, P + 1, nblk.value, P, 1, loss)
    return pred, loss


# ----------------------------------------------------------------------------------------------------------------
# GroupNorm(32) + SiLU on channels-last activations (SD-v1.5 UNet, SURVEY.md 8f N3)
# ----------------------------------------------------------------------------------------------------------------
def groupnorm_silu_fwd(x: Tensor, gamma: Tensor, beta: Tensor, eps: float, *, silu: bool = True) -> Tuple[Tensor, Tensor, Tensor]:
    """x: bf16 [B, HW, C] (channels last).  Returns (y bf16 [B, HW, C], mean f32 [B, 32], rstd f32 [B, 32])."""
    _check("groupnorm_silu_fwd", "x", x, _BF16, (None, None, None))
    B, HW, C = x.shape
    _check("groupnorm_silu_fwd", "gamma", gamma, _F32, (C,))
    _check("groupnorm_silu_fwd", "beta", beta, _F32, (C,))
    y = torch.empty_like(x)
    mean = torch.empty((B, 32), dtype=torch.float32, device=x.device)
    rstd = torch.empty((B, 32), dtype=torch.float32, device=x.device)
    ws = WORKSPACE.get(x.device, int(_cabi.lib().b200_groupnorm_workspace_floats(B, HW, C)), "groupnorm")
    call("b200_groupnorm_silu_fwd", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
         ws.data_ptr(), B, HW, C, float(eps), int(silu), _stream())
    return y, mean, rstd


def groupnorm_silu_bwd(x: Tensor, dy: Tensor, gamma: Tensor, beta: Tensor, mean: Tensor, rstd: Tensor, *, silu: bool = True,
                       dgamma: Optional[Tensor] = None, dbeta: Optional[Tensor] = None, accumulate: bool = False) -> Tuple[Tensor, Tensor, Tensor]:
    what = "groupnorm_silu_bwd"
    _check(what, "x", x, _BF16, (None, None, None))
    B, HW, C = x.shape
    _check(what, "dy", dy, _BF16, (B, HW, C))
    _check(what, "mean", mean, _F32, (B, 32))
    _check(what, "rstd", rstd, _F32, (B, 32))
    dx = torch.empty_like(x)
    if dgamma is None:
        dgamma = torch.empty(C, dtype=torch.float32, device=x.device)
        dbeta = torch.empty(C, dtype=torch.float32, device=x.device)
        accumulate = False
    for t, name in ((gamma, "gamma"), (beta, "beta"), (dgamma, "dgamma"), (dbeta, "dbeta")):
        _check(what, name, t, _F32, (C,))
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
    _check("conv3x3_wgrad", "x", x, _BF16, (None, None, None, None))
    B, H, W, Cin = x.shape
    _check("conv3x3_wgrad", "dy", dy, _BF16, (B, H, W, None))
    Cout = dy.shape[3]
    _check("conv3x3_wgrad", "out", out, None, contiguous=False, optional=True)  # any CUDA tensor, as before
    if out is None:
        out = torch.empty((Cout, 9 * Cin), dtype=torch.float32, device=x.device)
        accumulate = False
    n = Cout * 9 * Cin
    splits = pick_splits(Cout, 9 * Cin, B * H * W)
    part = WORKSPACE.get(x.device, splits * n, "splitk")[: splits * n]
    call("b200_conv3x3_wgrad_nhwc_bf16", dy.data_ptr(), Cout, x.data_ptr(), part.data_ptr(), B, H, W, Cin, Cout, splits, _stream())
    call("b200_splitk_reduce", part.data_ptr(), splits, n, out.data_ptr(), int(round_bf16), int(accumulate), _stream())
    return out


def conv3x3_weight_view(w_packed: Tensor, cin: int) -> Tensor:
    """[Cout, 9 * Cin] (tap-major) -> a [Cout, Cin, 3, 3] view of it in the reference's Conv2d.weight index order."""
    co = w_packed.shape[0]
    return w_packed.view(co, 3, 3, cin).permute(0, 3, 1, 2)


def unpack_conv3x3_weight(w_packed: Tensor, cin: int) -> Tensor:
    """[Cout, 9 * Cin] (tap-major) -> [Cout, Cin, 3, 3], the reference's Conv2d.weight layout."""
    return conv3x3_weight_view(w_packed, cin).contiguous()


def conv3x3(x: Tensor, w_packed: Tensor, bias: Optional[Tensor] = None, *, epilogue: int = EPI_BIAS_BF16, aux: Optional[Tensor] = None) -> Tensor:
    """x: bf16 [B, H, W, Cin] channels-last; w_packed: bf16 [Cout, 9 * Cin] -> bf16 (or fp32 with the residual epilogue) [B, H, W, Cout].
    ``EPI_BIAS_ADD_PER_IMAGE_BF16``: aux = contiguous bf16 [B, Cout], added to every pixel of its image;
    ``EPI_BIAS_RESID_CLAMP_BF16``: aux = contiguous bf16 [B, H, W, Cout] (or [B * H * W, Cout]), the sum clamped to bf16's finite range."""
    _check("conv3x3", "x", x, _BF16, (None, None, None, None))
    B, H, W, Cin = x.shape
    _check("conv3x3", "w_packed", w_packed, _BF16, (None, 9 * Cin))
    Cout = w_packed.shape[0]
    if Cout % 8 != 0:
        raise B200Error(f"conv3x3: need Cout % 8 == 0, got {Cout}")
    _check("conv3x3", "bias", bias, None, contiguous=False, optional=True)
    dtype, aux_kind, _ = EPILOGUES.get(epilogue, (_BF16, None, None))  # the C side refuses the others
    if aux_kind:
        _check("conv3x3", "aux", aux, dtype, rows=B if aux_kind == "image" else B * H * W, width=Cout)
    else:
        _check("conv3x3", "aux", aux, None, contiguous=False, optional=True)
    out = torch.empty((B, H, W, Cout), dtype=dtype, device=x.device)
    call("b200_conv3x3_nhwc_bf16", x.data_ptr(), w_packed.data_ptr(), _ptr(bias), out.data_ptr(), _ptr(aux), Cout, B, H, W, Cin, Cout, epilogue, _stream())
    return out


# ----------------------------------------------------------------------------------------------------------------
# resampling convolutions of the SD-v1.5 UNet (include/b200_cflearn_ext.h)
# ----------------------------------------------------------------------------------------------------------------
def _conv_resample(entry: str, what: str, x: Tensor, w_packed: Tensor, bias: Optional[Tensor], epilogue: int, aux: Optional[Tensor],
                   Ho: int, Wo: int) -> Tensor:
    B, H, W, Cin = x.shape
    _check(what, "w_packed", w_packed, _BF16, (None, 9 * Cin))
    Cout = w_packed.shape[0]
    _check(what, "bias", bias, None, contiguous=False, optional=True)
    dtype, aux_kind, _ = EPILOGUES.get(epilogue, (_BF16, None, None))  # the C side refuses the others
    if aux_kind:
        _check(what, "aux", aux, dtype, rows=B if aux_kind == "image" else B * Ho * Wo, width=Cout)
    else:
        _check(what, "aux", aux, None, contiguous=False, optional=True)
    out = torch.empty((B, Ho, Wo, Cout), dtype=dtype, device=x.device)
    call(entry, x.data_ptr(), w_packed.data_ptr(), _ptr(bias), out.data_ptr(), _ptr(aux), Cout, B, H, W, Cin, Cout, epilogue, _stream())
    return out


def conv3x3_s2(x: Tensor, w_packed: Tensor, bias: Optional[Tensor] = None, *, epilogue: int = EPI_BIAS_BF16,
               aux: Optional[Tensor] = None) -> Tensor:
    """3x3 convolution with stride 2 and zero padding 1: x bf16 [B, H, W, Cin] channels-last, w_packed bf16 [Cout, 9 * Cin] ->
    [B, H/2, W/2, Cout].  ``epilogue`` / ``aux`` as ``conv3x3`` (aux rows: the output's pixels)."""
    _check("conv3x3_s2", "x", x, _BF16, (None, None, None, None))
    return _conv_resample("b200_conv3x3_s2_nhwc_bf16", "conv3x3_s2", x, w_packed, bias, epilogue, aux, x.shape[1] // 2, x.shape[2] // 2)


def conv3x3_up2(x: Tensor, w_packed: Tensor, bias: Optional[Tensor] = None, *, epilogue: int = EPI_BIAS_BF16,
                aux: Optional[Tensor] = None) -> Tensor:
    """Nearest 2x upsampling then a 3x3 / padding 1 convolution, in one implicit GEMM that never writes the upsampled image:
    x bf16 [B, H, W, Cin] channels-last, w_packed bf16 [Cout, 9 * Cin] -> [B, 2H, 2W, Cout].  ``epilogue`` / ``aux`` as
    ``conv3x3`` (aux rows: the output's pixels)."""
    _check("conv3x3_up2", "x", x, _BF16, (None, None, None, None))
    return _conv_resample("b200_conv3x3_up2_nhwc_bf16", "conv3x3_up2", x, w_packed, bias, epilogue, aux, 2 * x.shape[1], 2 * x.shape[2])


# taps (ky, kx) of the input-gradient parity classes (py, px) of the stride-2 convolution, in b200_conv3x3_s2_dgrad_nhwc_bf16's order
_S2_DGRAD_TAPS = [(ky, kx) for py in (0, 1) for px in (0, 1) for ky in ((1,) if py == 0 else (0, 2)) for kx in ((1,) if px == 0 else (0, 2))]


def pack_conv3x3_weight_s2_dgrad(w: Tensor) -> Tensor:
    """[Cout, Cin, 3, 3] -> bf16 [Cin, 9 * Cout]: the weights of ``conv3x3_s2_dgrad``, class by class and tap by tap."""
    if tuple(w.shape[2:]) != (3, 3):
        raise B200Error("pack_conv3x3_weight_s2_dgrad: 3x3 kernels only")
    return torch.cat([w[:, :, ky, kx].t() for ky, kx in _S2_DGRAD_TAPS], dim=1).to(torch.bfloat16).contiguous()


def conv3x3_s2_dgrad(dy: Tensor, w_dgrad: Tensor) -> Tensor:
    """Input gradient of ``conv3x3_s2``: dy bf16 [B, H/2, W/2, Cout], w_dgrad = ``pack_conv3x3_weight_s2_dgrad(w)`` -> bf16
    [B, H, W, Cin]."""
    what = "conv3x3_s2_dgrad"
    _check(what, "dy", dy, _BF16, (None, None, None, None))
    B, h, w, Cout = dy.shape
    _check(what, "w_dgrad", w_dgrad, _BF16, (None, 9 * Cout))
    Cin = w_dgrad.shape[0]
    dx = torch.empty((B, 2 * h, 2 * w, Cin), dtype=torch.bfloat16, device=dy.device)
    call("b200_conv3x3_s2_dgrad_nhwc_bf16", dy.data_ptr(), w_dgrad.data_ptr(), dx.data_ptr(), B, 2 * h, 2 * w, Cin, Cout, _stream())
    return dx


def conv3x3_s2_wgrad(dy: Tensor, x: Tensor, out: Optional[Tensor] = None, *, round_bf16: bool = True, accumulate: bool = False) -> Tensor:
    """Weight gradient of ``conv3x3_s2``: dy bf16 [B, H/2, W/2, Cout], x bf16 [B, H, W, Cin] -> fp32 [Cout, 9 * Cin], packed as
    ``conv3x3_wgrad``'s."""
    what = "conv3x3_s2_wgrad"
    _check(what, "x", x, _BF16, (None, None, None, None))
    B, H, W, Cin = x.shape
    _check(what, "dy", dy, _BF16, (B, H // 2, W // 2, None))
    Cout = dy.shape[3]
    if out is None:
        out = torch.empty((Cout, 9 * Cin), dtype=torch.float32, device=x.device)
        accumulate = False
    _check(what, "out", out, _F32, (Cout, 9 * Cin))
    n = Cout * 9 * Cin
    splits = pick_splits(Cout, 9 * Cin, B * (H // 2) * (W // 2))
    part = WORKSPACE.get(x.device, splits * n, "splitk")[: splits * n]
    call("b200_conv3x3_s2_wgrad_nhwc_bf16", dy.data_ptr(), Cout, x.data_ptr(), part.data_ptr(), B, H, W, Cin, Cout, splits, _stream())
    call("b200_splitk_reduce", part.data_ptr(), splits, n, out.data_ptr(), int(round_bf16), int(accumulate), _stream())
    return out


def upsample_nearest2x(x: Tensor) -> Tensor:
    """Nearest 2x upsampling of bf16 [B, H, W, C] (channels-last): [B, 2H, 2W, C], an exact copy."""
    _check("upsample_nearest2x", "x", x, _BF16, (None, None, None, None))
    B, H, W, C = x.shape
    out = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.bfloat16, device=x.device)
    call("b200_upsample_nearest2x_bf16", x.data_ptr(), out.data_ptr(), B, H, W, C, _stream())
    return out


def sum2x2(x: Tensor) -> Tensor:
    """The backward of ``upsample_nearest2x``: bf16 [B, 2H, 2W, C] -> bf16 [B, H, W, C], each 2x2 block summed in fp32 and
    rounded once."""
    _check("sum2x2", "x", x, _BF16, (None, None, None, None))
    B, H2, W2, C = x.shape
    if H2 % 2 or W2 % 2:
        raise B200Error(f"sum2x2: x must have even height and width, got {list(x.shape)}")
    out = torch.empty((B, H2 // 2, W2 // 2, C), dtype=torch.bfloat16, device=x.device)
    call("b200_sum2x2_bf16", x.data_ptr(), out.data_ptr(), B, H2 // 2, W2 // 2, C, _stream())
    return out


# ----------------------------------------------------------------------------------------------------------------
# the two ends of the SD-v1.5 UNet's training step (include/b200_cflearn_ext.h)
# ----------------------------------------------------------------------------------------------------------------
def _layout(what: str, name: str, t: Tensor, dtypes: Tuple[torch.dtype, ...]) -> bool:
    """True for a dense channels-last [B, C, H, W] CUDA tensor, False for a contiguous NCHW one; anything else is refused."""
    ok = t is not None and t.is_cuda and t.dtype in dtypes and t.dim() == 4
    cl = ok and t.is_contiguous(memory_format=torch.channels_last)
    if not ok or not (cl or t.is_contiguous()):
        got = "None" if t is None else f"{t.dtype} {list(t.shape)} with strides {list(t.stride())} on {t.device}"
        raise B200Error(f"{what}: {name} must be a CUDA {' or '.join(str(d) for d in dtypes)} tensor [B, C, H, W], contiguous NCHW or "
                        f"channels-last (got {got})")
    return cl and not t.is_contiguous()


def pad_channels(x: Tensor, cp: int, *, out: Optional[Tensor] = None) -> Tensor:
    """x fp32 or bf16 [B, C, H, W] (contiguous NCHW or channels-last) -> bf16 [B, H, W, cp] with channels >= C zero: the
    round-to-nearest-even cast autocast applies, then zero padding to a width the convolutions take.  ``out``: write there
    (contiguous bf16 [B, H, W, cp]) instead of a new tensor."""
    cl = _layout("pad_channels", "x", x, (_F32, _BF16))
    B, C, H, W = x.shape
    if out is None:
        out = torch.empty((B, H, W, cp), dtype=torch.bfloat16, device=x.device)
    _check("pad_channels", "out", out, _BF16, (B, H, W, cp))
    call("b200_pad_channels_bf16", x.data_ptr(), int(x.dtype == _F32), int(cl), out.data_ptr(), B, C, H, W, cp, _stream())
    return out


def q_sample_pad(x0: Tensor, noise: Tensor, timesteps: Tensor, sqrt_alphas_cumprod: Tensor, sqrt_one_minus_alphas_cumprod: Tensor,
                 cp: int) -> Tuple[Tensor, Tensor]:
    """DDPM noising into the stem's input: x0 and noise fp32 [B, C, H, W] (both contiguous NCHW or both channels-last),
    timesteps int64 [B], the two fp32 [T] tables -> (bf16 [B, H, W, cp] = bf16(a[t] x0 + s[t] noise) in fp32 with no contraction,
    channels >= C zero; int32 [1] flag, non-zero if a timestep was outside [0, T), whose image is then NaN)."""
    what = "q_sample_pad"
    cl = _layout(what, "x0", x0, (_F32,))
    if _layout(what, "noise", noise, (_F32,)) != cl or noise.shape != x0.shape:
        raise B200Error(f"{what}: noise must have x0's shape {list(x0.shape)} and memory format")
    B, C, H, W = x0.shape
    _check(what, "timesteps", timesteps, torch.int64, (B,))
    _check(what, "sqrt_alphas_cumprod", sqrt_alphas_cumprod, _F32, (None,))
    T = sqrt_alphas_cumprod.shape[0]
    _check(what, "sqrt_one_minus_alphas_cumprod", sqrt_one_minus_alphas_cumprod, _F32, (T,))
    out = torch.empty((B, H, W, cp), dtype=torch.bfloat16, device=x0.device)
    bad = torch.zeros(1, dtype=torch.int32, device=x0.device)
    call("b200_q_sample_pad_bf16", x0.data_ptr(), noise.data_ptr(), int(cl), timesteps.data_ptr(), sqrt_alphas_cumprod.data_ptr(),
         sqrt_one_minus_alphas_cumprod.data_ptr(), T, bad.data_ptr(), out.data_ptr(), B, C, H, W, cp, _stream())
    return out, bad


def noise_prediction_loss(pred: Tensor, noise: Tensor, *, grad_out: Optional[Tensor] = None) -> Tensor:
    """The DDPM noise-prediction loss mean_b(mean_chw((pred - noise)^2)) of pred bf16 [B, C, H, W] and noise (fp32 or bf16, the
    same shape and memory format; contiguous NCHW or channels-last).  Without ``grad_out``: the fp32 loss [1].  With it (fp32
    [1] on the device, the loss's upstream gradient): d loss / d pred, bf16 in pred's layout."""
    what = "noise_prediction_loss"
    cl = _layout(what, "pred", pred, (_BF16,))
    if _layout(what, "noise", noise, (_F32, _BF16)) != cl or noise.shape != pred.shape:
        raise B200Error(f"{what}: noise must have pred's shape {list(pred.shape)} and memory format")
    _check(what, "grad_out", grad_out, _F32, (1,), optional=True)
    B = pred.shape[0]
    N = pred.numel() // max(B, 1)
    loss = dpred = None
    if grad_out is None:
        loss = torch.empty(1, dtype=torch.float32, device=pred.device)
    else:
        dpred = torch.empty_like(pred)
    call("b200_noise_prediction_loss_bf16", pred.data_ptr(), noise.data_ptr(), int(noise.dtype == _F32), _ptr(loss), _ptr(dpred),
         _ptr(grad_out), B, N, _stream())
    return loss if grad_out is None else dpred


def ddim_step(eps: Tensor, eps_uncond: Optional[Tensor], guidance_scale: float, x: Tensor, noise: Tensor, coef: Tensor,
              ts_table: Tensor, temperature: float, step_dev: Tensor, bad_flag: Tensor, next_in: Tensor, next_ts: Tensor, *,
              increment: bool = True) -> None:
    """One DDIM step in place (include/b200_cflearn_ext.h, ``b200_ddim_step_bf16``): eps (and eps_uncond, or None) bf16
    [B, C, H, W] with dense channels-last strides (the UNet's output, or a batch half of it); x, noise fp32 contiguous NCHW
    [B, C, H, W]; coef fp32 [S, 5] and ts_table int64 [S] (``ddim.DDIMTables``); step_dev and bad_flag int32 [1]; next_in bf16
    [copies B, H, W, Cp] and next_ts int64 [copies B], copies 1 or 2.  ``increment``: advance step_dev after the step."""
    what = "ddim_step"
    _check(what, "x", x, _F32, (None, None, None, None))
    B, C, H, W = x.shape
    _check(what, "noise", noise, _F32, (B, C, H, W))
    for name, e in (("eps", eps), ("eps_uncond", eps_uncond)):
        if e is None and name == "eps_uncond":
            continue
        if not (e.is_cuda and e.dtype == _BF16 and e.shape == (B, C, H, W) and e.is_contiguous(memory_format=torch.channels_last)):
            got = f"{e.dtype} {list(e.shape)} with strides {list(e.stride())} on {e.device}"
            raise B200Error(f"{what}: {name} must be a CUDA bf16 tensor [{B}, {C}, {H}, {W}] with dense channels-last strides (got {got})")
    _check(what, "coef", coef, _F32, (None, 5))
    S = coef.shape[0]
    _check(what, "ts_table", ts_table, torch.int64, (S,))
    _check(what, "step_dev", step_dev, torch.int32, (1,))
    _check(what, "bad_flag", bad_flag, torch.int32, (1,))
    _check(what, "next_in", next_in, _BF16, (None, H, W, None))
    copies = next_in.shape[0] // B
    if copies not in (1, 2) or next_in.shape[0] != copies * B:
        raise B200Error(f"{what}: next_in must hold 1 or 2 copies of the batch ([B or 2B, H, W, Cp]), got {list(next_in.shape)}")
    _check(what, "next_ts", next_ts, torch.int64, (copies * B,))
    call("b200_ddim_step_bf16", eps.data_ptr(), _ptr(eps_uncond), float(guidance_scale), x.data_ptr(), noise.data_ptr(), coef.data_ptr(),
         ts_table.data_ptr(), S, float(temperature), step_dev.data_ptr(), int(increment), bad_flag.data_ptr(), next_in.data_ptr(),
         next_ts.data_ptr(), copies, B, C, H, W, next_in.shape[3], _stream())
