"""ctypes binding of ``libb200_cflearn.so`` (the C-ABI declared in ``include/b200_cflearn.h`` and ``include/b200_cflearn_ext.h``).

The library is the product: there is no CPU or PyTorch fallback.  Importing this module never raises (so the
CPU test-suite can inspect the symbol table), but every compute entry point raises ``B200Error`` loudly when the
shared object is missing or a call returns a negative status.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_longlong, c_void_p, POINTER
from typing import Any, Callable, Dict, List, Optional

LIB_NAME = "libb200_cflearn.so"
# B200_LIB_PATH: load another BUILD of the same library (A/B timing of two kernel versions on one box); never a fallback
LIB_PATH = os.environ.get("B200_LIB_PATH") or os.path.join(os.path.dirname(os.path.abspath(__file__)), LIB_NAME)


class B200Error(RuntimeError):
    """Raised when the native library is missing or a C-ABI call fails."""


# name -> (restype, argtypes).  Order and types mirror include/b200_cflearn.h exactly.
_P = c_void_p
_LL = c_longlong
SIGNATURES: Dict[str, Any] = {
    "b200_abi_version": (c_int, []),
    "b200_last_error": (c_char_p, []),
    "b200_launch_count": (_LL, []),
    "b200_gemm_bf16": (
        c_int,
        [_P, _LL, c_int, _P, _LL, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _LL, c_int, c_int, _P],
    ),
    "b200_gemm_pick_splits": (c_int, [c_int, c_int, c_int]),
    "b200_set_gemm_multicast": (c_int, [c_int]),
    "b200_splitk_reduce": (c_int, [_P, c_int, _LL, _P, c_int, c_int, _P]),
    "b200_layernorm_fwd": (c_int, [_P, _LL, _P, _P, _P, _P, _P, _P, c_int, c_int, c_float, _P]),
    "b200_layernorm_bwd": (
        c_int,
        [_P, c_int, _P, _LL, _P, _P, _P, _P, _P, _LL, _P, _P, c_int, POINTER(c_int), c_int, c_int, c_int, _P],
    ),
    "b200_layernorm_bf16_fwd": (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, c_float, _P]),
    "b200_layernorm_bf16_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, c_int, POINTER(c_int), c_int, c_int, _P]),
    "b200_colsum_bf16": (c_int, [_P, _LL, c_int, c_int, _P, c_int, POINTER(c_int), _P]),
    "b200_colsum_finish": (c_int, [_P, _LL, c_int, c_int, _P, c_int, c_int, _P]),
    "b200_colsum_finish2": (c_int, [_P, _LL, c_int, c_int, _P, c_int, c_int, _P, c_int, c_int, _P]),
    "b200_colsum_per_image_workspace_floats": (_LL, [c_int, c_int, c_int]),
    "b200_colsum_per_image_bf16": (c_int, [_P, c_int, c_int, c_int, _P, _P, _P, _P]),
    "b200_attention_fwd": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_float, c_int, _P]),
    "b200_set_attention_fwd_version": (c_int, [c_int]),
    "b200_set_attention_bwd_version": (c_int, [c_int]),
    "b200_set_attention_prefetch": (c_int, [c_int]),
    "b200_attention_bwd": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_float, c_int, _P, _P]),
    "b200_attention_long_fwd": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_float, c_int, _P]),
    "b200_attention_long_bwd_workspace_floats": (_LL, [c_int, c_int, c_int]),
    "b200_attention_long_bwd": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_float, c_int, _P, _P, _P]),
    "b200_cross_attention_fwd": (c_int, [_P, _LL, _P, _P, _LL, _P, _LL, _P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, _P]),
    "b200_cross_attention_bwd_workspace_floats": (_LL, [c_int, c_int, c_int, c_int, c_int]),
    "b200_cross_attention_bwd": (
        c_int,
        [_P, _LL, _P, _P, _LL, _P, _LL, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, _P, _P],
    ),
    "b200_fcnn_step": (
        c_int,
        [_P, _P, _P, _P, _P, _P, c_int, c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int), c_int, c_int, c_float, c_float,
         POINTER(c_int), _P],
    ),
    "b200_patch_im2col": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "b200_patch_im2col_u8": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_double, POINTER(c_double), POINTER(c_double), _P]),
    "b200_assemble_tokens": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P]),
    "b200_assemble_tokens_bwd": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "b200_embedding_fwd": (c_int, [_P, _P, _P, _LL, c_int, c_int, _P, _P]),
    "b200_embedding_bwd": (c_int, [_P, _P, _P, _LL, c_int, c_int, c_int, _P]),
    "b200_argmax_gather_rows": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P]),
    "b200_scatter_rows": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "b200_add_pos": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "b200_add_pos_bwd": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "b200_softmax_xent_fwd_bwd": (c_int, [_P, _LL, _P, _P, _P, _P, _P, c_int, c_int, c_float, _P, _P]),
    "b200_symmetric_xent_fwd_bwd": (c_int, [_P, _LL, _P, _P, _P, c_int, c_float, _P, _P]),
    "b200_adam_step": (c_int, [_P, _P, _P, _P, _LL, c_float, c_float, c_float, c_float, c_float, c_int, _P, _P]),
    "b200_adam_step_dev": (c_int, [_P, _P, _P, _P, _LL, _P, _P, c_int, _P]),
    "b200_cast_f32_to_bf16": (c_int, [_P, _P, _LL, _P]),
    "b200_fill_f32": (c_int, [_P, c_float, _LL, _P]),
    "b200_conv3x3_nhwc_bf16": (c_int, [_P, _P, _P, _P, _P, _LL, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200_conv3x3_wgrad_nhwc_bf16": (c_int, [_P, _LL, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200_set_persistent_ctas": (c_int, [c_int, c_int]),
    "b200_groupnorm_workspace_floats": (_LL, [c_int, c_int, c_int]),
    "b200_groupnorm_silu_fwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_float, c_int, _P]),
    "b200_groupnorm_silu_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200_comm_unique_id": (c_int, [_P]),
    "b200_comm_init": (c_int, [_P, c_int, c_int, c_int, POINTER(c_void_p)]),
    "b200_comm_allreduce_bucket": (c_int, [_P, _P, _LL, c_int, _P]),
    "b200_comm_async_error": (c_int, [_P]),
    "b200_comm_finalize": (c_int, [_P, c_int]),
    "b200_comm_nccl_version": (c_int, []),
}

# The entry points declared in include/b200_cflearn_ext.h (after version 4 of the main header), exported by the same library.
EXT_SIGNATURES: Dict[str, Any] = {
    "b200_conv3x3_s2_nhwc_bf16": (c_int, [_P, _P, _P, _P, _P, _LL, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200_conv3x3_s2_dgrad_nhwc_bf16": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200_conv3x3_s2_wgrad_nhwc_bf16": (c_int, [_P, _LL, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200_conv3x3_up2_nhwc_bf16": (c_int, [_P, _P, _P, _P, _P, _LL, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200_upsample_nearest2x_bf16": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "b200_sum2x2_bf16": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "b200_pad_channels_bf16": (c_int, [_P, c_int, c_int, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200_noise_prediction_loss_bf16": (c_int, [_P, _P, c_int, _P, _P, _P, c_int, _LL, _P]),
    "b200_q_sample_pad_bf16": (c_int, [_P, _P, c_int, _P, _P, _P, _LL, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200_ddim_step_bf16": (c_int, [_P, _P, c_float, _P, _P, _P, _P, c_int, c_float, _P, c_int, _P, _P, _P, c_int, c_int, c_int, c_int,
                                    c_int, c_int, _P]),
    "b200_adamw_step": (c_int, [_P, _P, _P, _P, _LL, c_float, c_float, c_float, c_float, c_float, c_int, _P, _P]),
    "b200_adamw_step_dev": (c_int, [_P, _P, _P, _P, _LL, _P, _P, c_int, _P]),
}

_lib: Optional[ctypes.CDLL] = None
_load_error: Optional[str] = None


def _load() -> None:
    global _lib, _load_error
    if _lib is not None or _load_error is not None:
        return
    if not os.path.isfile(LIB_PATH):
        _load_error = (
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            f"(or `make -C carefree-learn_b200/csrc`). There is no CPU fallback."
        )
        return
    try:
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in {**SIGNATURES, **EXT_SIGNATURES}.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        if os.environ.get("B200_ATTN_FWD", "") in ("1", "2"):  # A/B switch for profiling
            lib.b200_set_attention_fwd_version(int(os.environ["B200_ATTN_FWD"]))
        if os.environ.get("B200_ATTN_PREFETCH", "") in ("0", "1"):
            lib.b200_set_attention_prefetch(int(os.environ["B200_ATTN_PREFETCH"]))
        if os.environ.get("B200_ATTN_BWD", "") in ("1", "2", "3"):
            lib.b200_set_attention_bwd_version(int(os.environ["B200_ATTN_BWD"]))
        if os.environ.get("B200_GEMM_MULTICAST", "") in ("0", "1", "2"):  # A/B/C switch for profiling; results are identical
            lib.b200_set_gemm_multicast(int(os.environ["B200_GEMM_MULTICAST"]))
        _lib = lib
    except (OSError, AttributeError) as err:  # pragma: no cover - depends on the build
        _load_error = f"failed to load {LIB_PATH}: {err}"


def available() -> bool:
    _load()
    return _lib is not None


def load_error() -> Optional[str]:
    _load()
    return _load_error


def lib() -> ctypes.CDLL:
    _load()
    if _lib is None:
        raise B200Error(_load_error or "libb200_cflearn.so unavailable")
    return _lib


def exported_symbols() -> List[str]:
    return [name for name in SIGNATURES if hasattr(lib(), name)]


def exported_ext_symbols() -> List[str]:
    return [name for name in EXT_SIGNATURES if hasattr(lib(), name)]


def last_error() -> str:
    msg = lib().b200_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(status: int, what: str) -> None:
    if status != 0:
        raise B200Error(f"{what} failed with status {status}: {last_error()}")


def call(name: str, *args: Any) -> None:
    """Invoke a status-returning entry point and raise on failure."""
    fn: Callable[..., int] = getattr(lib(), name)
    check(fn(*args), name)


def launch_count() -> int:
    return int(lib().b200_launch_count())
