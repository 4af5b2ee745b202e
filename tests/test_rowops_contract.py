"""The argument contract of the row, loss, optimizer and glue entry points (include/b200_cflearn.h), checked without a GPU, and
the tensor checks of the ops wrappers over them on one.

Every refusal of the C-ABI happens before anything is launched, so it is the same with or without a device.  The device pointers
are fake and never dereferenced: refused calls stop at the argument checks.  A call that passes them fails its first launch with
B200_ERR_LAUNCH on a machine without a GPU; the matrices that make such calls run only there, so no kernel ever sees a fake
pointer.  Host arrays (nparts_out, fcnn_step's dims and offsets) are real."""
import ast
import ctypes
import itertools
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import B200Error, _cabi, ops  # noqa: E402

ARG, ALIGN, LAUNCH = -1, -2, -4
FAKE = 1 << 20
POINTERS = (FAKE, None, FAKE + 8, FAKE + 4, FAKE + 2)  # valid, NULL, misaligned for 16, for 8, for 4
INT_MAX = 2 ** 31 - 1
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="accepted calls would launch kernels on fake pointers")

_NPARTS = ctypes.c_int(0)
HOST_INT = ctypes.byref(_NPARTS)  # nparts_out / nblocks_out: a host int the library writes
# fcnn_step: 10 -> 32 -> 1, W0 [32, 10] at 0, b0 at 320, W1 [1, 32] at 352, b1 at 384 in an arena of 388 floats
DIMS, WOFF, BOFF = (ctypes.c_int * 3)(10, 32, 1), (ctypes.c_int * 2)(0, 352), (ctypes.c_int * 2)(320, 384)
WIDE = (ctypes.c_int * 3)(10, 2000, 1)  # parameters + activations > 220 KB


def _ln_sizes(a, max_dim, vec):
    return [a["rows"] <= 0, a["dim"] <= 0, a["dim"] % vec != 0, a["dim"] > max_dim]


def _fcnn_rules(a):
    dims = a["dims"]
    arg = [a["M"] <= 0, not 1 <= a["n_layers"] <= 8, a["arena_len"] <= 0,
           a["part"] is not None and a["loss_mode"] == 0 and a["dpred"] is None,
           a["part"] is not None and a["loss_mode"] == 1 and a["y"] is None]
    if dims is not None and a["w_offsets"] is not None and a["b_offsets"] is not None and not any(arg[:2]):
        L = a["n_layers"]
        arg.append(dims is WIDE or any(a["w_offsets"][l] + dims[l] * dims[l + 1] > a["arena_len"] for l in range(min(L, 2))))
    return arg, []


# Per entry point, from the header: its parameters in signature order (stream excluded) with the value a valid call passes,
# each device pointer's (required, alignment), and its size / leading-dimension rules -> ([ARG rule broken], [ALIGN rule broken]).
R16, O16, R8, R4, O4, R2, O2 = (True, 16), (False, 16), (True, 8), (True, 4), (False, 4), (True, 2), (False, 2)
ENTRIES = {
    "b200_layernorm_fwd": (
        dict(x=R16, ld_x=768, gamma=R16, beta=R16, y_bf16=R16, y_f32=O16, mean=R4, rstd=R4, rows=64, dim=768, eps=1e-5),
        lambda a: (_ln_sizes(a, 1024, 4) + [a["ld_x"] < a["dim"]], [a["ld_x"] % 4 != 0])),
    "b200_layernorm_bwd": (
        dict(dy=R16, dy_is_f32=0, x=R16, ld_x=768, gamma=R16, mean=R4, rstd=R4, dres=O16, dx_out=R16, ld_dx=768, dx_bf16=O16,
             dgb_part=R4, max_parts=64, nparts_out=HOST_INT, rows=64, dim=768, dx_colsum=0),
        lambda a: (_ln_sizes(a, 1024, 4) + [a["max_parts"] < 1, a["dx_colsum"] and a["dy_is_f32"],
                                            a["dx_colsum"] and a["dx_bf16"] is None, a["ld_x"] < a["dim"], a["ld_dx"] < a["dim"]],
                   [a["ld_x"] % 4 != 0, a["ld_dx"] % 4 != 0])),
    "b200_layernorm_bf16_fwd": (
        dict(x=R16, gamma=R16, beta=R16, y=R16, mean=R4, rstd=R4, rows=64, dim=320, eps=1e-5),
        lambda a: (_ln_sizes(a, 2048, 8), [])),
    "b200_layernorm_bf16_bwd": (
        dict(dy=R16, x=R16, gamma=R16, mean=R4, rstd=R4, dres=O16, dx=R16, dgb_part=R4, max_parts=64, nparts_out=HOST_INT, rows=64,
             dim=320),
        lambda a: (_ln_sizes(a, 2048, 8) + [a["max_parts"] < 1], [])),
    "b200_colsum_bf16": (
        dict(x=R16, ld=1000, rows=64, cols=1000, part=R4, max_parts=64, nparts_out=HOST_INT),
        lambda a: ([a["rows"] <= 0, a["cols"] <= 0, a["max_parts"] < 1, a["ld"] < (a["cols"] + 7) // 8 * 8], [a["ld"] % 8 != 0])),
    "b200_colsum_finish": (
        dict(part=R4, part_ld=100, nparts=8, cols=100, out=R4, round_bf16=0, accumulate=0),
        lambda a: ([a["nparts"] <= 0, a["cols"] <= 0, a["part_ld"] < a["cols"]], [])),
    "b200_colsum_finish2": (
        dict(part=R4, part_ld=100, nparts=8, cols0=60, out0=R4, round0=0, cols1=40, out1=R4, round1=1, accumulate=0),
        lambda a: ([a["nparts"] <= 0, a["cols0"] <= 0, a["cols1"] <= 0, a["part_ld"] < a["cols0"] + a["cols1"]], [])),
    "b200_colsum_per_image_bf16": (
        dict(x=R16, B=2, HW=64, C=320, per_image=R4, total=R4, workspace=R4),
        lambda a: ([a["B"] <= 0, a["HW"] <= 0, a["C"] <= 0, a["C"] % 8 != 0, a["B"] * a["HW"] > INT_MAX], [])),
    "b200_splitk_reduce": (
        dict(partial=R16, splits=4, n=4096, out=R16, round_bf16=1, accumulate=0),
        lambda a: ([a["splits"] < 1, a["n"] <= 0, a["n"] % 4 != 0], [])),
    "b200_patch_im2col": (
        dict(x=R16, cols=R16, B=2, C=3, img=224, patch=16),
        lambda a: ([a["B"] <= 0, a["C"] <= 0, a["img"] <= 0, a["patch"] <= 0 or a["patch"] % 16 != 0 or a["img"] % a["patch"] != 0], [])),
    "b200_patch_im2col_u8": (
        dict(x=R16, cols=R16, B=2, C=3, img=224, patch=16, division=255.0, mean=None, std=None),
        lambda a: ([a["B"] <= 0, not 1 <= a["C"] <= 4, a["img"] <= 0, a["division"] == 0,
                    a["patch"] <= 0 or a["patch"] % 16 != 0 or a["img"] % a["patch"] != 0], [])),
    "b200_assemble_tokens": (
        dict(patch=R16, cls=R16, pos=R16, net=R16, B=2, np=196, D=768, conv_bias=O16),
        lambda a: ([a["B"] <= 0, a["np"] <= 0, a["D"] <= 0, a["D"] % 8 != 0], [])),
    "b200_assemble_tokens_bwd": (
        dict(dnet=R16, dpatch=R16, dpos=R16, dcls=R16, B=2, np=196, D=768, accumulate=0),
        lambda a: ([a["B"] <= 0, a["np"] <= 0, a["D"] <= 0, a["D"] % 4 != 0, (a["np"] + 1) * (a["D"] // 4) > INT_MAX], [])),
    "b200_embedding_fwd": (
        dict(ids=R8, weight=R16, out=R16, n=77, D=512, V=49408, flag=R4),
        lambda a: ([a["n"] <= 0, a["D"] <= 0, a["D"] % 4 != 0, a["V"] <= 0], [])),
    "b200_embedding_bwd": (
        dict(ids=R8, dnet=R4, dweight=R4, n=77, D=512, V=49408, padding_idx=0),
        lambda a: ([a["n"] <= 0, a["D"] <= 0, a["V"] <= 0], [])),
    "b200_argmax_gather_rows": (
        dict(ids=R8, x=R4, out=R4, pos=R4, B=2, T=77, D=512),
        lambda a: ([a["B"] <= 0, a["T"] <= 0, a["D"] <= 0], [])),
    "b200_scatter_rows": (
        dict(dout=R4, pos=R4, dx=R4, B=2, T=77, D=512),
        lambda a: ([a["B"] <= 0, a["T"] <= 0, a["D"] <= 0], [])),
    "b200_add_pos": (
        dict(x=R16, pos=R16, net=R16, B=2, T=77, D=512),
        lambda a: ([a["B"] <= 0, a["T"] <= 0, a["D"] <= 0, a["D"] % 4 != 0, a["T"] * (a["D"] // 4) > INT_MAX], [])),
    "b200_add_pos_bwd": (
        dict(dnet=R16, dpos=R16, B=2, T=77, D=512, accumulate=0),
        lambda a: ([a["B"] <= 0, a["T"] <= 0, a["D"] <= 0, a["D"] % 4 != 0, a["T"] * (a["D"] // 4) > INT_MAX], [])),
    "b200_softmax_xent_fwd_bwd": (
        dict(logits=R2, ldl=1000, labels=R8, loss_rows=R4, loss_mean=O4, dlogits=O2, flag=R4, B=64, C=1000, grad_scale=1.0,
             grad_scale_dev=O4),
        lambda a: ([a["B"] <= 0, a["C"] <= 0, a["ldl"] < a["C"]], [])),
    "b200_symmetric_xent_fwd_bwd": (
        dict(logits=R2, ldl=64, loss=R4, dlogits=O2, lse_ws=R4, B=64, grad_scale=1.0, grad_scale_dev=O4),
        lambda a: ([a["B"] <= 0, a["ldl"] < a["B"]], [])),
    "b200_adam_step": (
        dict(params=R16, grads=R16, exp_avg=R16, exp_avg_sq=R16, n=4096, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0,
             step=1, step_dev=O4),
        lambda a: ([a["n"] <= 0, a["n"] % 4 != 0, a["step_dev"] is None and a["step"] < 1], [])),
    "b200_adam_step_dev": (
        dict(params=R16, grads=R16, exp_avg=R16, exp_avg_sq=R16, n=4096, hyper_dev=R4, step_dev=R4, increment=1),
        lambda a: ([a["n"] <= 0, a["n"] % 4 != 0], [])),
    "b200_cast_f32_to_bf16": (dict(src=R16, dst=R16, n=1000), lambda a: ([a["n"] <= 0], [])),
    "b200_fill_f32": (dict(dst=R16, value=0.0, n=1000), lambda a: ([a["n"] <= 0], [])),
    "b200_groupnorm_silu_fwd": (
        dict(x=R16, gamma=R4, beta=R4, y=R16, mean=R4, rstd=R4, workspace=R4, B=2, HW=64, C=320, eps=1e-5, silu=1),
        lambda a: ([a["B"] <= 0, a["HW"] <= 0, a["C"] <= 0, a["C"] % 32 != 0, a["C"] > 2560], [])),
    "b200_groupnorm_silu_bwd": (
        dict(x=R16, dy=R16, gamma=R4, beta=R4, mean=R4, rstd=R4, dx=R16, dgamma=R4, dbeta=R4, workspace=R4, B=2, HW=64, C=320, silu=1,
             accumulate=0),
        lambda a: ([a["B"] <= 0, a["HW"] <= 0, a["C"] <= 0, a["C"] % 32 != 0, a["C"] > 2560], [])),
    "b200_fcnn_step": (
        dict(x=R4, y=O4, dpred=O4, params=R4, pred=O4, part=O4, M=128, n_layers=2, dims=DIMS, w_offsets=WOFF, b_offsets=BOFF,
             arena_len=388, loss_mode=1, w_mae=0.5, w_mse=0.5, nblocks_out=HOST_INT),
        _fcnn_rules),
}
HOST_ARRAYS = {"dims", "w_offsets", "b_offsets"}  # fcnn_step's required host pointers


def _pointers(entry):
    return {n: v for n, v in ENTRIES[entry][0].items() if isinstance(v, tuple)}


def call(entry, **kw):
    """Calls `entry` with the table's valid values, FAKE for every device pointer, and `kw` in place of them."""
    params = ENTRIES[entry][0]
    args = [kw[n] if n in kw else (FAKE if isinstance(v, tuple) else v) for n, v in params.items()]
    return getattr(_cabi.lib(), entry)(*args, None)


def expected(entry, **kw):
    """The statuses the contract allows for one call: the codes of every rule it breaks, or LAUNCH if it breaks none."""
    params, rules = ENTRIES[entry]
    a = {n: kw[n] if n in kw else (FAKE if isinstance(v, tuple) else v) for n, v in params.items()}
    arg, align = rules(a)
    for n, (required, al) in _pointers(entry).items():
        arg.append(required and a[n] is None)
        align.append(a[n] is not None and a[n] % al != 0)
    arg += [a[n] is None for n in HOST_ARRAYS & set(a)]
    return ({ARG} if any(arg) else set()) | ({ALIGN} if any(align) else set()) or {LAUNCH}


def check_all(entry, calls):
    bad = []
    for kw in calls:
        got = call(entry, **kw)
        if got not in expected(entry, **kw):
            bad.append((kw, got, _cabi.last_error()))
    assert not bad, f"{entry}: {len(bad)} of {len(calls)} calls disagree with the header, e.g. {bad[:3]}"


# Sizes on both sides of every rule (full product per entry).
SIZES = {
    "b200_layernorm_fwd": dict(rows=(0, 1, 64), dim=(0, 4, 6, 768, 1024, 1028), ld_x=(4, 768, 770, 1024, 1032)),
    "b200_layernorm_bwd": dict(dim=(0, 6, 768, 1028), ld_x=(768, 770, 1032), ld_dx=(4, 768, 1028), max_parts=(0, 1), dy_is_f32=(0, 1),
                               dx_colsum=(0, 1), rows=(0, 5)),
    "b200_layernorm_bf16_fwd": dict(rows=(0, 1, 7), dim=(0, 4, 8, 324, 2048, 2056)),
    "b200_layernorm_bf16_bwd": dict(rows=(0, 1, 7), dim=(0, 4, 8, 324, 2048, 2056), max_parts=(0, 1)),
    "b200_colsum_bf16": dict(rows=(0, 1), cols=(0, 1, 8, 1000, 1001), ld=(0, 8, 1000, 1004, 1008), max_parts=(0, 1)),
    "b200_colsum_finish": dict(nparts=(0, 1), cols=(0, 1, 100, 101), part_ld=(0, 100, 101)),
    "b200_colsum_finish2": dict(nparts=(0, 1), cols0=(0, 60), cols1=(0, 40, 41), part_ld=(60, 100, 101)),
    "b200_colsum_per_image_bf16": dict(B=(0, 1, 2, 65536), HW=(0, 64, 65536), C=(0, 4, 320, 324)),
    "b200_splitk_reduce": dict(splits=(0, 1, 4), n=(0, 2, 4, 4096, 4098)),
    "b200_patch_im2col": dict(B=(0, 2), C=(0, 3), img=(0, 8, 224, 232), patch=(0, 8, 16, 32)),
    "b200_patch_im2col_u8": dict(B=(0, 2), C=(0, 1, 4, 5), img=(0, 224, 232), patch=(0, 8, 16), division=(0.0, 255.0)),
    "b200_assemble_tokens": dict(B=(0, 2), np=(0, 1, 196), D=(0, 4, 8, 768)),
    "b200_assemble_tokens_bwd": dict(B=(0, 2), np=(0, 196, 2 ** 20, INT_MAX), D=(0, 2, 4, 768, 8192)),
    "b200_embedding_fwd": dict(n=(0, 1, 77), D=(0, 2, 4, 512), V=(0, 1)),
    "b200_embedding_bwd": dict(n=(0, 77), D=(0, 3), V=(0, 1)),
    "b200_argmax_gather_rows": dict(B=(0, 2), T=(0, 77), D=(0, 3)),
    "b200_scatter_rows": dict(B=(0, 2), T=(0, 77), D=(0, 3)),
    "b200_add_pos": dict(B=(0, 2), T=(0, 77, 2 ** 20, INT_MAX), D=(0, 2, 4, 512, 8192)),
    "b200_add_pos_bwd": dict(B=(0, 2), T=(0, 77, 2 ** 20, INT_MAX), D=(0, 2, 4, 512, 8192)),
    "b200_softmax_xent_fwd_bwd": dict(B=(0, 1), C=(0, 1, 1000, 1001), ldl=(0, 8, 1000, 1001, 1008)),
    "b200_symmetric_xent_fwd_bwd": dict(B=(0, 1, 64, 65), ldl=(0, 8, 64, 65, 72)),
    "b200_adam_step": dict(n=(0, 2, 4, 4096), step=(0, 1), step_dev=(None, FAKE)),
    "b200_adam_step_dev": dict(n=(0, 2, 4, 4096), increment=(0, 1)),
    "b200_cast_f32_to_bf16": dict(n=(-1, 0, 1, 1000)),
    "b200_fill_f32": dict(n=(-1, 0, 1, 1000)),
    "b200_groupnorm_silu_fwd": dict(B=(0, 2), HW=(0, 64), C=(0, 8, 32, 320, 2560, 2592)),
    "b200_groupnorm_silu_bwd": dict(B=(0, 2), HW=(0, 64), C=(0, 8, 32, 320, 2560, 2592)),
    "b200_fcnn_step": dict(M=(0, 1, 128), n_layers=(0, 2, 9), arena_len=(0, 300, 388), dims=(DIMS, WIDE), loss_mode=(0, 1),
                           part=(None, FAKE), dpred=(None, FAKE)),
}


@no_device
@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_sizes_follow_the_header(entry):
    names = list(SIZES[entry])
    check_all(entry, [dict(zip(names, vals)) for vals in itertools.product(*SIZES[entry].values())])


@no_device
@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_pointers_follow_the_header(entry):
    """Every pointer over FAKE / NULL / +8 / +4 / +2: all combinations where an entry has at most four, else one at a time."""
    names = list(_pointers(entry))
    if len(names) <= 4:
        calls = [dict(zip(names, ps)) for ps in itertools.product(POINTERS, repeat=len(names))]
    else:
        calls = [{n: p} for n in names for p in POINTERS]
    if entry == "b200_fcnn_step":
        calls += [{n: None} for n in sorted(HOST_ARRAYS)]
    check_all(entry, calls)


def test_refusals_name_the_rule():
    for entry in ENTRIES:
        required = [n for n, (req, _) in _pointers(entry).items() if req]
        assert call(entry, **{required[0]: None}) == ARG and "null" in _cabi.last_error(), entry
        aligned16 = [n for n, (_, al) in _pointers(entry).items() if al == 16]
        for n, (_, al) in _pointers(entry).items():
            bad = FAKE + (8 if al == 16 else al // 2)
            assert call(entry, **{n: bad}) == ALIGN and "aligned" in _cabi.last_error(), (entry, n)
        if aligned16:
            assert call(entry, **{aligned16[-1]: FAKE + 4}) == ALIGN, entry
    for entry in ("b200_layernorm_fwd", "b200_layernorm_bwd"):
        assert call(entry, ld_x=764) == ARG  # a row narrower than dim
    assert call("b200_colsum_bf16", ld=1004) == ALIGN
    assert call("b200_softmax_xent_fwd_bwd", ldl=8) == ARG and call("b200_symmetric_xent_fwd_bwd", ldl=8) == ARG
    assert call("b200_add_pos_bwd", T=2 ** 20, D=8192) == ARG and "overflow" in _cabi.last_error()
    assert call("b200_fcnn_step", dims=None) == ARG and "null" in _cabi.last_error()


NO_CONTRACT = {
    "b200_abi_version", "b200_last_error", "b200_launch_count", "b200_gemm_pick_splits", "b200_set_gemm_multicast",
    "b200_set_attention_fwd_version", "b200_set_attention_bwd_version", "b200_set_attention_prefetch", "b200_set_persistent_ctas",
    "b200_colsum_per_image_workspace_floats", "b200_attention_long_bwd_workspace_floats", "b200_cross_attention_bwd_workspace_floats",
    "b200_groupnorm_workspace_floats",
} | {n for n in _cabi.SIGNATURES if n.startswith("b200_comm_")}


def test_every_entry_point_has_a_contract():
    """Each name of the C-ABI is covered exactly once: by the GEMM contract (check_gemm_args), the attention contract, this
    file, or the list of entries that take no device pointers or talk to NCCL."""
    import test_attention_contract
    gemm = {"b200_gemm_bf16", "b200_conv3x3_nhwc_bf16", "b200_conv3x3_wgrad_nhwc_bf16"}
    attention = set(test_attention_contract.ENTRIES)
    groups = [gemm, attention, set(ENTRIES), NO_CONTRACT]
    for name in _cabi.SIGNATURES:
        assert sum(name in g for g in groups) == 1, name
    assert set().union(*groups) == set(_cabi.SIGNATURES)


def _names_in_code(path):
    """Identifiers, attribute names and whole string constants of a module: names in comments or docstrings do not count."""
    with open(path) as f:
        tree = ast.parse(f.read())
    return {n.id if isinstance(n, ast.Name) else n.attr if isinstance(n, ast.Attribute) else n.value for n in ast.walk(tree)
            if isinstance(n, (ast.Name, ast.Attribute)) or (isinstance(n, ast.Constant) and isinstance(n.value, str))}


def test_only_ops_calls_the_compute_entry_points():
    """ops.py is the one module that knows the compute entry points' arguments (and checks every tensor it hands them): each is
    named there and in no other module of the package but the ctypes binding."""
    compute = set(_cabi.SIGNATURES) - NO_CONTRACT
    pkg = os.path.join(ROOT, "carefree-learn_b200")
    assert not compute - _names_in_code(os.path.join(pkg, "ops.py"))
    for name in sorted(os.listdir(pkg)):
        if name.endswith(".py") and name not in ("ops.py", "_cabi.py"):
            assert not compute & _names_in_code(os.path.join(pkg, name)), name


# ---- moved unchanged from the ResBlock and SpatialTransformer test files ----------------------------------------------------
def test_colsum_per_image_rejects_bad_arguments():
    lib = _cabi.lib()
    null = ctypes.c_void_p(0)
    fake = ctypes.c_void_p(1 << 20)  # never dereferenced: every case fails its checks before any launch
    odd = ctypes.c_void_p((1 << 20) + 8)
    def cs(x=fake, B=2, HW=64, C=320, per=fake, tot=fake, ws=fake):
        return lib.b200_colsum_per_image_bf16(x, B, HW, C, per, tot, ws, null)

    assert cs(C=324) == -1 and cs(C=0) == -1 and cs(B=0) == -1 and cs(HW=0) == -1
    assert cs(x=null) == -1 and cs(per=null) == -1 and cs(tot=null) == -1 and cs(ws=null) == -1
    assert cs(x=odd) == -2
    assert lib.b200_colsum_per_image_workspace_floats(8, 4096, 320) >= 8 * 320
    assert lib.b200_colsum_per_image_workspace_floats(0, 64, 320) == 0


def test_layernorm_bf16_rejects_bad_arguments():
    lib = _cabi.lib()
    null = ctypes.c_void_p(0)
    fake = ctypes.c_void_p(1 << 20)  # never dereferenced: every case fails its checks before any launch
    odd = ctypes.c_void_p((1 << 20) + 8)

    def ln_fwd(x=fake, y=fake, gamma=fake, rows=16, dim=320):
        return lib.b200_layernorm_bf16_fwd(x, gamma, fake, y, fake, fake, rows, dim, 1e-5, null)

    def ln_bwd(dy=fake, dres=null, dx=fake, part=fake, rows=16, dim=320):
        n = ctypes.c_int(0)
        return lib.b200_layernorm_bf16_bwd(dy, fake, fake, fake, fake, dres, dx, part, 64, ctypes.byref(n), rows, dim, null)

    for dim in (0, 4, 324, 2056):
        assert ln_fwd(dim=dim) == -1 and ln_bwd(dim=dim) == -1, dim
    assert ln_fwd(rows=0) == -1 and ln_bwd(rows=0) == -1
    assert ln_fwd(x=null) == -1 and ln_bwd(dx=null) == -1 and ln_bwd(part=null) == -1
    assert "null" in _cabi.last_error()
    assert ln_fwd(x=odd) == -2 and ln_fwd(gamma=odd) == -2 and ln_bwd(dres=odd) == -2 and ln_bwd(dy=odd) == -2


# ---- ops: every tensor handed to the library is checked against the header's layout ------------------------------------------
def _f32(*shape):
    return torch.randn(*shape, device="cuda")


def _bf16(*shape):
    return _f32(*shape).to(torch.bfloat16)


def _refused(fn, *args, **kw):
    with pytest.raises(B200Error):
        fn(*args, **kw)


@pytest.mark.gpu
def test_ops_layernorm_refuses_bad_tensors():
    rows, dim = 64, 256
    x, g, b = _f32(rows, dim), _f32(dim), _f32(dim)
    fwd = lambda x=x, g=g, b=b, ld=dim, **kw: ops.layernorm_fwd(x, g, b, 1e-5, rows=rows, dim=dim, ld_x=ld, **kw)  # noqa: E731
    y, mean, rstd = fwd()
    _refused(fwd, x=x.half())                                  # dtype
    _refused(fwd, x=x[:-1])                                    # shape
    _refused(fwd, x=_f32(dim, rows).t())                       # not contiguous
    _refused(fwd, x=x, ld=2 * dim)                             # rows ld_x apart do not fit in x
    _refused(fwd, g=g.to(torch.bfloat16))
    _refused(fwd, b=b[:-1])
    _refused(fwd, g=_f32(dim, 2)[:, 0])
    _refused(fwd, y_f32=torch.empty(rows, dim, dtype=torch.bfloat16, device="cuda"))
    _refused(fwd, y_f32=torch.empty(rows, dim - 1, device="cuda"))
    _refused(fwd, y_f32=_f32(dim, rows).t())
    dy, dx, dxb = _bf16(rows, dim), torch.empty(rows, dim, device="cuda"), torch.empty(rows, dim, dtype=torch.bfloat16, device="cuda")

    def bwd(dy=dy, x=x, mean=mean, rstd=rstd, dres=None, dx=dx, dxb=dxb, dg=None, db=None, colsum=None):
        return ops.layernorm_bwd(dy, x, g, mean, rstd, rows=rows, dim=dim, ld_x=dim, dres=dres, dx_out=dx, ld_dx=dim, dx_bf16=dxb,
                                 dgamma=_f32(dim) if dg is None else dg, dbeta=_f32(dim) if db is None else db, dx_colsum=colsum)

    bwd()
    _refused(bwd, dy=dy.half())
    _refused(bwd, dy=dy[:-1])
    _refused(bwd, dy=_bf16(dim, rows).t())
    _refused(bwd, x=x.double())
    _refused(bwd, mean=mean[:-1])
    _refused(bwd, rstd=rstd.to(torch.bfloat16))
    _refused(bwd, dres=_f32(rows - 1, dim))
    _refused(bwd, dres=_f32(dim, rows).t())
    _refused(bwd, dx=dx.to(torch.bfloat16))
    _refused(bwd, dxb=dx)
    _refused(bwd, dxb=_bf16(rows, 2 * dim)[:, :dim])
    _refused(bwd, dg=_f32(dim + 1))
    _refused(bwd, db=_f32(dim).double())
    _refused(bwd, colsum=_f32(dim, 2)[:, 0])
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_ops_colsum_and_wgrad_refuse_bad_tensors():
    M, n_out, k_in = 128, 64, 96
    dy, x = _bf16(M, n_out), _bf16(M, k_in)
    ops.colsum(dy, _f32(n_out))
    _refused(ops.colsum, dy.float(), _f32(n_out))
    _refused(ops.colsum, dy, _f32(n_out - 1))
    _refused(ops.colsum, dy, _f32(n_out).to(torch.bfloat16))
    _refused(ops.colsum, _bf16(n_out, M).t(), _f32(n_out))
    _refused(ops.colsum, dy, _f32(n_out, 2)[:, 0])
    ops.wgrad(dy, x, _f32(n_out, k_in))
    _refused(ops.wgrad, dy.half(), x, _f32(n_out, k_in))
    _refused(ops.wgrad, dy, x.float(), _f32(n_out, k_in))
    _refused(ops.wgrad, dy, x, _f32(n_out, k_in).to(torch.bfloat16))
    _refused(ops.wgrad, dy, x, _f32(n_out, k_in + 8))
    _refused(ops.wgrad, dy, x, _f32(k_in, n_out).t())
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_ops_glue_refuses_bad_tensors():
    B, np_, D, T = 2, 16, 64, 17
    patch, cls, pos = _bf16(B * np_, D), _f32(1, 1, D), _f32(1, T, D)
    ops.assemble_tokens(patch, cls, pos, B, np_, D)
    _refused(ops.assemble_tokens, patch.float(), cls, pos, B, np_, D)
    _refused(ops.assemble_tokens, patch[:-1], cls, pos, B, np_, D)
    _refused(ops.assemble_tokens, _bf16(D, B * np_).t(), cls, pos, B, np_, D)
    _refused(ops.assemble_tokens, patch, cls.half(), pos, B, np_, D)
    _refused(ops.assemble_tokens, patch, cls, pos[:, :-1], B, np_, D)
    _refused(ops.assemble_tokens, patch, cls, pos, B, np_, D, conv_bias=_f32(D))
    dnet, dpos, dcls = _f32(B, T, D), _f32(T, D), _f32(D)
    ops.assemble_tokens_bwd(dnet, dpos, dcls, B, np_, D)
    _refused(ops.assemble_tokens_bwd, dnet.to(torch.bfloat16), dpos, dcls, B, np_, D)
    _refused(ops.assemble_tokens_bwd, dnet[:, :-1], dpos, dcls, B, np_, D)
    _refused(ops.assemble_tokens_bwd, dnet, _f32(D, T).t(), dcls, B, np_, D)
    _refused(ops.assemble_tokens_bwd, dnet, dpos, _f32(D + 1), B, np_, D)
    x = _f32(B, T, D)
    ops.add_pos(x, pos, B, T, D)
    _refused(ops.add_pos, x.half(), pos, B, T, D)
    _refused(ops.add_pos, x[:, :-1], pos, B, T, D)
    _refused(ops.add_pos, x.transpose(0, 1).contiguous().transpose(0, 1), pos, B, T, D)
    _refused(ops.add_pos, x, pos.double(), B, T, D)
    ops.add_pos_bwd(dnet, dpos, B, T, D)
    _refused(ops.add_pos_bwd, dnet, dpos[:-1], B, T, D)
    _refused(ops.add_pos_bwd, dnet.half(), dpos, B, T, D)
    _refused(ops.add_pos_bwd, dnet, _f32(D, T).t(), B, T, D)
    ops.fill_f32(_f32(1000), 0.0)
    _refused(ops.fill_f32, _f32(1000).to(torch.bfloat16), 0.0)
    _refused(ops.fill_f32, _f32(100, 2)[:, 0], 0.0)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_ops_groupnorm_refuses_bad_tensors():
    B, HW, C = 2, 64, 64
    x, dy, g, b = _bf16(B, HW, C), _bf16(B, HW, C), _f32(C), _f32(C)
    y, mean, rstd = ops.groupnorm_silu_fwd(x, g, b, 1e-5)
    _refused(ops.groupnorm_silu_fwd, x, g.to(torch.bfloat16), b, 1e-5)
    _refused(ops.groupnorm_silu_fwd, x, g, b[:-1], 1e-5)
    _refused(ops.groupnorm_silu_fwd, x, _f32(C, 2)[:, 0], b, 1e-5)
    bwd = lambda **kw: ops.groupnorm_silu_bwd(**dict(dict(x=x, dy=dy, gamma=g, beta=b, mean=mean, rstd=rstd), **kw))  # noqa: E731
    bwd()
    _refused(bwd, x=x.float())
    _refused(bwd, x=_bf16(B, C, HW).transpose(1, 2))
    _refused(bwd, gamma=g[:-1])
    _refused(bwd, beta=b.double())
    _refused(bwd, mean=mean.half())
    _refused(bwd, rstd=rstd[:, :-1])
    _refused(bwd, mean=_f32(32, B).t())
    _refused(bwd, dgamma=_f32(C + 1), dbeta=_f32(C))
    _refused(bwd, dgamma=_f32(C), dbeta=_f32(C, 2)[:, 0])
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_ops_text_glue_refuses_bad_tensors():
    V, D, B, T = 50, 64, 2, 7
    w, ids = _f32(V, D), torch.randint(0, V, (B, T), device="cuda")
    ops.embedding_fwd(ids, w)
    _refused(ops.embedding_fwd, ids.int(), w)                  # dtype
    _refused(ops.embedding_fwd, ids.t(), w)                    # not contiguous
    _refused(ops.embedding_fwd, ids, w.to(torch.bfloat16))     # e.g. the weight of CLIPB200.bfloat16()
    _refused(ops.embedding_fwd, ids, w.reshape(-1))            # shape
    _refused(ops.embedding_fwd, ids, _f32(D, V).t())
    dnet = _f32(B, T, D)
    ops.embedding_bwd(ids, dnet, V, D, 0)
    _refused(ops.embedding_bwd, ids.int(), dnet, V, D, 0)
    _refused(ops.embedding_bwd, ids.t(), dnet, V, D, 0)
    _refused(ops.embedding_bwd, ids, dnet.half(), V, D, 0)
    _refused(ops.embedding_bwd, ids, dnet[:-1], V, D, 0)
    _refused(ops.embedding_bwd, ids, dnet.transpose(0, 1), V, D, 0)
    net = _f32(B, T, D)
    _, pos = ops.argmax_gather_rows(net, ids)
    _refused(ops.argmax_gather_rows, net.half(), ids)
    _refused(ops.argmax_gather_rows, net.reshape(B * T, D), ids)
    _refused(ops.argmax_gather_rows, _f32(B, D, T).transpose(1, 2), ids)
    _refused(ops.argmax_gather_rows, net, ids.int())
    _refused(ops.argmax_gather_rows, net, ids[:, :-1])         # ids do not match net's [B, T]
    _refused(ops.argmax_gather_rows, _f32(B, T + 1, D), ids)
    _refused(ops.argmax_gather_rows, net, ids.t().contiguous().t())
    dout = _f32(B, D)
    ops.scatter_rows(dout, pos, T)
    _refused(ops.scatter_rows, dout.double(), pos, T)
    _refused(ops.scatter_rows, dout[:-1], pos, T)
    _refused(ops.scatter_rows, _f32(D, B).t(), pos, T)
    _refused(ops.scatter_rows, dout, pos.long(), T)
    _refused(ops.scatter_rows, dout, pos[:-1], T)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_ops_symmetric_xent_refuses_bad_tensors():
    B = 16
    logits, dl = _bf16(B, B), torch.empty(B, B, dtype=torch.bfloat16, device="cuda")
    ops.symmetric_xent(logits)
    ops.symmetric_xent(logits, dlogits=dl, grad_scale_dev=_f32(1))
    _refused(ops.symmetric_xent, logits.float())
    _refused(ops.symmetric_xent, logits[:, :-1])               # not square
    _refused(ops.symmetric_xent, _bf16(B, B).t())              # inner stride
    _refused(ops.symmetric_xent, logits, dlogits=dl.float())
    _refused(ops.symmetric_xent, logits, dlogits=dl[:-1])
    _refused(ops.symmetric_xent, logits, dlogits=_bf16(B, 2 * B)[:, :B])  # another row stride than the logits'
    _refused(ops.symmetric_xent, logits, grad_scale_dev=_f32(2))
    _refused(ops.symmetric_xent, logits, grad_scale_dev=_f32(1).half())
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_ops_adam_step_refuses_bad_tensors():
    n = 1024
    p, g, m, v = _f32(n), _f32(n), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    hyper, step = torch.tensor([1e-3, 0.9, 0.999, 1e-8, 0.0, 1.0], device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    host = lambda **kw: ops.adam_step(**dict(dict(params=p, grads=g, exp_avg=m, exp_avg_sq=v, hyper=(1e-3, 0.9, 0.999, 1e-8, 0.0),  # noqa: E731
                                                  step=1), **kw))
    dev = lambda **kw: ops.adam_step(**dict(dict(params=p, grads=g, exp_avg=m, exp_avg_sq=v, hyper_dev=hyper, step_dev=step), **kw))  # noqa: E731
    host()
    dev()
    _refused(host, params=p.double())
    _refused(host, params=_f32(2 * n)[::2])
    _refused(host, grads=g[:-4])
    _refused(host, exp_avg=_f32(2 * n)[::2])
    _refused(host, exp_avg_sq=v.to(torch.bfloat16))
    _refused(dev, hyper_dev=hyper[:5])
    _refused(dev, hyper_dev=hyper.double())
    _refused(dev, step_dev=step.long())
    _refused(dev, step_dev=None)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_ops_fcnn_step_refuses_bad_tensors():
    dims, woff, boff, P = [10, 32, 1], [0, 352], [320, 384], 388  # the arena of DIMS / WOFF / BOFF above
    M = 128
    params, x, y, grads = _f32(P) * 0.1, _f32(M, 10), _f32(M, 1), torch.empty(P, device="cuda")
    step = lambda **kw: ops.fcnn_step(**dict(dict(x=x, params=params, dims=dims, w_offsets=woff, b_offsets=boff, y=y,  # noqa: E731
                                                  grads=grads), **kw))
    step()
    step(y=None, dpred=_f32(M, 1))
    step(y=None, grads=None)
    _refused(step, x=x.double())
    _refused(step, x=_f32(M, 11))
    _refused(step, x=_f32(10, M).t())
    _refused(step, params=params.half())
    _refused(step, params=_f32(2 * P)[::2])
    _refused(step, y=y[:-1])
    _refused(step, y=y.half())
    _refused(step, y=None, dpred=_f32(M, 2))
    _refused(step, grads=grads[:-1])
    _refused(step, grads=_f32(P, 2)[:, 0])
    torch.cuda.synchronize()
