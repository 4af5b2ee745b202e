"""The SD-UNet's ResBlock on native kernels: the per-image and clamped-residual conv3x3 epilogues, the per-image column sums,
and ResidualBlockWithTimeEmbeddingB200 against oracle/unet_oracle.py::res_block.  The CPU cases check the C-ABI argument checks,
the module's parameters against the reference's and the refusals; the others need an H100 (pytest -m gpu)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import ops  # noqa: E402
from cflearn_b200._cabi import B200Error  # noqa: E402
from cflearn_b200.unet_blocks import ResidualBlockWithTimeEmbeddingB200 as ResBlock, res_block_forward  # noqa: E402
from _refs import rand_bf16, relerr  # noqa: E402

DEV = "cuda"
BF16_MAX = torch.finfo(torch.bfloat16).max


def _conv_case(B, side, Cin, Cout, seed):
    x = rand_bf16(B, side, side, Cin, seed=seed)
    w = rand_bf16(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=seed + 1)
    bias = rand_bf16(Cout, scale=0.1, seed=seed + 2)
    return x, ops.pack_conv3x3_weight(w), bias


# ---- 1. conv epilogues and the per-image column sums ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("side", [64, 32, 16, 8])
def test_per_image_epilogue(side):
    B, Cin, Cout = 3, 128, 320  # at 8x8 a 128-pixel tile holds two images, and B = 3 leaves the last tile half full
    x, wp, bias = _conv_case(B, side, Cin, Cout, seed=side)
    t = rand_bf16(B, Cout, seed=side + 3)
    out = ops.conv3x3(x, wp, bias, epilogue=ops.EPI_BIAS_ADD_PER_IMAGE_BF16, aux=t)
    expect = ops.conv3x3(x, wp, bias) + t[:, None, None, :]  # eager's bf16 add of the broadcast table
    assert torch.equal(out, expect)


@pytest.mark.gpu
def test_clamp_epilogue():
    B, side, Cin, Cout = 2, 16, 64, 256
    x, wp, _ = _conv_case(B, side, Cin, Cout, seed=20)
    # finite sums: the bf16 residual add, bit for bit
    aux = rand_bf16(B, side, side, Cout, seed=21)
    bias = rand_bf16(Cout, scale=0.1, seed=22)
    out = ops.conv3x3(x, wp, bias, epilogue=ops.EPI_BIAS_RESID_CLAMP_BF16, aux=aux)
    assert torch.equal(out, ops.conv3x3(x, wp, bias) + aux)
    # overflowing sums: +-inf becomes +-bf16 max, as torch.clamp to the finite range does; NaN stays NaN
    big = torch.full((Cout,), 1e37, device=DEV).to(torch.bfloat16)
    big[1::2] *= -1
    aux = torch.full((B, side, side, Cout), BF16_MAX, device=DEV, dtype=torch.bfloat16)
    aux[..., 1::2] *= -1          # same sign as the bias: those sums overflow
    aux[:, ::3, :, :4] *= -1      # opposite sign: finite
    aux[0, 1, 2, 5] = float("nan")
    aux[1, 3, 4, 0] = float("inf")
    out = ops.conv3x3(x, wp, big, epilogue=ops.EPI_BIAS_RESID_CLAMP_BF16, aux=aux)
    expect = (ops.conv3x3(x, wp, big) + aux).clamp(-BF16_MAX, BF16_MAX)
    nan = torch.isnan(out)
    assert torch.equal(nan, torch.isnan(expect)) and nan[0, 1, 2, 5] and nan.sum().item() == 1
    assert torch.equal(out[~nan], expect[~nan])
    assert not torch.isinf(out).any()
    assert (out == BF16_MAX).any() and (out == -BF16_MAX).any()


@pytest.mark.gpu
@pytest.mark.parametrize("B,HW,C", [(2, 4096, 320), (8, 1024, 640), (3, 64, 2560), (5, 72, 8)])
def test_colsum_per_image(B, HW, C):
    x = rand_bf16(B, HW, C, seed=B + C)
    dt, db = ops.colsum_per_image(x)
    dt2, db2 = ops.colsum_per_image(x)
    torch.cuda.synchronize()
    assert torch.equal(dt, dt2) and torch.equal(db, db2)  # deterministic: no atomics
    ref = x.double().sum(1)
    bad = (dt.double() - ref).abs() > 2.0 ** -8 * ref.abs() + 1e-4 * HW ** 0.5  # one bf16 rounding of an fp32 sum
    assert dt.dtype == torch.bfloat16 and bad.sum().item() == 0
    tot = ref.sum(0)
    assert db.dtype == torch.float32 and torch.equal(db, db.to(torch.bfloat16).float())  # the rounded sum, widened
    assert ((db.double() - tot).abs() > 2.0 ** -8 * tot.abs() + 1e-4 * (B * HW) ** 0.5).sum().item() == 0


# ---- 2. module parity against the oracle ---------------------------------------------------------------------------------------
def _block(Cin, Cout, tdim, seed):
    import unet_oracle as uo

    m = ResBlock(Cin, Cout, norm_eps=1e-5, time_embedding_channels=tdim)
    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=seed)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def _inputs(B, Cin, Cout, side, tdim, seed):
    g = torch.Generator().manual_seed(seed)
    net = torch.randn(B, Cin, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    tn = torch.randn(B, tdim, generator=g).to(DEV).to(torch.bfloat16)
    up = torch.randn(B, Cout, side, side, generator=g).to(DEV)
    return net, tn, up


def _check(ours, eager, fp32):
    for k in ours:
        floor = relerr(eager[k], fp32[k])
        assert relerr(ours[k], fp32[k]) <= 1.5 * floor + 1e-6, (k, relerr(ours[k], fp32[k]), floor)
        assert relerr(ours[k], eager[k]) <= 2.0 * floor + 1e-6, (k, relerr(ours[k], eager[k]), floor)


def _oracle_run(sd, net, tn, up):
    import unet_oracle as uo

    refs = []
    for autocast in (True, False):
        sdg = {k: v.detach().clone().to(DEV).requires_grad_(True) for k, v in sd.items()}
        x = (net if autocast else net.float()).detach().clone().requires_grad_(True)
        t = (tn if autocast else tn.float()).detach().clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            y = uo.res_block(sdg, "", x, t)
        (y.float() * up).sum().backward()
        refs.append({"out": y, "net": x.grad, "time_net": t.grad, **{k: v.grad for k, v in sdg.items()}})
    return refs


def _run_module(m, net, tn, up):
    x = net.detach().clone().requires_grad_(True)
    t = None if tn is None else tn.detach().clone().requires_grad_(True)
    y = m(x, t)
    (y.float() * up).sum().backward()
    assert y.dtype == torch.bfloat16 and x.grad.dtype == torch.bfloat16
    res = {"out": y, "net": x.grad, **{k: p.grad for k, p in m.named_parameters() if p.grad is not None}}
    if t is not None:
        res["time_net"] = t.grad
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,side,tdim", [(320, 320, 64, 1280), (320, 640, 32, 1280), (1920, 1280, 16, 1280),
                                                 (2560, 1280, 8, 1280), (128, 64, 16, 128)])
def test_res_block_parity(Cin, Cout, side, tdim):
    """SD-v1.5 shapes at B = 2, and the tiny UNet's output_blocks.0.0 (128 -> 64, time width 128)."""
    m, sd = _block(Cin, Cout, tdim, seed=Cin + Cout + side)
    net, tn, up = _inputs(2, Cin, Cout, side, tdim, seed=side)
    ours = _run_module(m, net, tn, up)
    assert ours["out"].is_contiguous(memory_format=torch.channels_last) and ours["time_net"].dtype == torch.bfloat16
    eager, fp32 = _oracle_run(sd, net, tn, up)
    _check(ours, eager, fp32)


@pytest.mark.gpu
def test_without_time_embedding():
    """time_net=None skips the add, as the reference does: the same block with a zeroed time embedding gives the same output
    and input gradient, and the time embedding gets no gradient."""
    Cin, Cout, side, tdim = 320, 640, 16, 1280
    m, sd = _block(Cin, Cout, tdim, seed=40)
    net, tn, up = _inputs(2, Cin, Cout, side, tdim, seed=41)
    none = _run_module(m, net, None, up)
    assert m.time_embedding.weight.grad is None and m.time_embedding.bias.grad is None
    m.zero_grad(set_to_none=True)
    with torch.no_grad():
        m.time_embedding.weight.zero_()
        m.time_embedding.bias.zero_()
    zero = _run_module(m, net, torch.zeros_like(tn), up)
    for k in none:  # conv1's bias gradient is summed in another order (per image first) when a time embedding is present
        if k == "conv1.bias":
            assert relerr(none[k], zero[k]) < 1e-2
        else:
            assert torch.equal(none[k], zero[k]), k
    sd0 = dict(sd, **{"time_embedding.weight": torch.zeros_like(sd["time_embedding.weight"]),
                      "time_embedding.bias": torch.zeros_like(sd["time_embedding.bias"])})
    eager, fp32 = _oracle_run(sd0, net, torch.zeros_like(tn), up)
    _check(none, eager, fp32)


@pytest.mark.gpu
@pytest.mark.parametrize("B,side,Cin,Cout", [(2, 64, 320, 320), (2, 16, 640, 1280), (3, 8, 1280, 1280)])
def test_res_block_forward_is_the_previous_composition(B, side, Cin, Cout):
    """res_block_forward now runs the fused epilogues; its output is bit-identical to the separate bf16 adds and clamp."""
    import unet_oracle as uo

    tdim = 1280
    m = ResBlock(Cin, Cout, time_embedding_channels=tdim)
    sd = {"b." + k: v.to(DEV) for k, v in uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=3).items()}
    x = rand_bf16(B, side, side, Cin, seed=4)
    tn = rand_bf16(B, tdim, seed=5)
    ours = res_block_forward(sd, "b.", x, tn)

    bf = lambda t: t.to(torch.bfloat16).contiguous()  # noqa: E731
    p = "b."
    y, _, _ = ops.groupnorm_silu_fwd(x.reshape(B, side * side, Cin), sd[p + "norm1.weight"].float().contiguous(), sd[p + "norm1.bias"].float().contiguous(), 1e-5)
    h = ops.conv3x3(y.view(B, side, side, Cin), ops.pack_conv3x3_weight(sd[p + "conv1.weight"]), bf(sd[p + "conv1.bias"]))
    t = ops.gemm(torch.nn.functional.silu(tn).contiguous(), bf(sd[p + "time_embedding.weight"]), bias=bf(sd[p + "time_embedding.bias"]))
    h = h + t[:, None, None, :]
    y2, _, _ = ops.groupnorm_silu_fwd(h.reshape(B, side * side, Cout), sd[p + "norm2.weight"].float().contiguous(), sd[p + "norm2.bias"].float().contiguous(), 1e-5)
    h2 = ops.conv3x3(y2.view(B, side, side, Cout), ops.pack_conv3x3_weight(sd[p + "conv2.weight"]), bf(sd[p + "conv2.bias"]))
    inp = x
    if Cin != Cout:
        ws = sd[p + "shortcut.weight"]
        inp = ops.gemm(x.reshape(-1, Cin), bf(ws.reshape(Cout, Cin)), bias=bf(sd[p + "shortcut.bias"])).view(B, side, side, Cout)
    expect = (inp + h2).clamp(-BF16_MAX, BF16_MAX)
    assert torch.equal(ours, expect)


@pytest.mark.gpu
def test_deterministic_and_memory_format():
    Cin, Cout, side, tdim = 640, 1280, 16, 1280
    m, _ = _block(Cin, Cout, tdim, seed=50)
    net, tn, up = _inputs(2, Cin, Cout, side, tdim, seed=51)
    runs = []
    for x in (net.contiguous(memory_format=torch.channels_last), net.contiguous(), net.contiguous(memory_format=torch.channels_last)):
        m.zero_grad(set_to_none=True)
        runs.append(_run_module(m, x, tn, up))
    for r in runs[1:]:
        for k in runs[0]:
            assert torch.equal(r[k], runs[0][k]), k


def _small_case():
    m, _ = _block(320, 640, 1280, seed=60)
    net, tn, _ = _inputs(2, 320, 640, 16, 1280, seed=61)
    return m, net, tn


@pytest.mark.gpu
def test_backward_twice_with_retain_graph():
    m, net, tn = _small_case()
    x, t = net.detach().requires_grad_(True), tn.detach().requires_grad_(True)
    y = m(x, t)
    up = torch.randn(y.shape, generator=torch.Generator().manual_seed(62)).to(DEV).to(y.dtype)
    y.backward(up, retain_graph=True)
    first = {"x": x.grad.clone(), "t": t.grad.clone(), **{k: p.grad.clone() for k, p in m.named_parameters()}}
    y.backward(up)
    second = {"x": x.grad, "t": t.grad, **{k: p.grad for k, p in m.named_parameters()}}
    for k in first:  # the second pass adds the same gradients again (doubling is exact)
        assert torch.equal(second[k], 2 * first[k]), k


@pytest.mark.gpu
def test_in_place_change_of_the_input_is_detected():
    m, net, tn = _small_case()
    leaf = net.detach().requires_grad_(True)
    inp = leaf * 1  # a non-leaf channels-last bf16 input, saved as is (no copy)
    y = m(inp, tn)
    inp.add_(1)
    with pytest.raises(RuntimeError, match="inplace"):
        y.backward(torch.ones_like(y))


@pytest.mark.gpu
def test_bf16_parameters():
    """After module.to(bfloat16) the GroupNorm parameters are bf16: the kernels get fp32 copies, the gradients come back bf16."""
    m, net, tn = _small_case()
    m = m.to(torch.bfloat16)
    x = net.detach().requires_grad_(True)
    m(x, tn).float().sum().backward()
    assert torch.isfinite(x.grad.float()).all()
    for k, p in m.named_parameters():
        assert p.grad.dtype == torch.bfloat16 and torch.isfinite(p.grad.float()).all(), k


_FIRST_WORK = """
import sys, torch
sys.path.insert(0, sys.argv[1])
import cflearn_b200
from cflearn_b200.unet_blocks import ResidualBlockWithTimeEmbeddingB200
torch.manual_seed(0)
m = ResidualBlockWithTimeEmbeddingB200(320, 640, time_embedding_channels=1280).cuda()
x = torch.randn(2, 320, 16, 16, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
t = torch.randn(2, 1280, device="cuda").to(torch.bfloat16).requires_grad_(True)
y = m(x, t)
y.backward(torch.ones_like(y))  # bf16 in y's layout: no cast runs before the Function's backward on autograd's thread
torch.cuda.synchronize()
assert torch.isfinite(x.grad.float()).all() and torch.isfinite(t.grad.float()).all()
print("ok")
"""


@pytest.mark.gpu
def test_backward_as_the_first_cuda_work_of_autograds_thread():
    """In a fresh process, the block's backward is the first CUDA work on autograd's device thread."""
    import subprocess

    res = subprocess.run([sys.executable, "-c", _FIRST_WORK, ROOT], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert res.returncode == 0 and res.stdout.strip().endswith("ok"), res.stdout[-3000:]


# ---- 3. CPU: C-ABI argument checks, parameters, refusals ----------------------------------------------------------------------
def _golden_shapes(prefix):
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "unet_tiny_reference.pt"), weights_only=False)
    return [(k[len(prefix):], tuple(s)) for k, s in fx["shapes"] if k.startswith(prefix)]


@pytest.mark.parametrize("prefix", ["input_blocks.1.0.", "input_blocks.3.0.", "output_blocks.0.0."])
def test_module_matches_reference_parameters(prefix):
    shapes = _golden_shapes(prefix)
    d = dict(shapes)
    Cin, Cout, tdim = d["norm1.weight"][0], d["conv1.weight"][0], d["time_embedding.weight"][1]
    m = ResBlock(Cin, Cout, norm_eps=1e-5, time_embedding_channels=tdim)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == shapes
    assert all(v.dtype == torch.float32 for v in m.state_dict().values())
    assert torch.count_nonzero(m.conv2.weight) == 0  # zero_module(conv2)
    sd = {k: torch.randn(s) for k, s in shapes}
    m.load_state_dict(sd, strict=True)
    back = ResBlock(Cin, Cout, norm_eps=1e-5, time_embedding_channels=tdim)
    back.load_state_dict(m.state_dict(), strict=True)
    assert all(torch.equal(back.state_dict()[k], sd[k]) for k in sd)


def test_module_refuses_unsupported_configurations():
    for kw in (dict(dropout=0.1), dict(use_scale_shift_norm=True), dict(integrate_upsample=True), dict(integrate_downsample=True),
               dict(signal_dim=3), dict(time_embedding_channels=0)):
        with pytest.raises(NotImplementedError):
            ResBlock(64, 64, **kw)
    with pytest.raises(NotImplementedError):
        ResBlock(64, 128, use_conv_shortcut=True)
    ResBlock(64, 64, use_conv_shortcut=True)  # no shortcut when the width is kept: accepted, as in the reference
    ResBlock(64, 64, use_checkpoint=True)     # accepted: memory only
    z = lambda *s, dtype=torch.bfloat16: torch.zeros(*s, dtype=dtype)  # noqa: E731
    bad = [
        (ResBlock(96, 96, time_embedding_channels=64), z(1, 96, 8, 8), "multiple of 64"),
        (ResBlock(2624, 64, time_embedding_channels=64), z(1, 2624, 8, 8), "at most 2560"),
        (ResBlock(64, 64, time_embedding_channels=64), z(1, 64, 12, 48), "divide 64"),
        (ResBlock(64, 64, time_embedding_channels=64), z(1, 64, 4, 4), "multiple of 64"),
        (ResBlock(64, 64, time_embedding_channels=64), z(1, 64, 8, 8), "CUDA"),
        (ResBlock(64, 64, time_embedding_channels=64), z(1, 64, 8, 8, dtype=torch.float32), "CUDA|bf16"),
    ]
    for m, x, reason in bad:
        with pytest.raises(B200Error, match=reason):
            m(x, z(1, 64))
    if torch.cuda.is_available():
        m = ResBlock(64, 64, time_embedding_channels=64).to(DEV)
        with pytest.raises(B200Error, match="bf16"):
            m(torch.zeros(1, 64, 8, 8, device=DEV), torch.zeros(1, 64, device=DEV, dtype=torch.bfloat16))
