"""The SD-UNet's SpatialTransformer on native kernels: the GEGLU / dGEGLU / bf16-residual GEMM epilogues, LayerNorm over bf16
rows, and SpatialTransformerBlockB200 / SpatialTransformerB200 against oracle/unet_oracle.py::transformer_block /
::spatial_transformer.  The CPU cases check the C-ABI argument checks, the modules' parameters against the reference's and the
refusals; the others need an H100 (pytest -m gpu)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import ops  # noqa: E402
from cflearn_b200._cabi import B200Error  # noqa: E402
from cflearn_b200.attention import CrossAttentionB200  # noqa: E402
from cflearn_b200.spatial_transformer import SpatialTransformerB200, SpatialTransformerBlockB200  # noqa: E402
from _refs import assert_ulp, rand_bf16, relerr  # noqa: E402

DEV = "cuda"


# ---- 1. GEMM epilogues -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("F_", [8, 200, 1280, 5120])
def test_geglu_epilogue(F_):
    M, K = 300, 320
    x, w1, b1 = rand_bf16(M, K, seed=1), rand_bf16(2 * F_, K, scale=K ** -0.5, seed=2), rand_bf16(2 * F_, scale=0.1, seed=3)
    outs = [ops.geglu(x, w1, b1, max_ctas=c) for c in (0, 5, 1)]
    torch.cuda.synchronize()
    hg, a = outs[0]
    for h2, a2 in outs[1:]:
        assert torch.equal(h2, hg) and torch.equal(a2, a)
    ref = x.float() @ w1.float().t() + b1.float()
    assert hg.shape == (M, 2 * F_) and a.shape == (M, F_)
    assert ((hg.float() - ref).abs() > 0.02 * ref.abs().clamp_min(1.0)).sum().item() == 0  # one bf16 rounding of the product
    assert torch.equal(hg, ops.gemm(x, w1, bias=b1))  # the same staging tile as the plain bias epilogue
    h, gate = hg.chunk(2, dim=-1)
    assert_ulp(a, h * F.gelu(gate), f"geglu F {F_}", ulps=2, floor=1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("F_", [8, 200, 1280])
def test_dgeglu_epilogue(F_):
    M, C = 300, 320
    dy, w2 = rand_bf16(M, C, seed=4), rand_bf16(C, F_, scale=C ** -0.5, seed=5)
    hg = rand_bf16(M, 2 * F_, seed=6)
    dhg = ops.gemm(dy, w2, b_mn_major=True, epilogue=ops.EPI_DGEGLU_BF16, aux=hg)
    da = ops.gemm(dy, w2, b_mn_major=True)  # the dgrad's own rounding of the upstream gradient
    torch.cuda.synchronize()
    h, gate = (t.detach().requires_grad_(True) for t in hg.chunk(2, dim=-1))
    (h * F.gelu(gate)).backward(da)
    dh, dgate = dhg.chunk(2, dim=-1)
    assert_ulp(dh, h.grad, f"dgeglu F {F_}: dh", ulps=2, floor=1e-3)
    assert_ulp(dgate, gate.grad, f"dgeglu F {F_}: dgate", ulps=2, floor=1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(300, 1003, 192), (77, 320, 640), (4096, 1280, 1280)])
def test_bf16_residual_epilogue(M, N, K):
    a, b, bias = rand_bf16(M, K, seed=7), rand_bf16(N, K, scale=K ** -0.5, seed=8), rand_bf16(N, seed=9)
    npad = (N + 7) // 8 * 8
    res = torch.empty(M, npad, dtype=torch.bfloat16, device=DEV)[:, :N]
    res.copy_(rand_bf16(M, N, seed=10))
    expect = ops.gemm(a, b, bias=bias) + res
    out = ops.gemm(a, b, bias=bias, epilogue=ops.EPI_BIAS_RESID_BF16, aux=res)
    assert torch.equal(out, expect)
    ops.gemm(a, b, bias=bias, epilogue=ops.EPI_BIAS_RESID_BF16, aux=res, out0=res)  # in place
    assert torch.equal(res, expect)


# ---- 2. LayerNorm over bf16 rows ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dim", [32, 320, 640, 1280])
@pytest.mark.parametrize("with_dres", [False, True])
def test_layernorm_bf16(dim, with_dres):
    rows = 4099
    x = rand_bf16(rows, dim, scale=2.0, seed=dim) + 0.5
    g = torch.Generator().manual_seed(1)
    gamma = (1 + 0.1 * torch.randn(dim, generator=g)).to(DEV)
    beta = (0.1 * torch.randn(dim, generator=g)).to(DEV)
    dy = rand_bf16(rows, dim, seed=dim + 1)
    dres = rand_bf16(rows, dim, seed=dim + 2) if with_dres else None
    y, mean, rstd = ops.layernorm_bf16_fwd(x, gamma, beta, 1e-5)
    dx, dgamma, dbeta = ops.layernorm_bf16_bwd(dy, x, gamma, mean, rstd, dres=dres)
    dx2, dgamma2, dbeta2 = ops.layernorm_bf16_bwd(dy, x, gamma, mean, rstd, dres=dres)
    torch.cuda.synchronize()
    assert torch.equal(dx, dx2) and torch.equal(dgamma, dgamma2) and torch.equal(dbeta, dbeta2)
    xf = x.float().requires_grad_(True)
    gf, bf = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    yf = F.layer_norm(xf, (dim,), gf, bf, 1e-5)
    yf.backward(dy.float())
    assert_ulp(y, yf.to(torch.bfloat16), f"layernorm_bf16 dim {dim}: y", floor=1e-3)
    ref_dx = xf.grad.to(torch.bfloat16)
    if dres is not None:
        ref_dx = ref_dx + dres  # eager: the LayerNorm gradient rounded to the bf16 input, then the bf16 residual add
    assert_ulp(dx, ref_dx, f"layernorm_bf16 dim {dim}: dx", ulps=2, floor=1e-3)
    assert relerr(dgamma, gf.grad) < 1e-4 and relerr(dbeta, bf.grad) < 1e-4


# ---- 3. module parity against the oracle ------------------------------------------------------------------------------------------
def _transformer_sd(C, ctx_dim, seed):
    import unet_oracle as uo

    m = SpatialTransformerB200(C, 8, C // 8, context_dim=ctx_dim)
    shapes = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    return uo.synthetic_state_dict(shapes, seed=seed)


def _check(ours, eager, fp32):
    for k in ours:
        floor = relerr(eager[k], fp32[k])
        assert relerr(ours[k], fp32[k]) <= 1.5 * floor + 1e-6, (k, relerr(ours[k], fp32[k]), floor)
        assert relerr(ours[k], eager[k]) <= 2.0 * floor + 1e-6, (k, relerr(ours[k], eager[k]), floor)


def _oracle_run(fn, sd, prefix, net, context, heads, up):
    refs = []
    for autocast in (True, False):
        sdg = {k: v.detach().clone().requires_grad_(True) for k, v in sd.items()}
        x = (net if autocast else net.float()).detach().clone().requires_grad_(True)
        c = context.detach().clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            y = fn(sdg, prefix, x, c, heads)
        (y.float() * up).sum().backward()
        refs.append({"out": y, "net": x.grad, "context": c.grad, **{k[len(prefix):]: v.grad for k, v in sdg.items()}})
    return refs


def _run_module(m, net, context, up):
    x = net.detach().clone().requires_grad_(True)
    c = context.detach().clone().requires_grad_(True)
    y = m(x, c)
    (y.float() * up).sum().backward()
    assert y.dtype == torch.bfloat16 and x.grad.dtype == torch.bfloat16 and c.grad.dtype == torch.float32
    return {"out": y, "net": x.grad, "context": c.grad, **{k: p.grad for k, p in m.named_parameters()}}


@pytest.mark.gpu
@pytest.mark.parametrize("C,side", [(320, 64), (1280, 16), (1280, 8)])
def test_transformer_parity(C, side):
    import unet_oracle as uo

    B, heads = 2, 8
    sd = _transformer_sd(C, 768, seed=C + side)
    m = SpatialTransformerB200(C, heads, C // heads, context_dim=768).to(DEV)
    m.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(5)
    net = torch.randn(B, C, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    context = torch.randn(B, 77, 768, generator=g).to(DEV)
    up = torch.randn(B, C, side, side, generator=g).to(DEV)
    ours = _run_module(m, net, context, up)
    assert ours["out"].is_contiguous(memory_format=torch.channels_last)
    eager, fp32 = _oracle_run(uo.spatial_transformer, {k: v.to(DEV) for k, v in sd.items()}, "", net, context, heads, up)
    _check(ours, eager, fp32)


@pytest.mark.gpu
@pytest.mark.parametrize("C,side", [(320, 64), (1280, 16), (1280, 8)])
def test_block_parity(C, side):
    import unet_oracle as uo

    B, heads = 2, 8
    blk = SpatialTransformerBlockB200(C, heads, C // heads, context_dim=768).to(DEV)
    shapes = [(k, tuple(v.shape)) for k, v in blk.state_dict().items()]
    sd = uo.synthetic_state_dict(shapes, seed=C)
    blk.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(6)
    net = torch.randn(B, side * side, C, generator=g).to(DEV).to(torch.bfloat16)
    context = torch.randn(B, 77, 768, generator=g).to(DEV)
    up = torch.randn(B, side * side, C, generator=g).to(DEV)
    ours = _run_module(blk, net, context, up)
    eager, fp32 = _oracle_run(uo.transformer_block, {k: v.to(DEV) for k, v in sd.items()}, "", net, context, heads, up)
    _check(ours, eager, fp32)


def _tiny_prefix_sd():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "unet_tiny_reference.pt"), weights_only=False)
    p = "input_blocks.1.1."
    return p, [(k[len(p):], tuple(s)) for k, s in fx["shapes"] if k.startswith(p)], fx


@pytest.mark.gpu
def test_tiny_unet_transformer_parity():
    import unet_oracle as uo

    p, shapes, fx = _tiny_prefix_sd()
    cfg = uo.unet_config("unet_tiny")
    C, heads = shapes[0][1][0], cfg["num_heads"]
    sd = uo.synthetic_state_dict(shapes, seed=11)
    m = SpatialTransformerB200(C, heads, C // heads, context_dim=cfg["context_dim"]).to(DEV)
    m.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(7)
    net = torch.randn(2, C, 16, 16, generator=g).to(DEV).to(torch.bfloat16)
    context = torch.randn(2, 77, cfg["context_dim"], generator=g).to(DEV)
    up = torch.randn(2, C, 16, 16, generator=g).to(DEV)
    ours = _run_module(m, net, context, up)
    eager, fp32 = _oracle_run(uo.spatial_transformer, {k: v.to(DEV) for k, v in sd.items()}, "", net, context, heads, up)
    _check(ours, eager, fp32)


@pytest.mark.gpu
def test_deterministic_and_memory_format():
    C, side, B = 640, 32, 2
    m = SpatialTransformerB200(C, 8, C // 8, context_dim=768).to(DEV)
    m.load_state_dict(_transformer_sd(C, 768, seed=3), strict=True)
    g = torch.Generator().manual_seed(8)
    net = torch.randn(B, C, side, side, generator=g).to(DEV).to(torch.bfloat16)
    context = torch.randn(B, 77, 768, generator=g).to(DEV)
    up = torch.randn(B, C, side, side, generator=g).to(DEV)
    runs = []
    for x in (net.contiguous(memory_format=torch.channels_last), net.contiguous(), net.contiguous(memory_format=torch.channels_last)):
        m.zero_grad(set_to_none=True)
        runs.append(_run_module(m, x, context, up))
    for r in runs[1:]:
        for k in runs[0]:
            assert torch.equal(r[k], runs[0][k]), k


_FIRST_WORK = """
import sys, torch
sys.path.insert(0, sys.argv[1])
import cflearn_b200
from cflearn_b200.attention import CrossAttentionB200
from cflearn_b200.spatial_transformer import SpatialTransformerB200, SpatialTransformerBlockB200
which = sys.argv[2]
torch.manual_seed(0)
if which == "transformer":
    m = SpatialTransformerB200(320, 8, 40).cuda()
    x = torch.randn(2, 320, 16, 16, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
else:
    m = (CrossAttentionB200(query_dim=320, num_heads=8, head_dim=40) if which == "cross_attention" else SpatialTransformerBlockB200(320, 8, 40)).cuda()
    x = torch.randn(2, 256, 320, device="cuda").to(torch.bfloat16)
x.requires_grad_(True)
y = m(x)
y.backward(torch.ones_like(y))  # bf16 in y's layout: no cast runs before the Function's backward on autograd's thread
torch.cuda.synchronize()
assert torch.isfinite(x.grad.float()).all()
print("ok")
"""


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["cross_attention", "block", "transformer"])
def test_backward_as_the_first_cuda_work_of_autograds_thread(which):
    """In a fresh process, the module's backward is the first CUDA work on autograd's device thread, so its first GEMM encodes a
    tensor map before anything there has made a CUDA context current."""
    import subprocess

    res = subprocess.run([sys.executable, "-c", _FIRST_WORK, ROOT, which], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         timeout=600)
    assert res.returncode == 0 and res.stdout.strip().endswith("ok"), res.stdout[-3000:]


def _small_case(which):
    g = torch.Generator().manual_seed(12)
    if which == "transformer":
        m = SpatialTransformerB200(320, 8, 40, context_dim=768).to(DEV)
        m.load_state_dict(_transformer_sd(320, 768, seed=12), strict=True)
        x = torch.randn(2, 320, 16, 16, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    else:
        m = (CrossAttentionB200(query_dim=320, context_dim=768, num_heads=8, head_dim=40) if which == "cross_attention"
             else SpatialTransformerBlockB200(320, 8, 40, context_dim=768)).to(DEV)
        x = torch.randn(2, 256, 320, generator=g).to(DEV).to(torch.bfloat16)
    context = torch.randn(2, 77, 768, generator=g).to(DEV)
    call = (lambda inp, c: m(inp, context=c)) if which == "cross_attention" else (lambda inp, c: m(inp, c))
    return m, x, context, call


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["cross_attention", "block", "transformer"])
def test_backward_twice_with_retain_graph(which):
    m, x, context, call = _small_case(which)
    x = x.detach().requires_grad_(True)
    c = context.detach().requires_grad_(True)
    y = call(x, c)
    up = torch.randn(y.shape, generator=torch.Generator().manual_seed(13)).to(DEV).to(y.dtype)
    y.backward(up, retain_graph=True)
    first = {"x": x.grad.clone(), "c": c.grad.clone(), **{k: p.grad.clone() for k, p in m.named_parameters()}}
    y.backward(up)
    second = {"x": x.grad, "c": c.grad, **{k: p.grad for k, p in m.named_parameters()}}
    for k in first:  # the second pass adds the same gradients again (doubling is exact)
        assert torch.equal(second[k], 2 * first[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["cross_attention", "block"])
def test_in_place_change_of_the_input_is_detected(which):
    m, x, context, call = _small_case(which)
    leaf = x.detach().requires_grad_(True)
    inp = leaf * 1  # a non-leaf bf16 input, saved as is (no cast, no copy)
    y = call(inp, context)
    inp.add_(1)
    with pytest.raises(RuntimeError, match="inplace"):
        y.backward(torch.ones_like(y))


@pytest.mark.gpu
def test_bf16_parameters_and_layernorm_argument_checks():
    """After module.to(bfloat16) the LayerNorm parameters are bf16: the module hands the kernels fp32 copies, and the wrappers
    refuse anything but contiguous fp32 [dim] gamma / beta and [rows] mean / rstd."""
    m, x, context, call = _small_case("block")
    m = m.to(torch.bfloat16)
    x = x.detach().requires_grad_(True)
    call(x, context.to(torch.bfloat16)).float().sum().backward()
    assert torch.isfinite(x.grad.float()).all()
    assert m.norm1.weight.grad.dtype == torch.bfloat16 and torch.isfinite(m.norm1.weight.grad.float()).all()
    xs = rand_bf16(64, 320, seed=14)
    g32, b32 = torch.ones(320, device=DEV), torch.zeros(320, device=DEV)
    for bad in (g32.to(torch.bfloat16), torch.ones(321, device=DEV), torch.ones(640, device=DEV)[::2]):
        with pytest.raises(B200Error):
            ops.layernorm_bf16_fwd(xs, bad, b32, 1e-5)
    _, mean, rstd = ops.layernorm_bf16_fwd(xs, g32, b32, 1e-5)
    with pytest.raises(B200Error):
        ops.layernorm_bf16_bwd(xs, xs, g32, mean[:32], rstd)
    with pytest.raises(B200Error):
        ops.layernorm_bf16_bwd(xs, xs, g32, mean, rstd.to(torch.bfloat16))


# ---- 4. CPU: C-ABI argument checks, parameters, refusals ----------------------------------------------------------------------
def test_modules_match_reference_parameters():
    p, shapes, _ = _tiny_prefix_sd()
    C = shapes[0][1][0]
    ctx_dim = dict(shapes)["blocks.0.attn2.to_k.weight"][1]
    heads = 2
    m = SpatialTransformerB200(C, heads, C // heads, context_dim=ctx_dim)
    got = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    assert got == shapes
    assert all(v.dtype == torch.float32 for v in m.state_dict().values())
    sd = {k: torch.randn(s) for k, s in shapes}
    m.load_state_dict(sd, strict=True)
    back = SpatialTransformerB200(C, heads, C // heads, context_dim=ctx_dim)
    back.load_state_dict(m.state_dict(), strict=True)
    assert all(torch.equal(back.state_dict()[k], sd[k]) for k in sd)
    blk_shapes = [(k[len("blocks.0."):], s) for k, s in shapes if k.startswith("blocks.0.")]
    blk = SpatialTransformerBlockB200(C, heads, C // heads, context_dim=ctx_dim)
    assert [(k, tuple(v.shape)) for k, v in blk.state_dict().items()] == blk_shapes
    blk.load_state_dict({k: sd["blocks.0." + k] for k, _ in blk_shapes}, strict=True)


def test_modules_refuse_unsupported_configurations():
    with pytest.raises(NotImplementedError):
        SpatialTransformerBlockB200(64, 8, 8, dropout=0.1)
    with pytest.raises(NotImplementedError):
        SpatialTransformerBlockB200(64, 8, 8, hooks_kwargs={})
    with pytest.raises(NotImplementedError):
        SpatialTransformerBlockB200(64, 8, 8, feedforward_activation="GELU")
    with pytest.raises(NotImplementedError):
        SpatialTransformerBlockB200(64, 8, 8, feedforward_multiplier=1.1)  # F = 70
    with pytest.raises(NotImplementedError):
        SpatialTransformerB200(64, 8, 8, use_linear=True)
    with pytest.raises(NotImplementedError):
        SpatialTransformerB200(64, 8, 8, dropout=0.1)
    with pytest.raises(NotImplementedError):
        SpatialTransformerB200(64, 8, 8, hooks_kwargs={"tome_info": {}})
    SpatialTransformerB200(64, 8, 8, use_checkpoint=True)  # accepted: memory only
    m = SpatialTransformerB200(64, 8, 8, context_dim=32)
    with pytest.raises(B200Error):
        m(torch.zeros(1, 64, 4, 4, dtype=torch.bfloat16), torch.zeros(1, 7, 32))
    blk = SpatialTransformerBlockB200(64, 8, 8)
    with pytest.raises(B200Error):
        blk(torch.zeros(1, 16, 64, dtype=torch.bfloat16))
    if torch.cuda.is_available():
        with pytest.raises(B200Error):
            m(torch.zeros(1, 64, 4, 4, device=DEV), torch.zeros(1, 7, 32, device=DEV))
