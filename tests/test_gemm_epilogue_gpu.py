"""GPU tests of the GEMM's epilogue warps: the MMA warpgroups hand t = bf16(acc + bias) over through a shared-memory staging
tile and the epilogue warps finish it (GELU, residual, dGELU, edges).  Checks that results do not depend on how tiles are
spread over CTAs (the staging phases wrap many times on one CTA), the M / N edges, and that the epilogue variants agree
with each other bit for bit."""
import pytest
import torch
import torch.nn.functional as F

import cflearn_b200  # noqa: F401  (registers the package)
from cflearn_b200 import ops
from _refs import rand_bf16

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _padded(M, N, dtype):
    """[M, N] view of a buffer whose rows are padded to 16 bytes (the layout ops.gemm allocates)."""
    npad = (N + 7) // 8 * 8
    return torch.empty(M, npad, device=DEV, dtype=dtype)[:, :N]


def _gelu_pair(a, b, bias, M, N, max_ctas=0, epilogue=ops.EPI_BIAS_GELU_BF16):
    g = _padded(M, N, torch.bfloat16)
    h = ops.gemm(a, b, bias=bias, epilogue=epilogue, out1=g, max_ctas=max_ctas)
    return h, g


@pytest.mark.parametrize("epilogue", [ops.EPI_BIAS_BF16, ops.EPI_BIAS_GELU_BF16, ops.EPI_BIAS_RESID_F32])
def test_result_independent_of_cta_count(epilogue):
    # 4096 x 2048: 256 tiles; one CTA runs all of them, so the staging tile's full / empty phases wrap 256 times
    M, N, K = 4096, 2048, 256
    a, b, bias = rand_bf16(M, K, seed=1), rand_bf16(N, K, scale=0.5, seed=2), rand_bf16(N, seed=3)
    res = torch.randn(M, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    outs = []
    for ctas in (0, 5, 1):
        kw = dict(bias=bias, epilogue=epilogue, max_ctas=ctas)
        if epilogue == ops.EPI_BIAS_GELU_BF16:
            kw["out1"] = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
        if epilogue == ops.EPI_BIAS_RESID_F32:
            kw["aux"] = res
        out = ops.gemm(a, b, **kw)
        outs.append((out, kw.get("out1")))
    torch.cuda.synchronize()
    for out, g in outs[1:]:
        assert torch.equal(out, outs[0][0])
        if g is not None:
            assert torch.equal(g, outs[0][1])
    term = (a.float() @ b.float().t() + bias.float()).to(torch.bfloat16).float()
    got = outs[0][0] - res if epilogue == ops.EPI_BIAS_RESID_F32 else outs[0][0].float()
    # up to one-ulp flips of the bf16 term, measured against the term (a residual may cancel it)
    assert ((got - term).abs() > 0.02 * term.abs().clamp_min(1.0)).sum().item() == 0


@pytest.mark.parametrize("M,N,K", [(300, 1003, 192), (129, 257, 64), (1000, 13, 128), (77, 3072, 768)])
def test_edges_and_cross_epilogue_consistency(M, N, K):
    """M / N edges (N not a multiple of 8 included); h of the GELU epilogue == the bias epilogue; the residual epilogue ==
    aux + float(bias epilogue), in place or not; dGELU == dGELU(h) applied to the plain GEMM, all bit for bit."""
    a, b, bias = rand_bf16(M, K, seed=11), rand_bf16(N, K, scale=0.5, seed=12), rand_bf16(N, seed=13)
    t = ops.gemm(a, b, bias=bias)
    torch.cuda.synchronize()
    ref = (a.float() @ b.float().t() + bias.float()).to(torch.bfloat16)
    assert ((t.float() - ref.float()).abs() > 0.02 * ref.float().abs().clamp_min(1.0)).sum().item() == 0

    h, g = _gelu_pair(a, b, bias, M, N)
    assert torch.equal(h, t)
    assert ((g.float() - F.gelu(t.float())).abs() > 0.01 * g.float().abs().clamp_min(0.1)).sum().item() == 0
    hq, gq = _gelu_pair(a, b, bias, M, N, epilogue=ops.EPI_BIAS_QGELU_BF16)
    assert torch.equal(hq, t)

    res = _padded(M, N, torch.float32)
    res.copy_(torch.randn(M, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(14)))
    expect = res + t.float()
    out = ops.gemm(a, b, bias=bias, epilogue=ops.EPI_BIAS_RESID_F32, aux=res)
    assert torch.equal(out, expect)
    inplace = res.clone()  # clone of a strided view: give it the padded layout again
    buf = _padded(M, N, torch.float32)
    buf.copy_(inplace)
    ops.gemm(a, b, bias=bias, epilogue=ops.EPI_BIAS_RESID_F32, out0=buf, aux=buf)
    assert torch.equal(buf, expect)

    # dGELU: dG[M, N] = dY[M, K] . W[K, N] (MN-major B) times gelu'(h); the plain GEMM of the same operands gives bf16(acc)
    w = _padded(K, N, torch.bfloat16)  # TMA needs 16-byte row strides
    w.copy_(rand_bf16(K, N, scale=0.05, seed=15))
    hh = _padded(M, N, torch.bfloat16)
    hh.copy_(rand_bf16(M, N, seed=16))
    dacc = ops.gemm(a, w, b_mn_major=True)
    dg = ops.gemm(a, w, b_mn_major=True, epilogue=ops.EPI_DGELU_BF16, aux=hh)
    torch.cuda.synchronize()
    hf = hh.float().requires_grad_(True)
    F.gelu(hf).backward(dacc.float())
    ref_dg = hf.grad
    bad = (dg.float() - ref_dg).abs() > 2 * 2.0 ** -7 * ref_dg.abs() + 1e-3 * ref_dg.abs().max()
    assert bad.sum().item() == 0


def test_conv3x3_through_epilogue_warps():
    B, H, W, Cin, Cout = 2, 16, 16, 64, 200
    x = rand_bf16(B, H, W, Cin, seed=21)
    w = rand_bf16(Cout, Cin, 3, 3, scale=0.05, seed=22)
    bias = rand_bf16(Cout, seed=23)
    wp = ops.pack_conv3x3_weight(w)
    y = ops.conv3x3(x, wp, bias)
    res = torch.randn(B, H, W, Cout, device=DEV, generator=torch.Generator(device=DEV).manual_seed(24))
    yr = ops.conv3x3(x, wp, bias, epilogue=ops.EPI_BIAS_RESID_F32, aux=res)
    torch.cuda.synchronize()
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias.float(), padding=1).permute(0, 2, 3, 1)
    refb = ref.to(torch.bfloat16)
    assert ((y.float() - refb.float()).abs() > 0.02 * refb.float().abs().clamp_min(1.0)).sum().item() == 0
    assert torch.equal(yr, res + y.float())
