"""GPU parity tests of every C-ABI kernel against plain PyTorch references of the same op (fp32 math, bf16 rounding at the same
points the reference's autocast path rounds) and the float64 references of _refs.py.  Run on an H100: pytest -m gpu."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

import cflearn_b200  # noqa: F401,E402  (registers the package)
from cflearn_b200 import ops
from _refs import assert_bf16_close, assert_ulp, packed_attention, rand_bf16, relerr, with_grads

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ------------------------------------------------------------------------------------------------------------
# row kernels
# ------------------------------------------------------------------------------------------------------------
def test_cast_and_fill():
    x = torch.randn(1000003, device=DEV)
    y = ops.cast_bf16(x)
    assert torch.equal(y, x.to(torch.bfloat16))
    z = torch.empty(12345, device=DEV)
    ops.fill_f32(z, 2.5)
    assert torch.equal(z, torch.full_like(z, 2.5))


@pytest.mark.parametrize("rows,dim", [(50432 // 8, 768), (1000, 512), (77, 1024), (5, 256)])
def test_layernorm_fwd(rows, dim):
    torch.manual_seed(0)
    x = torch.randn(rows, dim, device=DEV) * 2 + 0.5
    g = torch.randn(dim, device=DEV)
    b = torch.randn(dim, device=DEV)
    y, mean, rstd = ops.layernorm_fwd(x, g, b, 1e-6, rows=rows, dim=dim, ld_x=dim)
    ref = F.layer_norm(x, (dim,), g, b, 1e-6)
    assert_bf16_close(y, ref, "layernorm_fwd")
    assert torch.allclose(mean, x.mean(-1), atol=1e-5)
    assert torch.allclose(rstd, (x.var(-1, unbiased=False) + 1e-6).rsqrt(), rtol=1e-4)


def test_layernorm_fwd_strided_head():
    # head LN reads only token 0 of every image (row stride = T * D)
    B, T, D = 16, 197, 768
    net = torch.randn(B, T, D, device=DEV)
    g = torch.randn(D, device=DEV)
    b = torch.randn(D, device=DEV)
    y, _, _ = ops.layernorm_fwd(net, g, b, 1e-6, rows=B, dim=D, ld_x=T * D)
    assert_bf16_close(y, F.layer_norm(net[:, 0], (D,), g, b, 1e-6), "layernorm_fwd strided")


@pytest.mark.parametrize("rows,dim,with_res", [(4096, 768, True), (333, 512, False), (50, 1024, True)])
def test_layernorm_bwd(rows, dim, with_res):
    torch.manual_seed(1)
    x = (torch.randn(rows, dim, device=DEV) * 1.5 + 0.3).requires_grad_(True)
    g = torch.randn(dim, device=DEV, requires_grad=True)
    b = torch.randn(dim, device=DEV, requires_grad=True)
    dy = torch.randn(rows, dim, device=DEV).to(torch.bfloat16)
    dres = torch.randn(rows, dim, device=DEV) if with_res else None
    y = F.layer_norm(x, (dim,), g, b, 1e-6)
    y.backward(dy.float())
    _, mean, rstd = ops.layernorm_fwd(x.detach(), g.detach(), b.detach(), 1e-6, rows=rows, dim=dim, ld_x=dim)
    dx = torch.empty(rows, dim, device=DEV)
    dxb = torch.empty(rows, dim, device=DEV, dtype=torch.bfloat16)
    dg = torch.empty(dim, device=DEV)
    db = torch.empty(dim, device=DEV)
    ops.layernorm_bwd(dy, x.detach(), g.detach(), mean, rstd, rows=rows, dim=dim, ld_x=dim, dres=dres, dx_out=dx,
                      ld_dx=dim, dx_bf16=dxb, dgamma=dg, dbeta=db)
    ref_dx = x.grad + (dres if with_res else 0)
    assert relerr(dx, ref_dx) < 1e-5
    assert torch.equal(dxb, dx.to(torch.bfloat16))
    assert relerr(dg, g.grad) < 1e-5
    assert relerr(db, b.grad) < 1e-5
    # fused bias gradient: bf16-rounded column sums of the bf16 dx (what a separate colsum pass over dx_bf16 returns)
    dxs = torch.full((dim,), 7.0, device=DEV)
    dxb2 = torch.empty_like(dxb)
    dg2, db2 = torch.empty_like(dg), torch.empty_like(db)
    ops.layernorm_bwd(dy, x.detach(), g.detach(), mean, rstd, rows=rows, dim=dim, ld_x=dim, dres=dres, dx_out=dx,
                      ld_dx=dim, dx_bf16=dxb2, dgamma=dg2, dbeta=db2, dx_colsum=dxs)
    assert torch.equal(dxb2, dxb)
    assert relerr(dg2, g.grad) < 1e-5 and relerr(db2, b.grad) < 1e-5
    ref = dxb.double().sum(0)
    assert (dxs.double() - ref).abs().max().item() <= 2.0 ** -8 * ref.abs().max().item() + 1e-6
    assert torch.equal(dxs, dxs.to(torch.bfloat16).float())


@pytest.mark.parametrize("rows,cols", [(50432 // 4, 2304), (1000, 768), (256, 1000), (7, 3072)])
def test_colsum(rows, cols):
    x = rand_bf16(rows, cols, seed=3)
    out = torch.empty(cols, device=DEV)
    ops.colsum(x, out, round_bf16=False)
    assert relerr(out, x.float().sum(0)) < 1e-5
    ops.colsum(x, out, round_bf16=True, accumulate=True)
    ref = x.float().sum(0) + x.float().sum(0).to(torch.bfloat16).float()
    assert relerr(out, ref) < 1e-3


def test_patch_glue():
    B, C, S, P, D = 4, 3, 224, 16, 768
    torch.manual_seed(0)
    x = torch.randn(B, C, S, S, device=DEV)
    cols = ops.patch_im2col(x, P)
    ref = F.unfold(x, kernel_size=P, stride=P).transpose(1, 2).reshape(B * 196, C * P * P)
    assert torch.equal(cols, ref.to(torch.bfloat16))
    patch = rand_bf16(B * 196, D, seed=4)
    cls = torch.randn(1, 1, D, device=DEV)
    pos = torch.randn(1, 197, D, device=DEV)
    net = ops.assemble_tokens(patch, cls, pos, B, 196, D)
    ref_net = torch.cat([cls.expand(B, 1, D), patch.view(B, 196, D).float()], 1) + pos
    assert torch.equal(net, ref_net)
    dnet = torch.randn(B, 197, D, device=DEV)
    dpos = torch.empty(197, D, device=DEV)
    dcls = torch.empty(D, device=DEV)
    dpatch = ops.assemble_tokens_bwd(dnet, dpos, dcls, B, 196, D)
    assert torch.equal(dpatch, dnet[:, 1:].reshape(B * 196, D).to(torch.bfloat16))
    assert relerr(dpos, dnet.sum(0)) < 1e-6
    assert relerr(dcls, dnet[:, 0].sum(0)) < 1e-6


def test_patch_im2col_p32():
    x = torch.randn(2, 3, 224, 224, device=DEV)
    cols = ops.patch_im2col(x, 32)
    ref = F.unfold(x, kernel_size=32, stride=32).transpose(1, 2).reshape(2 * 49, 3 * 32 * 32)
    assert torch.equal(cols, ref.to(torch.bfloat16))


@pytest.mark.parametrize("B,C", [(256, 1000), (32, 10), (3, 50000)])
def test_softmax_xent(B, C):
    torch.manual_seed(2)
    logits = (torch.randn(B, C, device=DEV) * 3).to(torch.bfloat16)
    labels = torch.randint(0, C, (B,), device=DEV)
    loss_mean, loss_rows, dlogits, bad = ops.softmax_xent(logits, labels)
    lf = logits.float().requires_grad_(True)
    ref_rows = -F.log_softmax(lf, dim=1).gather(1, labels[:, None])[:, 0]
    ref_rows.mean().backward()
    assert bad.item() == 0
    assert torch.allclose(loss_rows, ref_rows, rtol=1e-5, atol=1e-5)
    assert abs(loss_mean.item() - ref_rows.mean().item()) < 1e-5 * max(1.0, abs(ref_rows.mean().item()))
    assert_bf16_close(dlogits, lf.grad, "dlogits")
    # integer label path is exact: the gathered logit equals logits[row, label] bit for bit
    picked = logits.gather(1, labels[:, None])[:, 0].float()
    lse = torch.logsumexp(logits.float(), 1)
    assert torch.allclose(loss_rows, lse - picked, rtol=1e-5, atol=1e-5)


def test_softmax_xent_bad_label_is_flagged():
    logits = torch.zeros(4, 8, device=DEV, dtype=torch.bfloat16)
    labels = torch.tensor([0, 9, 2, -1], device=DEV)
    _, _, _, bad = ops.softmax_xent(logits, labels)
    assert bad.item() == 1


# ------------------------------------------------------------------------------------------------------------
# wgmma GEMM
# ------------------------------------------------------------------------------------------------------------
GEMM_SHAPES = [(128, 256, 64), (256, 256, 128), (384, 512, 192), (300, 264, 200), (2048, 768, 768), (256, 1000, 768)]


def _operands(M, N, K, a_mn, b_mn, seed=0):
    a = rand_bf16(M, K, seed=seed)
    b = rand_bf16(N, K, scale=0.5, seed=seed + 1)
    a_arg = a.t().contiguous() if a_mn else a
    b_arg = b.t().contiguous() if b_mn else b
    return a, b, a_arg, b_arg


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_kmajor_bias(M, N, K):
    a, b, a_arg, b_arg = _operands(M, N, K, False, False)
    bias = rand_bf16(N, seed=7)
    out = ops.gemm(a_arg, b_arg, bias=bias)
    torch.cuda.synchronize()
    ref = a.float() @ b.float().t() + bias.float()
    assert_bf16_close(out, ref, f"gemm {M}x{N}x{K}")


# (1152, 768, 512) and (200, 520, 136): even and odd (3, 2) numbers of m tiles, every pair of majors
GEMM_MAJOR_CASES = ([(M, N, K, a, b) for M, N, K in [(256, 256, 128), (384, 512, 192), (328, 264, 200), (768, 768, 4096)]
                     for a, b in [(False, True), (True, False), (True, True)]]
                    + [(M, N, K, a, b) for M, N, K in [(1152, 768, 512), (200, 520, 136)] for a, b in [(False, False), (False, True), (True, True)]])


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", GEMM_MAJOR_CASES)
def test_gemm_mn_major(M, N, K, a_mn, b_mn):
    a, b, a_arg, b_arg = _operands(M, N, K, a_mn, b_mn, seed=11)
    out = ops.gemm(a_arg, b_arg, a_mn_major=a_mn, b_mn_major=b_mn)
    torch.cuda.synchronize()
    assert_bf16_close(out, a.float() @ b.float().t(), f"gemm mn-major a={a_mn} b={b_mn} {M}x{N}x{K}")


def test_gemm_persistent_many_tiles():
    # 8192 x 2304 x 768: 576 tiles over 132 CTAs -> several tiles per CTA, the smem ring phases wrap
    M, N, K = 8192, 2304, 768
    a, b, a_arg, b_arg = _operands(M, N, K, False, False, seed=21)
    bias = rand_bf16(N, seed=22)
    out = ops.gemm(a_arg, b_arg, bias=bias)
    torch.cuda.synchronize()
    assert_bf16_close(out, a.float() @ b.float().t() + bias.float(), "gemm persistent")
    out2 = ops.gemm(a_arg, b_arg, bias=bias, max_ctas=5)
    assert torch.equal(out, out2), "result must not depend on the number of CTAs"


def test_gemm_gelu_epilogue():
    M, N, K = 1024, 3072, 768
    a, b, a_arg, b_arg = _operands(M, N, K, False, False, seed=31)
    bias = rand_bf16(N, seed=32)
    g = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    h = ops.gemm(a_arg, b_arg, bias=bias, epilogue=ops.EPI_BIAS_GELU_BF16, out1=g)
    torch.cuda.synchronize()
    ref_h = (a.float() @ b.float().t() + bias.float())
    assert_bf16_close(h, ref_h, "gelu epilogue: h")
    ref_g = F.gelu(h.float())  # GELU of the ROUNDED pre-activation, evaluated in fp32, like ATen on bf16
    assert_bf16_close(g, ref_g, "gelu epilogue: gelu(h)")


@pytest.mark.parametrize("inplace", [True, False])
def test_gemm_residual_epilogue(inplace):
    M, N, K = 1024, 768, 3072
    a, b, a_arg, b_arg = _operands(M, N, K, False, False, seed=41)
    bias = rand_bf16(N, seed=42)
    res = torch.randn(M, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(43))
    term = (a.float() @ b.float().t() + bias.float()).to(torch.bfloat16).float()
    ref = res + term
    if inplace:
        out = res.clone()
        ops.gemm(a_arg, b_arg, bias=bias, epilogue=ops.EPI_BIAS_RESID_F32, out0=out, aux=out)
    else:
        out = ops.gemm(a_arg, b_arg, bias=bias, epilogue=ops.EPI_BIAS_RESID_F32, aux=res)
    torch.cuda.synchronize()
    err = (out - ref).abs()
    # identical up to bf16 rounding flips of the matmul term (one ulp of THAT term: the residual may cancel it, so the
    # bound must not be relative to the sum -- an unseeded residual made this fail about one run in thirty)
    assert (err > 0.02 * term.abs().clamp_min(1.0)).float().mean().item() == 0.0
    assert relerr(out, ref) < 1e-3


def test_gemm_dgelu_epilogue():
    M, N, K = 512, 3072, 768  # dG[M, 3072] = dY[M, 768] . W2[768, 3072] ; W2 is MN-major B
    dy = rand_bf16(M, K, seed=51)
    w2 = rand_bf16(K, N, scale=0.05, seed=52)  # [768, 3072] row-major == reference layout [out=768, in=3072]
    h = rand_bf16(M, N, seed=53)
    out = ops.gemm(dy, w2, b_mn_major=True, epilogue=ops.EPI_DGELU_BF16, aux=h)
    torch.cuda.synchronize()
    dg = (dy.float() @ w2.float()).to(torch.bfloat16)
    hf = h.float().requires_grad_(True)
    F.gelu(hf).backward(dg.float())
    assert_bf16_close(out, hf.grad, "dgelu epilogue", max_ulps=2.01)


@pytest.mark.parametrize("n_out,k_in,M", [(768, 768, 4096), (2304, 768, 2048), (1000, 768, 256), (768, 3072, 1024)])
def test_wgrad_splitk(n_out, k_in, M):
    dy = rand_bf16(M, n_out, seed=61)
    x = rand_bf16(M, k_in, seed=62)
    out = torch.empty(n_out, k_in, device=DEV)
    ops.wgrad(dy, x, out, round_bf16=False)
    torch.cuda.synchronize()
    ref = dy.float().t() @ x.float()
    assert relerr(out, ref) < 1e-5
    ops.wgrad(dy, x, out, round_bf16=True)
    # bf16 rounding of two fp32 sums that differ in the last bits may flip: rarely the other neighbour, never further
    assert (out != ref.to(torch.bfloat16).float()).float().mean().item() < 1e-3
    assert_ulp(out, ref, "wgrad rounded", floor=1e-5)


# ------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,T,H,causal", [(2, 197, 12, False), (3, 77, 8, True), (2, 50, 12, False), (1, 256, 2, False), (2, 128, 1, True)])
def test_attention_fwd(B, T, H, causal):
    _attention_fwd_case(B, T, H, causal)


def test_attention_fwd_many_items_per_cta():
    """More (batch, head) items than SMs: several waves of CTAs (the small cases above fit in one)."""
    _attention_fwd_case(40, 197, 12, False)
    _attention_fwd_case(64, 77, 8, True)
    _attention_fwd_case(37, 50, 12, False)


def _attention_fwd_case(B, T, H, causal):
    qkv = rand_bf16(B * T, 3 * H * 64, seed=71)
    out, lse = ops.attention_fwd(qkv, B, T, H, causal=causal)
    torch.cuda.synchronize()
    ref_o, ref_lse = packed_attention(qkv, B, T, H, causal=causal)
    assert relerr(out, ref_o) < 5e-3, relerr(out, ref_o)
    assert torch.allclose(lse.double(), ref_lse, rtol=1e-4, atol=1e-4)
    # and against the kernel the reference itself dispatches to (toolkit.py:959-963)
    q, k, v = qkv.view(B, T, 3, H, 64).permute(2, 0, 3, 1, 4)
    sdpa = F.scaled_dot_product_attention(q, k, v, is_causal=causal).permute(0, 2, 1, 3).reshape(B * T, H * 64)
    assert relerr(out, sdpa) < 5e-3


@pytest.mark.parametrize("B,T,H,causal", [(2, 197, 12, False), (3, 77, 8, True), (2, 50, 12, False), (1, 256, 2, False), (2, 130, 2, False), (2, 16, 1, True)])
def test_attention_bwd(B, T, H, causal):
    _attention_bwd_case(B, T, H, causal)


def test_attention_bwd_many_items_per_cta():
    """More (batch, head) items than SMs: several waves of CTAs, odd and even numbers of 64-row tiles per item."""
    _attention_bwd_case(40, 197, 12, False)
    _attention_bwd_case(64, 77, 8, True)
    _attention_bwd_case(37, 50, 12, False)
    _attention_bwd_case(30, 130, 6, False)
    _attention_bwd_case(33, 256, 5, True)


def _attention_bwd_case(B, T, H, causal):
    D = H * 64
    qkv = rand_bf16(B * T, 3 * D, seed=81)
    dout = rand_bf16(B * T, D, seed=82)
    out, lse = ops.attention_fwd(qkv, B, T, H, causal=causal)
    dqkv = ops.attention_bwd(qkv, out, dout, lse, B, T, H, causal=causal)
    torch.cuda.synchronize()
    _, (ref,) = with_grads(packed_attention, (qkv,), dout, B, T, H, 0.125, causal)
    for name, sl in (("dq", slice(0, D)), ("dk", slice(D, 2 * D)), ("dv", slice(2 * D, 3 * D))):
        e = relerr(dqkv[:, sl], ref[:, sl])
        assert e < 1e-2, f"{name}: {e}"
    # eager bf16 SDPA backward as a second opinion
    q2 = qkv.clone().requires_grad_(True)
    q, k, v = q2.view(B, T, 3, H, 64).permute(2, 0, 3, 1, 4)
    o2 = F.scaled_dot_product_attention(q, k, v, is_causal=causal).permute(0, 2, 1, 3).reshape(B * T, D)
    o2.backward(dout)
    assert relerr(dqkv, q2.grad) < 1.5e-2
    # fused qkv-bias gradient: bf16-rounded column sums of the dqkv just written
    dbias = torch.full((3 * D,), 3.0, device=DEV)
    dqkv2 = ops.attention_bwd(qkv, out, dout, lse, B, T, H, causal=causal, dbias=dbias)
    assert torch.equal(dqkv2, dqkv)
    ref_b = dqkv.double().sum(0)
    assert (dbias.double() - ref_b).abs().max().item() <= 2.0 ** -8 * ref_b.abs().max().item() + 1e-6
    assert torch.equal(dbias, dbias.to(torch.bfloat16).float())


def test_gemm_quick_gelu_epilogues_follow_eager_rounding():
    """QuickGELU (CLIP towers): forward and backward must reproduce eager's op-by-op bf16 rounding
    (``net * torch.sigmoid(1.702 * net)`` is three elementwise kernels on a bf16 tensor)."""
    M, N, K = 1024, 1024, 256
    a, b, a_arg, b_arg = _operands(M, N, K, False, False, seed=61)
    bias = rand_bf16(N, seed=62)
    g = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    h = ops.gemm(a_arg, b_arg, bias=bias, epilogue=ops.EPI_BIAS_QGELU_BF16, out1=g)
    torch.cuda.synchronize()
    assert_bf16_close(h, a.float() @ b.float().t() + bias.float(), "quick-gelu epilogue: h")
    hh = h.clone().requires_grad_(True)
    ref = hh * torch.sigmoid(1.702 * hh)  # eager, bf16 tensors
    fl = (g != ref.detach()).float().mean().item()
    assert fl < 2e-3, f"forward flips {fl}"  # identical up to ulp flips of the approximate sigmoid
    assert_bf16_close(g, ref.detach().float(), "quick-gelu epilogue: act")
    # backward: dh = autograd of the three bf16 ops; dY . W with W MN-major as in the FF2 dgrad
    dy = rand_bf16(M, K, seed=63)
    w2 = rand_bf16(K, N, seed=64)
    dact = ops.gemm(dy, w2, b_mn_major=True)  # bf16(acc) exactly as the fused kernel sees it (same main loop)
    assert_bf16_close(dact, dy.float() @ w2.float(), "quick-gelu backward: dact")
    ref.backward(dact)
    dh = ops.gemm(dy, w2, b_mn_major=True, epilogue=ops.EPI_DQGELU_BF16, aux=h)
    torch.cuda.synchronize()
    fl = (dh != hh.grad).float().mean().item()
    big = ((dh.float() - hh.grad.float()).abs() > 0.02 * hh.grad.float().abs().clamp_min(1e-3)).float().mean().item()
    # same rounding points as autograd's CUDA kernels (incl. the per-operator bf16 rounding inside sigmoid_backward);
    # what is left are flips from the approximate sigmoid propagating through the five roundings
    assert fl < 1e-2 and big < 1e-3, f"backward flips {fl}, beyond one ulp {big}"
    assert_bf16_close(dh, hh.grad.float(), "quick-gelu backward epilogue")


@pytest.mark.parametrize("rows,dim", [(1000, 768), (77, 512)])
def test_layernorm_bwd_fp32_upstream(rows, dim):
    """LayerNorm whose output is the fp32 residual stream (CLIP's embedding_norm): dy arrives in fp32."""
    torch.manual_seed(3)
    x = (torch.randn(rows, dim, device=DEV) * 1.3 - 0.2).requires_grad_(True)
    g = torch.randn(dim, device=DEV, requires_grad=True)
    b = torch.randn(dim, device=DEV, requires_grad=True)
    dy = torch.randn(rows, dim, device=DEV)
    F.layer_norm(x, (dim,), g, b, 1e-5).backward(dy)
    _, mean, rstd = ops.layernorm_fwd(x.detach(), g.detach(), b.detach(), 1e-5, rows=rows, dim=dim, ld_x=dim)
    dx, dg, db = torch.empty(rows, dim, device=DEV), torch.empty(dim, device=DEV), torch.empty(dim, device=DEV)
    ops.layernorm_bwd(dy, x.detach(), g.detach(), mean, rstd, rows=rows, dim=dim, ld_x=dim, dres=None, dx_out=dx, ld_dx=dim,
                      dx_bf16=None, dgamma=dg, dbeta=db)
    assert relerr(dx, x.grad) < 1e-5 and relerr(dg, g.grad) < 1e-5 and relerr(db, b.grad) < 1e-5


@pytest.mark.parametrize("B", [5, 64, 256])
def test_symmetric_xent_matches_fp32_reference(B):
    """CLIP's contrastive loss kernel: (CE(L) + CE(L^T)) / 2 on bf16 logits, fp32 maths, ONE bf16 rounding of the gradient."""
    g = torch.Generator().manual_seed(123)
    ld = (B + 7) // 8 * 8
    logits = torch.zeros(B, ld, dtype=torch.bfloat16, device=DEV)[:, :B]
    logits.copy_((torch.randn(B, B, generator=g) * 4).to(DEV))
    dl = torch.zeros(B, ld, dtype=torch.bfloat16, device=DEV)[:, :B]
    loss = ops.symmetric_xent(logits, dlogits=dl)
    torch.cuda.synchronize()
    lf = logits.float().clone().requires_grad_(True)
    tgt = torch.arange(B, device=DEV)
    ref = 0.5 * (F.cross_entropy(lf, tgt) + F.cross_entropy(lf.t(), tgt))
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-5 * max(1.0, abs(ref.item()))
    assert_bf16_close(dl.contiguous(), lf.grad, "symmetric xent gradient")


@pytest.mark.parametrize("B,C,S,P,norm", [(3, 3, 224, 16, True), (2, 3, 224, 32, False), (2, 1, 64, 16, True), (2, 4, 32, 16, True)])
def test_patch_im2col_u8_fuses_the_input_pipeline_bit_exactly(B, C, S, P, norm):
    """SURVEY.md N4: raw uint8 HWC batch -> normalised bf16 im2col matrix in one kernel == the reference's host-side blocks
    (oracle/input_oracle.py: float64 normalise, hwc_to_chw, float32) followed by the fp32 im2col kernel.  Bit-exact: every
    rounding point (float64 -> float32 -> bf16) is reproduced and the rest is an integer-indexed copy."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import input_oracle as io

    g = torch.Generator().manual_seed(5)
    x = torch.randint(0, 256, (B, S, S, C), dtype=torch.uint8, generator=g)
    mean = [0.485, 0.456, 0.406, 0.5][:C] if norm else None
    std = [0.229, 0.224, 0.225, 0.25][:C] if norm else None
    ref = io.input_pipeline(x.numpy(), 255.0, mean, std).to(DEV)           # float32 [B, C, S, S], what the reference feeds the model
    want = ops.patch_im2col(ref.contiguous(), P)                           # (itself exact vs F.unfold: test_patch_glue)
    got = ops.patch_im2col_u8(x.to(DEV), P, 255.0, mean, std)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------------------
# SD-v1.5 UNet building blocks (SURVEY.md 8f row N3): GroupNorm(32) + SiLU on channels-last activations
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,C,silu,eps", [(2, 64, 64, 320, True, 1e-5), (2, 8, 8, 1280, True, 1e-5), (2, 16, 16, 2560, True, 1e-5),
                                              (3, 32, 32, 640, False, 1e-6), (1, 16, 16, 960, True, 1e-5)])
def test_groupnorm_silu_fwd_bwd_matches_eager_autocast(B, H, W, C, silu, eps):
    """Real SD-v1.5 shapes (320 ch @ 64x64, 1280 ch @ 8x8, the 2560-channel skip concatenation, the SpatialTransformer's plain
    GroupNorm).  Reference = what eager does under bf16 autocast (oracle/unet_oracle.py::res_block): F.group_norm in fp32 on
    the bf16 activation, F.silu in fp32, ONE bf16 cast at the conv input; backward through the same graph."""
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(B, C, H, W, generator=g) * 1.5 + 0.3).to(DEV).to(torch.bfloat16)        # NCHW, as the reference holds it
    gamma = (1.0 + 0.1 * torch.randn(C, generator=g)).to(DEV)
    beta = (0.05 * torch.randn(C, generator=g)).to(DEV)
    dy = torch.randn(B, C, H, W, generator=g).to(DEV).to(torch.bfloat16)
    xr = x.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    z = F.group_norm(xr.float(), 32, gr, br, eps)
    ref = (F.silu(z) if silu else z)
    ref_bf16 = ref.to(torch.bfloat16)
    ref_bf16.backward(dy)
    # channels-last views for the kernel
    nhwc = lambda t: t.permute(0, 2, 3, 1).reshape(B, H * W, C).contiguous()  # noqa: E731
    y, mean, rstd = ops.groupnorm_silu_fwd(nhwc(x), gamma, beta, eps, silu=silu)
    dx, dgamma, dbeta = ops.groupnorm_silu_bwd(nhwc(x), nhwc(dy), gamma, beta, mean, rstd, silu=silu)
    torch.cuda.synchronize()
    assert_bf16_close(y, nhwc(ref.detach()), "groupnorm+silu forward")
    xs = x.float().view(B, 32, -1)
    assert torch.allclose(mean, xs.mean(-1), rtol=1e-4, atol=1e-5)
    assert torch.allclose(rstd, (xs.var(-1, unbiased=False) + eps).rsqrt(), rtol=1e-4, atol=1e-5)
    assert_bf16_close(dx, nhwc(xr.grad.float()), "groupnorm+silu backward dx")
    assert relerr(dgamma, gr.grad) < 1e-4 and relerr(dbeta, br.grad) < 1e-4
    # deterministic: a second run is bit-identical
    y2, _, _ = ops.groupnorm_silu_fwd(nhwc(x), gamma, beta, eps, silu=silu)
    dx2, dg2, db2 = ops.groupnorm_silu_bwd(nhwc(x), nhwc(dy), gamma, beta, mean, rstd, silu=silu)
    assert torch.equal(y, y2) and torch.equal(dx, dx2) and torch.equal(dgamma, dg2) and torch.equal(dbeta, db2)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 64, 64, 320, 320), (2, 8, 8, 1280, 1280), (3, 8, 8, 1280, 640), (2, 32, 32, 640, 320),
                                            (1, 16, 16, 2560, 1280), (2, 16, 16, 64, 8)])
def test_conv3x3_implicit_gemm_matches_conv2d(B, H, W, Cin, Cout):
    """3x3 / stride 1 / zero padding 1 convolution on channels-last bf16 activations as an implicit GEMM (no im2col matrix; the
    halo is the TMA unit's out-of-bound zero fill) at real SD-v1.5 shapes, forward and input gradient, against F.conv2d in fp32
    on the same bf16 operands, rounded to bf16 at the same point (the conv output under autocast)."""
    g = torch.Generator().manual_seed(21)
    x = torch.randn(B, Cin, H, W, generator=g).to(DEV).to(torch.bfloat16)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (0.7 / math.sqrt(9 * Cin))).to(DEV).to(torch.bfloat16)
    bias = (0.1 * torch.randn(Cout, generator=g)).to(DEV).to(torch.bfloat16)
    ref = F.conv2d(x.float(), w.float(), bias.float(), padding=1)                                 # fp32 reference, NCHW
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    out = ops.conv3x3(x_nhwc, ops.pack_conv3x3_weight(w), bias)
    torch.cuda.synchronize()
    assert tuple(out.shape) == (B, H, W, Cout)
    assert_bf16_close(out.reshape(-1, Cout), ref.permute(0, 2, 3, 1).reshape(-1, Cout), "conv3x3 forward")
    # residual epilogue: fp32 stream + bf16(conv)
    res = torch.randn(B, H, W, Cout, generator=g).to(DEV)
    out_r = ops.conv3x3(x_nhwc, ops.pack_conv3x3_weight(w), bias, epilogue=ops.EPI_BIAS_RESID_F32, aux=res)
    assert torch.allclose(out_r, res + out.float(), rtol=0, atol=0)
    # input gradient = the same kernel with flipped / transposed weights
    if Cout % 64 == 0:
        dy = torch.randn(B, Cout, H, W, generator=g).to(DEV).to(torch.bfloat16)
        xr = x.float().clone().requires_grad_(True)
        F.conv2d(xr, w.float(), None, padding=1).backward(dy.float())
        dx = ops.conv3x3(dy.permute(0, 2, 3, 1).contiguous(), ops.pack_conv3x3_weight_dgrad(w))
        torch.cuda.synchronize()
        assert_bf16_close(dx.reshape(-1, Cin), xr.grad.permute(0, 2, 3, 1).reshape(-1, Cin), "conv3x3 input gradient")


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 64, 64, 320, 320), (2, 8, 8, 1280, 1280), (3, 8, 8, 1280, 640), (2, 32, 32, 640, 320),
                                            (1, 16, 16, 2560, 1280), (2, 16, 16, 64, 8)])
def test_conv3x3_weight_gradient_matches_conv2d(B, H, W, Cin, Cout):
    """dW of the 3x3 convolution as ONE split-K implicit GEMM over the pixels (dy MN-major, the activation behind a 4-D tensor map,
    every 64-channel box shifted by its own tap) against autograd of F.conv2d in fp32 on the same bf16 operands."""
    g = torch.Generator().manual_seed(23)
    x = torch.randn(B, Cin, H, W, generator=g).to(DEV).to(torch.bfloat16)
    dy = torch.randn(B, Cout, H, W, generator=g).to(DEV).to(torch.bfloat16)
    w = torch.zeros(Cout, Cin, 3, 3, device=DEV, requires_grad=True)
    F.conv2d(x.float(), w, None, padding=1).backward(dy.float())
    dw = ops.conv3x3_wgrad(dy.permute(0, 2, 3, 1).contiguous(), x.permute(0, 2, 3, 1).contiguous(), round_bf16=False)
    torch.cuda.synchronize()
    assert tuple(dw.shape) == (Cout, 9 * Cin)
    got = ops.unpack_conv3x3_weight(dw, Cin)
    e = relerr(got, w.grad)
    assert e < 2e-5, e   # fp32 accumulation of exact bf16 products: only the summation order differs
    # every tap separately (a shifted tap shows up as an O(1) error in that tap only)
    for ky in range(3):
        for kx in range(3):
            assert relerr(got[:, :, ky, kx], w.grad[:, :, ky, kx]) < 5e-5, (ky, kx)
    # rounded like eager's bf16 backward, accumulated into an existing gradient
    acc = torch.ones(Cout, 9 * Cin, device=DEV)
    ops.conv3x3_wgrad(dy.permute(0, 2, 3, 1).contiguous(), x.permute(0, 2, 3, 1).contiguous(), acc, accumulate=True)
    assert torch.equal(acc - 1.0, (dw.to(torch.bfloat16).float() + 1.0) - 1.0) or relerr(acc - 1.0, dw.to(torch.bfloat16).float()) < 1e-3
