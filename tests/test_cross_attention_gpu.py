"""Attention with separate Q / K / V and head dims up to 160 (b200_cross_attention_*, ops.cross_attention_*, CrossAttentionB200):
kernel parity against float64 math and torch SDPA, determinism (including the query-split dK / dV grid), equality with the packed
Dh-64 entry points, and module parity against oracle/unet_oracle.py::cross_attention at SD-v1.5 widths.  The CPU cases check the
module's parameters and its refusals (the entry points' argument checks and workspace formula are in test_attention_contract.py);
the others need an H100 (pytest -m gpu)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import _cabi, ops  # noqa: E402
from cflearn_b200.attention import CrossAttentionB200  # noqa: E402
from _refs import attention_rows, rand_bf16, relerr, with_grads  # noqa: E402

DEV = "cuda"


def _heads(x, B, H):  # [B*T, >= H*Dh] view -> [B, H, T, Dh]
    Dh = x.shape[1] // H
    return x.reshape(B, -1, H, Dh).permute(0, 2, 1, 3)


def _operands(B, Tq, Tk, H, Dh, packed, seed):
    """q / k / v as column views of packed projection outputs (self: one [M, 3L] buffer; cross: q [M, L] + kv [Mc, 2L]) or as
    separate contiguous tensors."""
    L = H * Dh
    if packed and Tq == Tk:
        qkv = rand_bf16(B * Tq, 3 * L, seed=seed)
        return qkv[:, :L], qkv[:, L:2 * L], qkv[:, 2 * L:]
    if packed:
        kv = rand_bf16(B * Tk, 2 * L, seed=seed + 1)
        return rand_bf16(B * Tq, L, seed=seed), kv[:, :L], kv[:, L:]
    return rand_bf16(B * Tq, L, seed=seed), rand_bf16(B * Tk, L, seed=seed + 1), rand_bf16(B * Tk, L, seed=seed + 2)


def _bwd(q, k, v, out, dout, lse, B, H, causal, packed):
    if not packed:
        return ops.cross_attention_bwd(q, k, v, out, dout, lse, B, H, causal=causal)
    L = q.shape[1]
    if q.stride(0) == 3 * L:  # self-attention: one packed [M, 3L] gradient
        g = torch.empty((q.shape[0], 3 * L), dtype=torch.bfloat16, device=DEV)
        return ops.cross_attention_bwd(q, k, v, out, dout, lse, B, H, causal=causal, dq=g[:, :L], dk=g[:, L:2 * L], dv=g[:, 2 * L:])
    g = torch.empty((k.shape[0], 2 * L), dtype=torch.bfloat16, device=DEV)
    return ops.cross_attention_bwd(q, k, v, out, dout, lse, B, H, causal=causal, dq=torch.empty_like(q), dk=g[:, :L], dv=g[:, L:])


def _run_case(B, Tq, Tk, H, Dh, causal, packed, seed=0):
    q, k, v = _operands(B, Tq, Tk, H, Dh, packed, seed)
    out, lse = ops.cross_attention_fwd(q, k, v, B, H, causal=causal)
    torch.cuda.synchronize()
    scale = Dh ** -0.5
    ref_o, ref_lse = attention_rows(q, k, v, B, H, scale, causal)
    assert relerr(out, ref_o) < 5e-3, relerr(out, ref_o)
    assert torch.allclose(lse.double(), ref_lse, rtol=1e-4, atol=1e-4), (lse.double() - ref_lse).abs().max().item()
    sdpa = F.scaled_dot_product_attention(*(_heads(t, B, H) for t in (q, k, v)), is_causal=causal)
    assert relerr(out, sdpa.permute(0, 2, 1, 3).reshape(B * Tq, H * Dh)) < 5e-3
    dout = rand_bf16(B * Tq, H * Dh, seed=seed + 7)
    dq, dk, dv = _bwd(q, k, v, out, dout, lse, B, H, causal, packed)
    torch.cuda.synchronize()
    _, (dq64, dk64, dv64) = with_grads(attention_rows, (q, k, v), dout, B, H, scale, causal)
    for name, ours, ref in (("dq", dq, dq64), ("dk", dk, dk64), ("dv", dv, dv64)):
        if name != "dv" and Tk == 1:  # one key: P = 1 and dS = 0, so dQ / dK are 0 up to rounding and a relative error means nothing
            assert ours.double().norm() <= 1e-2 * dv64.norm(), ours.float().norm().item()
            continue
        e = relerr(ours, ref)
        assert e < 1e-2, f"{name}: {e}"
    return q, k, v, out, dout, lse, (dq, dk, dv)


# ---- 1. kernel parity ----------------------------------------------------------------------------------------------------
DHS = [8, 40, 64, 80, 128, 160]


@pytest.mark.gpu
@pytest.mark.parametrize("Dh", DHS)
@pytest.mark.parametrize("T", [1, 77, 300, 1024, 4096])
@pytest.mark.parametrize("causal", [False, True])
def test_self_attention(T, Dh, causal):
    B, H = (2, 3) if T <= 300 else (1, 2)
    _run_case(B, T, T, H, Dh, causal, packed=(T + Dh) % 2 == 0, seed=T + Dh)


@pytest.mark.gpu
@pytest.mark.parametrize("Dh", DHS)
@pytest.mark.parametrize("Tq,Tk", [(64, 77), (300, 1), (1024, 77), (4096, 77), (256, 200), (4096, 200)])
@pytest.mark.parametrize("packed", [False, True])
def test_cross_attention(Tq, Tk, Dh, packed):
    B, H = (2, 4) if Tq <= 1024 else (1, 2)
    _run_case(B, Tq, Tk, H, Dh, False, packed, seed=Tq + Tk + Dh)


# ---- 2. determinism, including the query-split dK / dV grid (small B * H, 77 keys) -----------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("Dh", [40, 80, 160])
@pytest.mark.parametrize("B,H,Tq,Tk", [(1, 2, 4096, 77), (8, 8, 4096, 77), (2, 2, 1024, 1024)])
def test_backward_is_deterministic(B, H, Tq, Tk, Dh):
    if B * H * Tq > 2 * 4096 * 8 and Dh == 160:
        Tq = 1024
    q, k, v, out, dout, lse, g1 = _run_case(B, Tq, Tk, H, Dh, False, packed=False, seed=3)
    g2 = ops.cross_attention_bwd(q, k, v, out, dout, lse, B, H)
    for a, b in zip(g1, g2):
        assert torch.equal(a, b)


# ---- 3. the packed Dh-64 entry points are the same kernels ----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,T,H,causal", [(8, 577, 12, False), (4, 1025, 12, True), (16, 300, 8, False)])
def test_matches_long_entry_points(B, T, H, causal):
    """Grids of >= 132 dK / dV CTAs: the new entry does not split the queries, so it must equal b200_attention_long_* bit for bit."""
    D = H * 64
    qkv = rand_bf16(B * T, 3 * D, seed=T)
    dout = rand_bf16(B * T, D, seed=T + 1)
    stream = torch.cuda.current_stream().cuda_stream
    out_l = torch.empty((B * T, D), dtype=torch.bfloat16, device=DEV)
    lse_l = torch.empty((B, H, T), dtype=torch.float32, device=DEV)
    _cabi.call("b200_attention_long_fwd", qkv.data_ptr(), out_l.data_ptr(), lse_l.data_ptr(), B, T, H, 64, 0.125, int(causal), stream)
    dqkv_l = torch.empty((B * T, 3 * D), dtype=torch.bfloat16, device=DEV)
    ws = torch.empty(int(_cabi.lib().b200_attention_long_bwd_workspace_floats(B, T, H)), device=DEV)
    _cabi.call("b200_attention_long_bwd", qkv.data_ptr(), out_l.data_ptr(), dout.data_ptr(), lse_l.data_ptr(), dqkv_l.data_ptr(), B, T, H, 64,
               0.125, int(causal), None, ws.data_ptr(), stream)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    out, lse = ops.cross_attention_fwd(q, k, v, B, H, causal=causal)
    assert torch.equal(out, out_l) and torch.equal(lse, lse_l)
    dqkv = torch.empty_like(dqkv_l)
    ops.cross_attention_bwd(q, k, v, out, dout, lse, B, H, causal=causal, dq=dqkv[:, :D], dk=dqkv[:, D:2 * D], dv=dqkv[:, 2 * D:])
    assert torch.equal(dqkv, dqkv_l)


# ---- 4. module parity at SD-v1.5 widths -------------------------------------------------------------------------------------
def _module_sd(query_dim, context_dim, L, seed):
    g = torch.Generator().manual_seed(seed)
    return {"to_q.weight": torch.randn(L, query_dim, generator=g) * query_dim ** -0.5,
            "to_k.weight": torch.randn(L, context_dim, generator=g) * context_dim ** -0.5,
            "to_v.weight": torch.randn(L, context_dim, generator=g) * context_dim ** -0.5,
            "out_linear.0.weight": torch.randn(query_dim, L, generator=g) * L ** -0.5,
            "out_linear.0.bias": torch.randn(query_dim, generator=g) * 0.1}


def _oracle(sd, net, context, heads, autocast):
    import unet_oracle as uo

    sdg = {k: v.detach().clone().requires_grad_(True) for k, v in sd.items()}
    net = net.detach().clone().requires_grad_(True)
    ctx = None if context is None else context.detach().clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        y = uo.cross_attention(sdg, "", net, ctx, heads)
    return y, net, ctx, sdg


@pytest.mark.gpu
@pytest.mark.parametrize("query_dim,side", [(320, 64), (1280, 16)])
@pytest.mark.parametrize("cross", [False, True])
def test_module_parity(query_dim, side, cross):
    heads, B = 8, 2
    L = query_dim
    context_dim = 768 if cross else None
    sd = _module_sd(query_dim, context_dim or query_dim, L, seed=query_dim + int(cross))
    m = CrossAttentionB200(query_dim=query_dim, context_dim=context_dim, num_heads=heads, head_dim=L // heads).to(DEV)
    m.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(5)
    net = torch.randn(B, side * side, query_dim, generator=g).to(DEV)
    context = torch.randn(B, 77, 768, generator=g).to(DEV) if cross else None
    up = torch.randn(B, side * side, query_dim, generator=g).to(DEV)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    xin = net.clone().requires_grad_(True)
    cin = None if context is None else context.clone().requires_grad_(True)
    y = m(xin, context=cin)
    assert y.dtype == torch.bfloat16
    (y.float() * up).sum().backward()
    ours = {"out": y, "net": xin.grad, **{k: p.grad for k, p in m.named_parameters()}}
    if cross:
        ours["context"] = cin.grad
        assert cin.grad.dtype == torch.float32
    refs = []
    for autocast in (True, False):
        ye, ne, ce, sdg = _oracle(sdd, net, context, heads, autocast)
        (ye.float() * up).sum().backward()
        r = {"out": ye, "net": ne.grad, **{k: sdg[k].grad for k in sd}}
        if cross:
            r["context"] = ce.grad
        refs.append(r)
    eager, fp32 = refs
    for k in ours:
        floor = relerr(eager[k], fp32[k])
        assert relerr(ours[k], fp32[k]) <= 1.5 * floor + 1e-6, (k, relerr(ours[k], fp32[k]), floor)
        assert relerr(ours[k], eager[k]) <= 2.0 * floor + 1e-6, (k, relerr(ours[k], eager[k]), floor)


# ---- 5. CPU: the module's parameters and refusals ----------------------------------------------------------------------------
def _reference_attn_shapes():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "unet_tiny_reference.pt"), weights_only=False)
    groups = {}
    for key, shape in fx["shapes"]:
        for tag in (".attn1.", ".attn2."):
            if tag in key:
                pre, rest = key.split(tag)
                groups.setdefault(pre + tag, []).append((rest, tuple(shape)))
    return groups


def test_module_parameters_match_reference():
    groups = _reference_attn_shapes()
    assert groups
    for prefix, items in groups.items():
        shapes = dict(items)
        L, query_dim = shapes["to_q.weight"]
        context_dim = shapes["to_k.weight"][1] if prefix.endswith("attn2.") else None
        m = CrossAttentionB200(query_dim=query_dim, context_dim=context_dim, num_heads=8, head_dim=L // 8)
        got = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
        assert got == items, prefix
        assert all(v.dtype == torch.float32 for v in m.state_dict().values())
        sd = {k: torch.randn(s) for k, s in items}
        m.load_state_dict(sd, strict=True)
        back = CrossAttentionB200(query_dim=query_dim, context_dim=context_dim, num_heads=8, head_dim=L // 8)
        back.load_state_dict(m.state_dict(), strict=True)
        assert all(torch.equal(back.state_dict()[k], sd[k]) for k in sd)


def test_module_refuses_dropout_and_masks():
    with pytest.raises(NotImplementedError):
        CrossAttentionB200(query_dim=64, num_heads=8, head_dim=8, dropout=0.1)
    m = CrossAttentionB200(query_dim=64, num_heads=8, head_dim=8)
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 4, 64), mask=torch.ones(1, 4, 4, dtype=torch.bool))
