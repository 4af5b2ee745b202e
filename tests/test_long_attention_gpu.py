"""Streamed attention for sequences longer than 256 tokens (b200_attention_long_*): kernel parity against float64 references
and torch SDPA, determinism, the T dispatch in ops, and end-to-end training at ViT 384 px / a 300-token text tower.  The CPU case
checks the geometry limits (the entry points' argument checks are in test_attention_contract.py); the others need an H100
(pytest -m gpu)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import _cabi, ops, registry, vit  # noqa: E402
from _refs import packed_attention, rand_bf16, relerr, with_grads  # noqa: E402

DEV = "cuda"
LENGTHS = [257, 300, 384, 577, 1025, 2048, 4096]
# (B, H) per length: more CTAs than two per SM at every length up to 1025, a small B * H at 2048 / 4096
SHAPES = {257: (8, 12), 300: (5, 12), 384: (3, 8), 577: (4, 12), 1025: (2, 12), 2048: (1, 8), 4096: (1, 2)}


def _long_fwd(qkv, B, T, H, causal):
    out = torch.empty((B * T, H * 64), dtype=torch.bfloat16, device=DEV)
    lse = torch.empty((B, H, T), dtype=torch.float32, device=DEV)
    _cabi.call("b200_attention_long_fwd", qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, T, H, 64, 0.125, int(causal),
               torch.cuda.current_stream().cuda_stream)
    return out, lse


def _long_bwd(qkv, out, dout, lse, B, T, H, causal):
    """dqkv and the per-image column sums dbias_part [B, 3 * H * 64] straight from the entry point."""
    D = H * 64
    dqkv = torch.empty((B * T, 3 * D), dtype=torch.bfloat16, device=DEV)
    part = torch.full((B, 3 * D), float("nan"), dtype=torch.float32, device=DEV)
    ws = torch.full((int(_cabi.lib().b200_attention_long_bwd_workspace_floats(B, T, H)),), float("nan"), device=DEV)
    _cabi.call("b200_attention_long_bwd", qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), B, T, H, 64,
               0.125, int(causal), part.data_ptr(), ws.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return dqkv, part


def _check_fwd(out, lse, qkv, B, T, H, causal):
    torch.cuda.synchronize()
    ref_o, ref_lse = packed_attention(qkv, B, T, H, causal=causal)
    assert relerr(out, ref_o) < 5e-3, relerr(out, ref_o)
    assert torch.allclose(lse.double(), ref_lse, rtol=1e-4, atol=1e-4), (lse.double() - ref_lse).abs().max().item()
    q, k, v = qkv.view(B, T, 3, H, 64).permute(2, 0, 3, 1, 4)
    sdpa = F.scaled_dot_product_attention(q, k, v, is_causal=causal).permute(0, 2, 1, 3).reshape(B * T, H * 64)
    assert relerr(out, sdpa) < 5e-3, relerr(out, sdpa)


def _check_bwd(dqkv, part, qkv, dout, B, T, H, causal):
    torch.cuda.synchronize()
    D = H * 64
    _, (ref,) = with_grads(packed_attention, (qkv,), dout, B, T, H, 0.125, causal)
    for name, sl in (("dq", slice(0, D)), ("dk", slice(D, 2 * D)), ("dv", slice(2 * D, 3 * D))):
        e = relerr(dqkv[:, sl], ref[:, sl])
        assert e < 1e-2, f"{name}: {e}"
    ref_b = dqkv.float().view(B, T, 3 * D).sum(1)  # fp32 column sums of the bf16 rows returned, per image
    assert (part - ref_b).abs().max().item() <= 1e-5 * ref_b.abs().max().item(), (part - ref_b).abs().max().item()


# ---- 1. forward kernel -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("T", LENGTHS)
def test_long_attention_fwd(T, causal):
    B, H = SHAPES[T]
    qkv = rand_bf16(B * T, 3 * H * 64, seed=T)
    out, lse = ops.attention_fwd(qkv, B, T, H, causal=causal)
    _check_fwd(out, lse, qkv, B, T, H, causal)


# ---- 2. backward kernel: accuracy, fused bias gradient, bit-identical reruns ---------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("T", LENGTHS)
def test_long_attention_bwd(T, causal):
    B, H = SHAPES[T]
    if T == 4096:
        B, H = 1, 1
    D = H * 64
    qkv = rand_bf16(B * T, 3 * D, seed=T + 1)
    dout = rand_bf16(B * T, D, seed=T + 2)
    out, lse = ops.attention_fwd(qkv, B, T, H, causal=causal)
    dqkv, part = _long_bwd(qkv, out, dout, lse, B, T, H, causal)
    _check_bwd(dqkv, part, qkv, dout, B, T, H, causal)
    dqkv2, part2 = _long_bwd(qkv, out, dout, lse, B, T, H, causal)
    assert torch.equal(dqkv2, dqkv) and torch.equal(part2, part)
    # through ops: same dqkv, and the bias gradient is the bf16-rounded batch sum of the same column sums
    dbias = torch.zeros(3 * D, device=DEV)
    dqkv3 = ops.attention_bwd(qkv, out, dout, lse, B, T, H, causal=causal, dbias=dbias)
    assert torch.equal(dqkv3, dqkv)
    ref = part.double().sum(0)
    assert (dbias.double() - ref).abs().max().item() <= 2.0 ** -8 * ref.abs().max().item() + 1e-6
    assert torch.equal(dbias, dbias.to(torch.bfloat16).float())


# ---- 3. the new entry points over the short end of their range -----------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,T,H,causal", [(3, 16, 2, False), (5, 77, 8, True), (4, 197, 12, False), (2, 256, 4, False), (2, 256, 3, True)])
def test_long_entry_points_at_short_T(B, T, H, causal):
    D = H * 64
    qkv = rand_bf16(B * T, 3 * D, seed=T + 5)
    dout = rand_bf16(B * T, D, seed=T + 6)
    out, lse = _long_fwd(qkv, B, T, H, causal)
    _check_fwd(out, lse, qkv, B, T, H, causal)
    dqkv, part = _long_bwd(qkv, out, dout, lse, B, T, H, causal)
    _check_bwd(dqkv, part, qkv, dout, B, T, H, causal)


# ---- 4. dispatch boundary ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_dispatch_boundary():
    stream = torch.cuda.current_stream().cuda_stream
    # T = 256: the resident kernels, byte-for-byte
    B, T, H = 3, 256, 4
    D = H * 64
    qkv, dout = rand_bf16(B * T, 3 * D, seed=11), rand_bf16(B * T, D, seed=12)
    out, lse = ops.attention_fwd(qkv, B, T, H)
    out_r = torch.empty_like(out)
    lse_r = torch.empty_like(lse)
    _cabi.call("b200_attention_fwd", qkv.data_ptr(), out_r.data_ptr(), lse_r.data_ptr(), B, T, H, 64, 0.125, 0, stream)
    assert torch.equal(out, out_r) and torch.equal(lse, lse_r)
    dqkv = ops.attention_bwd(qkv, out, dout, lse, B, T, H)
    dqkv_r = torch.empty_like(dqkv)
    _cabi.call("b200_attention_bwd", qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv_r.data_ptr(), B, T, H, 64,
               0.125, 0, None, stream)
    assert torch.equal(dqkv, dqkv_r)
    # T = 257: the streamed kernels
    T = 257
    qkv, dout = rand_bf16(B * T, 3 * D, seed=13), rand_bf16(B * T, D, seed=14)
    out, lse = ops.attention_fwd(qkv, B, T, H, causal=True)
    out_l, lse_l = _long_fwd(qkv, B, T, H, True)
    assert torch.equal(out, out_l) and torch.equal(lse, lse_l)
    dqkv = ops.attention_bwd(qkv, out, dout, lse, B, T, H, causal=True)
    dqkv_l, _ = _long_bwd(qkv, out, dout, lse, B, T, H, True)
    assert torch.equal(dqkv, dqkv_l)


# ---- 5-7. end to end -----------------------------------------------------------------------------------------------------
VS_FP32_FACTOR = 1.5
VS_EAGER_FACTOR = 2.0
SLACK = 1e-3


def _cfg(name, **over):
    import vit_oracle as vo

    cfg = vo.vit_config(name)
    cfg.update(over)
    return cfg


def _build(cfg, sd):
    m = registry.build_module(
        "cv_clf", config=dict(in_channels=cfg["in_channels"], num_classes=cfg["num_classes"], img_size=cfg["img_size"],
                              latent_dim=cfg["latent_dim"], encoder="vit",
                              encoder_config=dict(patch_size=cfg["patch_size"], num_layers=cfg["num_layers"])))
    m.load_state_dict(sd, strict=True)
    return m.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("name,batch", [("vit_small", 4), ("vit_b16", 8)])
def test_train_step_parity_384px(name, batch):
    """T = 577 (384 px, patch 16): the three-way criterion against the oracle run eagerly in bf16 autocast and in fp32."""
    import vit_oracle as vo

    cfg = _cfg(name, img_size=384)
    sd = vo.init_state_dict(cfg, seed=0)
    x, y = vo.synthetic_batch(cfg, batch, seed=1)
    x, y = x.to(DEV), y.to(DEV)
    m = _build(cfg, sd)
    assert m.geo.T == 577
    logits = m(x)[vit.PREDICTIONS_KEY]
    loss = vit.cross_entropy(logits, y)
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().clone() for k, p in m.named_arena_parameters()}
    logits = logits.detach()
    sdg = {k: v.to(DEV) for k, v in sd.items()}
    e_loss, e_grads, e_taps = vo.train_step(sdg, x, y, cfg, autocast_bf16=True, want_taps=True)
    f_loss, f_grads, f_taps = vo.train_step(sdg, x, y, cfg, autocast_bf16=False, want_taps=True)
    floor = relerr(e_taps["logits"], f_taps["logits"])
    assert relerr(logits, e_taps["logits"]) < VS_EAGER_FACTOR * floor + SLACK
    assert relerr(logits, f_taps["logits"]) < VS_FP32_FACTOR * floor + SLACK
    assert abs(loss.item() - f_loss.item()) < 1.5 * abs(e_loss.item() - f_loss.item()) + 2e-3 * max(1.0, abs(f_loss.item()))
    assert set(grads) == set(e_grads)
    for k in sorted(grads):
        ours_vs_eager, ours_vs_fp32, eager_vs_fp32 = relerr(grads[k], e_grads[k]), relerr(grads[k], f_grads[k]), relerr(e_grads[k], f_grads[k])
        assert ours_vs_eager < VS_EAGER_FACTOR * eager_vs_fp32 + SLACK, f"{k}: ours vs eager {ours_vs_eager}, floor {eager_vs_fp32}"
        assert ours_vs_fp32 < VS_FP32_FACTOR * eager_vs_fp32 + SLACK, (k, ours_vs_fp32, eager_vs_fp32)


@pytest.mark.gpu
def test_text_stack_parity_context_300():
    """TeTEncoder with a 300-token causal context: the criterion of the CLIP text-stack parity test."""
    import vit_oracle as vo

    cfg = vo.tet_config("clip_text_small")
    cfg["context_length"] = 300
    d, t, batch = cfg["latent_dim"], cfg["context_length"], 4
    sd = vo.tet_init_state_dict(cfg, seed=0)
    m = registry.build_module("tet", config=dict(latent_dim=d, context_length=t, use_triu_attn_mask=True, num_layers=cfg["num_layers"],
                                                 norm_kwargs={"eps": cfg["eps"]}, attention_kwargs={"num_heads": d // 64},
                                                 feedforward_kwargs={"activation": "quick_gelu"}, head_pooler=None))
    m.load_state_dict(sd, strict=False)
    m = m.to(DEV)
    g = torch.Generator().manual_seed(7)
    x = (torch.randn(batch, t, d, generator=g) * 0.5).to(DEV)
    up = torch.randn(batch, t, d, generator=g).to(DEV)
    xin = x.clone().requires_grad_(True)
    out = m(xin)
    (out * up).sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    sdg = {k: v.to(DEV) for k, v in sd.items()}
    e_out, e_dx, e_grads = vo.tet_train_step(sdg, x, up, cfg, autocast_bf16=True)
    f_out, f_dx, f_grads = vo.tet_train_step(sdg, x, up, cfg, autocast_bf16=False)
    floor = relerr(e_out, f_out)
    assert relerr(out, e_out) < VS_EAGER_FACTOR * floor + SLACK and relerr(out, f_out) < VS_FP32_FACTOR * floor + SLACK
    dfloor = relerr(e_dx, f_dx)
    assert relerr(xin.grad, e_dx) < VS_EAGER_FACTOR * dfloor + SLACK and relerr(xin.grad, f_dx) < VS_FP32_FACTOR * dfloor + SLACK
    assert set(grads) == set(e_grads)
    for k in sorted(grads):
        ours_vs_eager, ours_vs_fp32, eager_vs_fp32 = relerr(grads[k], e_grads[k]), relerr(grads[k], f_grads[k]), relerr(e_grads[k], f_grads[k])
        assert ours_vs_eager < VS_EAGER_FACTOR * eager_vs_fp32 + SLACK, f"{k}: ours vs eager {ours_vs_eager}, floor {eager_vs_fp32}"
        assert ours_vs_fp32 < VS_FP32_FACTOR * eager_vs_fp32 + SLACK, (k, ours_vs_fp32, eager_vs_fp32)


@pytest.mark.gpu
def test_graphed_train_step_at_577_tokens():
    """CUDA-graphed zero_grad + fwd + CE + bwd + Adam == three eager steps at T = 577 (the attention workspace is sized
    during the warm-up and replayed as is)."""
    import vit_oracle as vo
    from cflearn_b200.optim import ArenaAdam, GraphedTrainStep

    cfg = _cfg("vit_tiny", img_size=384)
    sd = vo.init_state_dict(cfg, seed=0)
    xs = [vo.synthetic_batch(cfg, 4, seed=s) for s in (1, 2, 3)]
    eager = _build(cfg, sd)
    opt_e = ArenaAdam(eager, lr=1e-3)
    losses_e = []
    for x, y in xs:
        opt_e.zero_grad()
        losses_e.append(eager.train_step(x.to(DEV), y.to(DEV)).item())
        opt_e.step()
    graphed = _build(cfg, sd)
    graphed.arena.ensure()
    opt_g = ArenaAdam(graphed, lr=1e-3, capturable=True)
    gs = GraphedTrainStep(graphed, opt_g, batch=4, warmup=2)
    losses_g = [gs.step(x.to(DEV), y.to(DEV)).item() for x, y in xs]
    torch.cuda.synchronize()
    for a, b in zip(losses_e, losses_g):
        assert abs(a - b) < 1e-5 * max(1.0, abs(a)), (losses_e, losses_g)
    for (k, p), (_, q) in zip(eager.named_parameters(), graphed.named_parameters()):
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), k


# ---- 8. CPU: geometry limits -------------------------------------------------------------------------------------------
def test_long_geometries_build_without_gpu():
    m = registry.build_module("cv_clf", config=dict(in_channels=3, num_classes=8, img_size=384, latent_dim=64, encoder="vit",
                                                    encoder_config=dict(patch_size=16, num_layers=1)))
    assert m.geo.T == 577
    e = registry.build_module("encoders.vit", config=dict(img_size=512, patch_size=16, in_channels=3, latent_dim=64, num_layers=1))
    assert e is not None
    t = registry.build_module("tet", config=dict(latent_dim=64, context_length=ops.ATTENTION_MAX_T, num_layers=1,
                                                 attention_kwargs={"num_heads": 1}, head_pooler=None))
    assert tuple(t.state_dict()["encoder.pos_encoding.pos_encoding"].shape) == (1, ops.ATTENTION_MAX_T, 64)
    assert ops.ATTENTION_MAX_T == 16384
    with pytest.raises(NotImplementedError):  # 129 x 129 patches + the head token = 16642 tokens
        registry.build_module("cv_clf", config=dict(in_channels=3, num_classes=8, img_size=16 * 129, latent_dim=64, encoder="vit",
                                                    encoder_config=dict(patch_size=16, num_layers=1)))
    with pytest.raises(NotImplementedError):
        registry.build_module("tet", config=dict(latent_dim=64, context_length=ops.ATTENTION_MAX_T + 1, num_layers=1,
                                                 attention_kwargs={"num_heads": 1}, head_pooler=None))
