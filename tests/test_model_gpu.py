"""End-to-end parity of the native ViT classifier training step against the oracle (oracle/vit_oracle.py, pinned to the
reference), on the GPU.  Three comparisons per configuration:

  (1) vs the oracle run EAGERLY ON THE SAME GPU under bf16 autocast -- "the reference's own PyTorch-eager path":
      relative L2 error of logits / loss / every parameter gradient within the tolerances below;
  (2) vs the fp32 oracle: our bf16 path must be as close to the exact answer as eager bf16 is (<= 1.5x its error);
  (3) vs the golden vectors generated from the real reference on CPU (tests/golden/vit_tiny_reference.pt).

Tolerances (relative L2).  Single ops match bf16(exact) to < 3e-4 (tests/test_kernels_gpu.py), inside BASELINE.json's
1e-3.  End to end that figure is NOT attainable between ANY two bf16 pipelines: the reference's own eager-autocast path
sits several 1e-3 away from its own fp32 path, and once one bf16 rounding decision differs, downstream roundings decorrelate
within a layer or two.  The end-to-end criterion is therefore "as close to the exact answer as the reference's bf16 path is":
    err(ours, fp32)  <= 1.5 x err(eager_bf16, fp32) + 1e-3      and      err(ours, eager_bf16) <= 2 x err(eager_bf16, fp32) + 1e-3
The integer label path is exact.
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import golden_sample  # noqa: E402
import vit_oracle as vo  # noqa: E402

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import registry, vit  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"

VS_FP32_FACTOR = 1.5
VS_EAGER_FACTOR = 2.0
SLACK = 1e-3


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


def build(cfg, sd):
    m = registry.build_module(
        "cv_clf", config=dict(in_channels=cfg["in_channels"], num_classes=cfg["num_classes"], img_size=cfg["img_size"],
                              latent_dim=cfg["latent_dim"], encoder="vit",
                              encoder_config=dict(patch_size=cfg["patch_size"], num_layers=cfg["num_layers"])))
    m.load_state_dict(sd, strict=True)
    return m.to(DEV)


def run_ours(cfg, sd, x, y):
    m = build(cfg, sd)
    logits = m(x)[vit.PREDICTIONS_KEY]
    loss = vit.cross_entropy(logits, y)
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().clone() for k, p in m.named_arena_parameters()}  # ViTEncoder keys + head.linear.*: the oracle's names
    return logits.detach(), loss.detach(), grads, m


def oracle_on_gpu(cfg, sd, x, y, autocast):
    sdg = {k: v.to(DEV) for k, v in sd.items()}
    loss, grads, taps = vo.train_step(sdg, x, y, cfg, autocast_bf16=autocast, want_taps=True)
    return taps["logits"], loss, grads


@pytest.mark.parametrize("name,batch", [("vit_tiny", 4), ("vit_small", 6), ("vit_b16", 8)])
def test_train_step_parity(name, batch):
    cfg = vo.vit_config(name)
    sd = vo.init_state_dict(cfg, seed=0)
    x, y = vo.synthetic_batch(cfg, batch, seed=1)
    x, y = x.to(DEV), y.to(DEV)
    logits, loss, grads, _ = run_ours(cfg, sd, x, y)
    e_logits, e_loss, e_grads = oracle_on_gpu(cfg, sd, x, y, True)   # eager bf16 autocast: the parity target
    f_logits, f_loss, f_grads = oracle_on_gpu(cfg, sd, x, y, False)  # fp32: the exact answer
    assert set(grads) == set(e_grads)
    assert logits.dtype == torch.bfloat16 and e_logits.dtype == torch.bfloat16
    err_logits = rel(logits, e_logits)
    floor = rel(e_logits, f_logits)
    assert err_logits < VS_EAGER_FACTOR * floor + SLACK, f"logits vs eager: {err_logits} (eager vs fp32 {floor})"
    assert rel(logits, f_logits) < VS_FP32_FACTOR * floor + SLACK
    assert abs(loss.item() - f_loss.item()) < 1.5 * abs(e_loss.item() - f_loss.item()) + 2e-3 * max(1.0, abs(f_loss.item()))
    worst = 0.0
    for k in sorted(grads):
        ours_vs_eager = rel(grads[k], e_grads[k])
        ours_vs_fp32 = rel(grads[k], f_grads[k])
        eager_vs_fp32 = rel(e_grads[k], f_grads[k])
        worst = max(worst, ours_vs_fp32 / max(eager_vs_fp32, 1e-12))
        assert ours_vs_eager < VS_EAGER_FACTOR * eager_vs_fp32 + SLACK, f"{k}: ours vs eager {ours_vs_eager}, floor {eager_vs_fp32}"
        assert ours_vs_fp32 < VS_FP32_FACTOR * eager_vs_fp32 + SLACK, (k, ours_vs_fp32, eager_vs_fp32)
    print(f"{name}: logits vs eager {err_logits:.2e} (bf16 floor {floor:.2e}); worst grad err ratio ours/eager vs fp32 {worst:.2f}")


def test_against_reference_golden_vectors():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "vit_tiny_reference.pt"), weights_only=False)
    cfg = vo.vit_config(fx["config_name"])
    sd = vo.init_state_dict(cfg, seed=fx["weights_seed"])
    x, y = fx["x"].to(DEV), fx["labels"].to(DEV)
    logits, loss, grads, _ = run_ours(cfg, sd, x, y)
    ref_bf16, ref_fp32 = fx["reference"]["bf16"], fx["reference"]["fp32"]
    assert rel(logits.cpu(), ref_fp32["logits"]) < 1e-2
    assert abs(loss.item() - ref_fp32["loss"].item()) < 1e-2
    for k, g in ref_fp32["grads"].items():
        ours = rel(golden_sample.take(grads[k], fx["grad_sample"][k]), g)
        theirs = rel(ref_bf16["grads"][k], g)  # how far the reference's own bf16 (CPU autocast) path is from its fp32 path
        assert ours < max(2.0 * theirs, 5e-3), (k, ours, theirs)


def test_label_path_is_integer_exact():
    cfg = vo.vit_config("vit_tiny")
    sd = vo.init_state_dict(cfg, seed=0)
    x, y = vo.synthetic_batch(cfg, 4, seed=1)
    m = build(cfg, sd)
    logits = m(x.to(DEV))[vit.PREDICTIONS_KEY].detach()
    from cflearn_b200 import ops

    _, rows, _, bad = ops.softmax_xent(logits, y.to(DEV).reshape(-1), need_grad=False)
    ref = -torch.log_softmax(logits.float(), 1).gather(1, y.to(DEV))[:, 0]
    assert bad.item() == 0
    assert torch.allclose(rows, ref, rtol=1e-6, atol=1e-6)
    # permuting labels permutes exactly which logit is picked: loss difference equals the logit difference
    y2 = (y + 1) % cfg["num_classes"]
    _, rows2, _, _ = ops.softmax_xent(logits, y2.to(DEV).reshape(-1), need_grad=False)
    picked = logits.float().gather(1, y.to(DEV))[:, 0] - logits.float().gather(1, y2.to(DEV))[:, 0]
    assert torch.allclose(rows2 - rows, picked, rtol=1e-5, atol=1e-5)


def test_encoder_module_and_registry_surface():
    cfg = vo.vit_config("vit_small")
    enc = registry.build_encoder("vit", config=dict(img_size=cfg["img_size"], patch_size=cfg["patch_size"], in_channels=3,
                                                    latent_dim=cfg["latent_dim"], num_layers=cfg["num_layers"], unknown_key=1))
    sd = {k: v for k, v in vo.init_state_dict(cfg, seed=3).items() if not k.startswith("head.linear")}
    enc.load_state_dict(sd, strict=True)
    enc = enc.to(DEV)
    x, _ = vo.synthetic_batch(cfg, 5, seed=2)
    out = enc.encode(x.to(DEV))
    assert out.dtype == torch.float32 and out.shape == (5, cfg["latent_dim"])
    sdg = {k: v.to(DEV) for k, v in sd.items()}
    with torch.autocast("cuda", dtype=torch.bfloat16):
        ref = vo.encoder_forward(sdg, x.to(DEV), cfg)
    exact = vo.encoder_forward(sdg, x.to(DEV), cfg)
    assert rel(out, exact) < VS_FP32_FACTOR * rel(ref, exact) + SLACK
    assert rel(out, ref) < VS_EAGER_FACTOR * rel(ref, exact) + SLACK
    out.sum().backward()
    assert all(p.grad is not None for p in enc.parameters())
    with pytest.raises(NotImplementedError):
        registry.build_encoder("vit", config=dict(img_size=32, patch_size=16, in_channels=3, latent_dim=128, dropout=0.1))


def test_gradient_accumulation_and_adam_step():
    from cflearn_b200.optim import ArenaAdam

    cfg = vo.vit_config("vit_tiny")
    sd = vo.init_state_dict(cfg, seed=0)
    x, y = vo.synthetic_batch(cfg, 4, seed=1)
    x, y = x.to(DEV), y.to(DEV)
    m = build(cfg, sd)
    m.train_step(x, y)
    g1 = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.train_step(x, y)  # p.grad still set -> accumulates
    for k, p in m.named_parameters():
        assert rel(p.grad, 2 * g1[k]) < 1e-6, k
    # Adam: compare one step with torch.optim.Adam on the same gradients
    ref_params = [p.detach().clone().requires_grad_(True) for p in m.parameters()]
    for rp, p in zip(ref_params, m.parameters()):
        rp.grad = p.grad.clone()
    torch.optim.Adam(ref_params, lr=1e-3).step()
    opt = ArenaAdam(m, lr=1e-3)
    opt.step()
    torch.cuda.synchronize()
    for rp, p in zip(ref_params, m.parameters()):
        assert torch.allclose(p, rp, rtol=1e-5, atol=1e-7)
    opt.zero_grad()
    assert all(p.grad is None for p in m.parameters())
    m.train_step(x, y)
    assert all(p.grad is not None for p in m.parameters())


def test_graphed_train_step_matches_eager_steps():
    """CUDA-graphed zero_grad + fwd + CE + bwd + Adam == the same three steps launched eagerly (same kernels)."""
    from cflearn_b200.optim import ArenaAdam, GraphedTrainStep

    cfg = vo.vit_config("vit_tiny")
    sd = vo.init_state_dict(cfg, seed=0)
    xs = [vo.synthetic_batch(cfg, 4, seed=s) for s in (1, 2, 3)]
    eager = build(cfg, sd)
    opt_e = ArenaAdam(eager, lr=1e-3)
    losses_e = []
    for x, y in xs:
        opt_e.zero_grad()
        losses_e.append(eager.train_step(x.to(DEV), y.to(DEV)).item())
        opt_e.step()
    graphed = build(cfg, sd)
    graphed.arena.ensure()
    opt_g = ArenaAdam(graphed, lr=1e-3, capturable=True)
    # the capture's warm-up steps (real Adam updates on an all-zero batch) must leave no trace: no manual reset here
    gs = GraphedTrainStep(graphed, opt_g, batch=4, warmup=2)
    assert int(opt_g.step_dev.item()) == 0 and float(opt_g.exp_avg.abs().max()) == 0.0
    for k, p in graphed.named_arena_parameters():
        assert torch.equal(p.detach().cpu(), sd[k]), k
    losses_g = [gs.step(x.to(DEV), y.to(DEV)).item() for x, y in xs]
    torch.cuda.synchronize()
    assert gs.launches_per_replay > 50
    for a, b in zip(losses_e, losses_g):
        assert abs(a - b) < 1e-5 * max(1.0, abs(a)), (losses_e, losses_g)
    for (k, p), (_, q) in zip(eager.named_parameters(), graphed.named_parameters()):
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), k


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_bucketed_allreduce_matches_single_process():
    import subprocess

    res = subprocess.run(
        [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
         "--master-port", "29533", os.path.join(ROOT, "tools", "dp_check.py")],
        stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert res.returncode == 0 and "dp_check: world 2" in res.stdout, res.stdout[-2000:]


# ---- FCNN (BASELINE.json configs[0]; reference: modules/ml/fcnn.py + multi_task[mae, mse]) --------------------------
@pytest.mark.gpu
def test_fcnn_step_matches_reference_golden_and_oracle():
    """fp32 fused FCNN step vs (1) the golden vectors written from the REAL reference on the toy batch and (2) the fp32
    oracle on 1000 rows (8 blocks, ragged tail).  Tolerance 1e-5 relative (fp32, different summation order)."""
    import fcnn_oracle as fo

    dev = torch.device("cuda", 0)
    g = torch.load(os.path.join(ROOT, "tests", "golden", "fcnn_reference.pt"))
    sd = fo.init_state_dict(10, 1, seed=g["weights_seed"])
    m = registry.build_module("fcnn", config=dict(input_dim=10, output_dim=1)).to(dev)
    m.load_state_dict(sd, strict=True)

    def rel(a, b):
        return ((a.detach().cpu().double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()

    loss, pred = m.train_step(g["x"].to(dev), g["y"].to(dev))
    assert rel(pred, g["pred"]) < 1e-5 and abs(loss.item() - g["loss"].item()) < 1e-5 * abs(g["loss"].item())
    for k, p in m.named_parameters():
        assert rel(p.grad, g["grads"][k]) < 1e-5, k
    # plain forward (inference) and the autograd route with a user-side loss
    with torch.no_grad():
        assert rel(m(g["x"].to(dev)), g["pred"]) < 1e-5
    for p in m.parameters():
        p.grad = None
    out = m(g["x"].to(dev))
    yd = g["y"].to(dev)
    (torch.nn.functional.l1_loss(out, yd) + torch.nn.functional.mse_loss(out, yd)).backward()
    for k, p in m.named_parameters():
        assert rel(p.grad, g["grads"][k]) < 1e-5, k
    # 1000 rows: 8 blocks of 128 with a ragged tail, against the oracle
    x_all, y_all = fo.toy_data()
    o_loss, o_pred, o_grads = fo.train_step(sd, x_all, y_all)
    loss, pred = m.train_step(x_all.to(dev), y_all.to(dev))
    assert rel(pred, o_pred) < 1e-5 and abs(loss.item() - o_loss.item()) < 1e-5 * abs(o_loss.item())
    for k, p in m.named_parameters():
        assert rel(p.grad, o_grads[k]) < 2e-5, k
    # a wider / deeper network with 3 outputs and no bias
    sd2 = fo.init_state_dict(7, 3, hidden=[48, 64, 16], seed=3)
    sd2 = {k: v for k, v in sd2.items() if not k.endswith("bias")}
    m2 = registry.build_module("fcnn", input_dim=7, output_dim=3, hidden_units=[48, 64, 16], bias=False).to(dev)
    m2.load_state_dict(sd2, strict=True)
    x2, y2 = torch.randn(300, 7), torch.randn(300, 3)
    params = {k: v.clone().requires_grad_(True) for k, v in sd2.items()}
    net = x2
    for i in range(3):
        net = torch.relu(net @ params[f"net.{i}.linear.linear.weight"].t())
    ref_pred = net @ params["net.3.weight"].t()
    ref_loss = (ref_pred - y2).abs().mean() + ((ref_pred - y2) ** 2).mean()
    ref_loss.backward()
    loss, pred = m2.train_step(x2.to(dev), y2.to(dev))
    assert rel(pred, ref_pred.detach()) < 1e-5 and abs(loss.item() - ref_loss.item()) < 1e-5 * abs(ref_loss.item())
    for k, p in m2.named_parameters():
        assert rel(p.grad, params[k].grad) < 2e-5, k


# ---- CLIP vision tower: the ViTEncoder CLIP._init_vision builds (multimodal/clip.py:121-135) --------------------------
def _clip_vision_module(cfg, sd):
    d = cfg["latent_dim"]
    m = registry.build_module("encoders.vit", config=dict(
        img_size=cfg["img_size"], patch_size=cfg["patch_size"], in_channels=cfg["in_channels"], latent_dim=d,
        to_patches_config={"bias": False}, num_layers=cfg["num_layers"], norm_kwargs={"eps": cfg["eps"]},
        embedding_norm=torch.nn.LayerNorm(d, cfg["eps"]), attention_kwargs={"num_heads": d // 64},
        feedforward_kwargs={"activation": "quick_gelu"}, norm_after_head=True, output_dim=cfg["output_dim"]))
    m.load_state_dict(sd, strict=True)
    return m.to(DEV)


@pytest.mark.parametrize("name,batch", [("clip_vision_tiny", 3), ("clip_vision_small", 5), ("clip_vision_b32", 8)])
def test_clip_vision_tower_parity(name, batch):
    """Same three-way criterion as the classifier: ours vs the oracle eagerly on this GPU under bf16 autocast, both against
    the fp32 oracle; the scalar is sum(out * upstream) (the reference defines no loss for CLIP)."""
    cfg = vo.vit_config(name)
    sd = vo.init_state_dict(cfg, seed=0)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(batch, cfg["in_channels"], cfg["img_size"], cfg["img_size"], generator=g).to(DEV)
    up = torch.randn(batch, cfg["output_dim"], generator=g).to(DEV)
    m = _clip_vision_module(cfg, sd)
    out = m(x)
    assert out.dtype == torch.bfloat16 and tuple(out.shape) == (batch, cfg["output_dim"])
    (out.float() * up).sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    sdg = {k: v.to(DEV) for k, v in sd.items()}
    e_out, e_grads, _ = vo.encoder_train_step(sdg, x, up, cfg, autocast_bf16=True)
    f_out, f_grads, _ = vo.encoder_train_step(sdg, x, up, cfg, autocast_bf16=False)
    floor = rel(e_out, f_out)
    assert rel(out, e_out) < VS_EAGER_FACTOR * floor + SLACK and rel(out, f_out) < VS_FP32_FACTOR * floor + SLACK
    assert set(grads) == set(e_grads)
    worst = 0.0
    for k in sorted(grads):
        ours_vs_eager, ours_vs_fp32, eager_vs_fp32 = rel(grads[k], e_grads[k]), rel(grads[k], f_grads[k]), rel(e_grads[k], f_grads[k])
        worst = max(worst, ours_vs_fp32 / max(eager_vs_fp32, 1e-12))
        assert ours_vs_eager < VS_EAGER_FACTOR * eager_vs_fp32 + SLACK, f"{k}: ours vs eager {ours_vs_eager}, floor {eager_vs_fp32}"
        assert ours_vs_fp32 < VS_FP32_FACTOR * eager_vs_fp32 + SLACK, (k, ours_vs_fp32, eager_vs_fp32)
    print(f"{name}: out vs eager {rel(out, e_out):.2e} (bf16 floor {floor:.2e}); worst grad err ratio {worst:.2f}")


def test_clip_vision_against_reference_golden_vectors():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "clip_vision_tiny_reference.pt"), weights_only=False)
    cfg = vo.vit_config(fx["config_name"])
    m = _clip_vision_module(cfg, vo.init_state_dict(cfg, seed=fx["weights_seed"]))
    out = m(fx["x"].to(DEV))
    (out.float() * fx["upstream"].to(DEV)).sum().backward()
    ref_bf16, ref_fp32 = fx["reference"]["bf16"], fx["reference"]["fp32"]
    assert rel(out.cpu(), ref_fp32["out"]) < max(2.0 * rel(ref_bf16["out"], ref_fp32["out"]), 5e-3)
    for k, p in m.named_parameters():
        ours = rel(golden_sample.take(p.grad, fx["grad_sample"][k]), ref_fp32["grads"][k])
        theirs = rel(ref_bf16["grads"][k], ref_fp32["grads"][k])
        assert ours < max(2.0 * theirs, 5e-3), (k, ours, theirs)


# ---- CLIP text tower stack: TeTEncoder (nlp/encoder/transformer.py) with the causal mask -----------------------------
@pytest.mark.parametrize("name,batch", [("clip_text_tiny", 3), ("clip_text_small", 4), ("clip_text", 8)])
def test_clip_text_stack_parity(name, batch):
    cfg = vo.tet_config(name)
    d, t = cfg["latent_dim"], cfg["context_length"]
    sd = vo.tet_init_state_dict(cfg, seed=0)
    m = registry.build_module("tet", config=dict(latent_dim=d, context_length=t, use_triu_attn_mask=True, num_layers=cfg["num_layers"],
                                                 norm_kwargs={"eps": cfg["eps"]}, attention_kwargs={"num_heads": d // 64},
                                                 feedforward_kwargs={"activation": "quick_gelu"}, head_pooler=None))
    assert list(m.state_dict().keys())[0] == "attention_mask"
    m.load_state_dict(sd, strict=False)
    m = m.to(DEV)
    g = torch.Generator().manual_seed(7)
    x = (torch.randn(batch, t, d, generator=g) * 0.5).to(DEV)
    up = torch.randn(batch, t, d, generator=g).to(DEV)
    xin = x.clone().requires_grad_(True)
    out = m(xin)
    assert out.dtype == torch.float32 and tuple(out.shape) == (batch, t, d)
    (out * up).sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    sdg = {k: v.to(DEV) for k, v in sd.items()}
    e_out, e_dx, e_grads = vo.tet_train_step(sdg, x, up, cfg, autocast_bf16=True)
    f_out, f_dx, f_grads = vo.tet_train_step(sdg, x, up, cfg, autocast_bf16=False)
    floor = rel(e_out, f_out)
    assert rel(out, e_out) < VS_EAGER_FACTOR * floor + SLACK and rel(out, f_out) < VS_FP32_FACTOR * floor + SLACK
    assert rel(xin.grad, e_dx) < VS_EAGER_FACTOR * rel(e_dx, f_dx) + SLACK and rel(xin.grad, f_dx) < VS_FP32_FACTOR * rel(e_dx, f_dx) + SLACK
    assert set(grads) == set(e_grads)
    worst = 0.0
    for k in sorted(grads):
        ours_vs_eager, ours_vs_fp32, eager_vs_fp32 = rel(grads[k], e_grads[k]), rel(grads[k], f_grads[k]), rel(e_grads[k], f_grads[k])
        worst = max(worst, ours_vs_fp32 / max(eager_vs_fp32, 1e-12))
        assert ours_vs_eager < VS_EAGER_FACTOR * eager_vs_fp32 + SLACK, f"{k}: ours vs eager {ours_vs_eager}, floor {eager_vs_fp32}"
        assert ours_vs_fp32 < VS_FP32_FACTOR * eager_vs_fp32 + SLACK, (k, ours_vs_fp32, eager_vs_fp32)
    print(f"{name}: out vs eager {rel(out, e_out):.2e} (bf16 floor {floor:.2e}); worst grad err ratio {worst:.2f}")


# ---- full CLIP: both towers + embedding / arg-max pooling / text_projection / l2-normalise / logits --------------------
def _clip_module(cfg, sd):
    v, t = cfg["vision"], cfg["text"]
    m = registry.build_module("clip", config=dict(
        img_size=v["img_size"], latent_dim=cfg["latent_dim"], in_channels=v["in_channels"], vision_latent_dim=v["latent_dim"],
        vision_patch_size=v["patch_size"], vision_num_heads=v["latent_dim"] // 64, vision_num_layers=v["num_layers"],
        vocab_size=cfg["vocab_size"], context_length=t["context_length"], text_latent_dim=t["latent_dim"],
        text_num_heads=t["latent_dim"] // 64, text_num_layers=t["num_layers"]))
    missing = m.load_state_dict(sd, strict=False)
    assert missing.missing_keys == ["text_transformer.attention_mask"] and not missing.unexpected_keys
    return m.to(DEV)


@pytest.mark.parametrize("name,batch", [("clip_tiny", 4), ("clip", 8)])
def test_clip_forward_backward_parity(name, batch):
    """``CLIP.forward`` (logits_per_image) and every parameter gradient for a seeded upstream gradient: ours vs the oracle
    eagerly on this GPU under bf16 autocast, both against the fp32 oracle.  The embedding gather / scatter and the arg-max
    pooling are integer-indexed copies: the gradient of the token embedding is non-zero on exactly the rows eager touches."""
    import clip_oracle as co

    cfg = co.clip_config(name)
    sd = co.init_state_dict(cfg, seed=0)
    x, ids = co.synthetic_batch(cfg, batch, seed=3)
    up = torch.randn(batch, batch, generator=torch.Generator().manual_seed(9))
    x, ids, up = x.to(DEV), ids.to(DEV), up.to(DEV)
    m = _clip_module(cfg, sd)
    logits = m(x, ids)
    assert logits.dtype == torch.bfloat16 and tuple(logits.shape) == (batch, batch)
    (logits.float() * up).sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    sdg = {k: v.to(DEV) for k, v in sd.items()}
    e_logits, e_grads = co.train_step(sdg, x, ids, up, cfg, autocast_bf16=True)
    f_logits, f_grads = co.train_step(sdg, x, ids, up, cfg, autocast_bf16=False)
    assert e_logits.dtype == torch.bfloat16
    floor = rel(e_logits, f_logits)
    assert rel(logits, e_logits) < VS_EAGER_FACTOR * floor + SLACK and rel(logits, f_logits) < VS_FP32_FACTOR * floor + SLACK
    assert set(grads) == set(e_grads)
    for k in sorted(grads):
        ours_vs_eager, ours_vs_fp32, eager_vs_fp32 = rel(grads[k], e_grads[k]), rel(grads[k], f_grads[k]), rel(e_grads[k], f_grads[k])
        assert ours_vs_eager < VS_EAGER_FACTOR * eager_vs_fp32 + SLACK, f"{k}: ours vs eager {ours_vs_eager}, floor {eager_vs_fp32}"
        assert ours_vs_fp32 < VS_FP32_FACTOR * eager_vs_fp32 + SLACK, (k, ours_vs_fp32, eager_vs_fp32)
    ge, ee = grads["token_embedding.weight"], e_grads["token_embedding.weight"]
    assert torch.equal(ge.abs().sum(1) > 0, ee.abs().sum(1) > 0) and ge[0].abs().sum().item() == 0.0  # padding row untouched
    # integer ops alone: gather and arg-max pooling are bit-exact copies
    from cflearn_b200.clip import _ArgmaxPoolFn, _EmbeddingFn

    w = sdg["token_embedding.weight"]
    assert torch.equal(_EmbeddingFn.apply(ids, w, 0), torch.nn.functional.embedding(ids, w))
    seq = torch.randn(batch, ids.shape[1], 64, device=DEV)
    assert torch.equal(_ArgmaxPoolFn.apply(seq, ids), seq[torch.arange(batch, device=DEV), ids.argmax(-1)])
    print(f"{name}: logits vs eager {rel(logits, e_logits):.2e} (bf16 floor {floor:.2e})")


@pytest.mark.parametrize("name,batch", [("clip_tiny", 6), ("clip", 16)])
def test_clip_train_step_symmetric_cross_entropy(name, batch):
    """The product-side CLIP step (VERDICT r1 item 6): ``CLIPB200.train_step`` = forward + symmetric cross-entropy + backward.
    Loss and all 303 parameter gradients against the oracle's definition of the same step (``clip_oracle.forward`` +
    ``symmetric_cross_entropy``) run eagerly on this GPU under bf16 autocast and in fp32; gradients land in the three
    flat arenas the optimizer / the data-parallel reducer work on."""
    import clip_oracle as co
    from cflearn_b200.optim import ArenaAdam

    cfg = co.clip_config(name)
    sd = co.init_state_dict(cfg, seed=0)
    x, ids = co.synthetic_batch(cfg, batch, seed=4)
    x, ids = x.to(DEV), ids.to(DEV)
    m = _clip_module(cfg, sd)
    loss = m.train_step(x, ids)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    sdg = {k: v.to(DEV) for k, v in sd.items()}

    def oracle(autocast):
        params = {k: v.detach().clone().requires_grad_(True) for k, v in sdg.items()}
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            lg = co.forward(params, x, ids, cfg)
            ls = co.symmetric_cross_entropy(lg)
        ls.backward()
        return ls.detach(), {k: v.grad for k, v in params.items()}

    e_loss, e_grads = oracle(True)
    f_loss, f_grads = oracle(False)
    assert abs(loss.item() - f_loss.item()) < 1.5 * abs(e_loss.item() - f_loss.item()) + 2e-3 * max(1.0, abs(f_loss.item())), (loss.item(), e_loss.item(), f_loss.item())
    assert set(grads) == set(e_grads)
    for k in sorted(grads):
        ours_vs_eager, ours_vs_fp32, eager_vs_fp32 = rel(grads[k], e_grads[k]), rel(grads[k], f_grads[k]), rel(e_grads[k], f_grads[k])
        assert ours_vs_eager < VS_EAGER_FACTOR * eager_vs_fp32 + SLACK, f"{k}: ours vs eager {ours_vs_eager}, floor {eager_vs_fp32}"
        assert ours_vs_fp32 < VS_FP32_FACTOR * eager_vs_fp32 + SLACK, (k, ours_vs_fp32, eager_vs_fp32)
    # the loose parameters' gradients were moved into the glue arena (what Adam and the all-reduce see)
    for k in ("logit_scale", "token_embedding.weight", "text_projection.weight", "text_projection.bias"):
        assert torch.equal(m.glue.g(k), grads[k]) and m.glue.params[k].grad.data_ptr() == m.glue.g(k).data_ptr()
    # one fused Adam step over the three arenas == torch.optim.Adam on the same gradients
    ref_params = [p.detach().clone().requires_grad_(True) for p in m.parameters()]
    for rp, p in zip(ref_params, m.parameters()):
        rp.grad = p.grad.clone()
    torch.optim.Adam(ref_params, lr=1e-3).step()
    ArenaAdam(m, lr=1e-3).step()
    torch.cuda.synchronize()
    for rp, p in zip(ref_params, m.parameters()):
        assert torch.allclose(rp, p, rtol=1e-5, atol=1e-7)
    print(f"{name}: loss ours {loss.item():.5f} eager {e_loss.item():.5f} fp32 {f_loss.item():.5f}")


def test_clip_graphed_train_step_matches_eager_steps():
    """The CUDA-graphed CLIP step (what `bench.py --config clip` times) reproduces eagerly launched steps."""
    import clip_oracle as co
    from cflearn_b200.optim import ArenaAdam, GraphedTrainStep

    cfg = co.clip_config("clip_tiny")
    sd = co.init_state_dict(cfg, seed=0)
    batches = [co.synthetic_batch(cfg, 6, seed=10 + i) for i in range(3)]
    eager, graphed = _clip_module(cfg, sd), _clip_module(cfg, sd)
    opt_e = ArenaAdam(eager, lr=1e-3)
    losses_e = []
    for x, ids in batches:
        opt_e.zero_grad()
        losses_e.append(eager.train_step(x.to(DEV), ids.to(DEV)).item())
        opt_e.step()
    opt_g = ArenaAdam(graphed, lr=1e-3, capturable=True)
    x0, i0 = batches[0]
    gs = GraphedTrainStep(graphed, opt_g, 6, warmup=2, inputs=[torch.zeros_like(x0, device=DEV), torch.zeros_like(i0, device=DEV)])
    losses_g = [gs.step(x.to(DEV), ids.to(DEV)).item() for x, ids in batches]
    torch.cuda.synchronize()
    for a, b in zip(losses_e, losses_g):
        assert abs(a - b) < 1e-4 * max(1.0, abs(a)), (losses_e, losses_g)
    for (k, p), (_, q) in zip(eager.named_parameters(), graphed.named_parameters()):
        assert torch.allclose(p, q, rtol=1e-4, atol=1e-6), k


def test_trainer_seam_matches_reference_update_sequence():
    """N2 (trainer seam): ``B200TrainStep`` = forward/loss/backward -> clip_norm_step -> optimizer.step -> zero_grad ->
    scheduler.step (cflearn/schema.py:977-986).  Three runs over the same batches must agree: (a) eager launches,
    (b) the whole step as ONE CUDA graph (clip coefficient and learning rate read from device memory), (c) our gradients fed
    to torch.nn.utils.clip_grad_norm_ + torch.optim.Adam + the same scheduler class."""
    from cflearn_b200.optim import ArenaAdam
    from cflearn_b200.trainer import B200TrainStep

    cfg = vo.vit_config("vit_tiny")
    sd = vo.init_state_dict(cfg, seed=0)
    batches = [vo.synthetic_batch(cfg, 4, seed=20 + i) for i in range(6)]
    sched = lambda opt: torch.optim.lr_scheduler.LambdaLR(opt, lambda k: 1.0 + 0.5 * min(k, 3) - 0.2 * max(k - 3, 0))  # noqa: E731 warm-up then decay
    clip = 0.05  # small enough to be active on these gradients

    def run(graph):
        m = build(cfg, sd)
        opt = ArenaAdam(m, lr=1e-3, capturable=True)
        step = B200TrainStep(m, opt, scheduler=sched(opt), clip_norm=clip, graph=graph, batch=4)
        losses = [step.step(x.to(DEV), y.to(DEV)).item() for x, y in batches]
        torch.cuda.synchronize()
        return m, losses

    m_e, l_e = run(False)
    m_g, l_g = run(True)
    for a, b in zip(l_e, l_g):
        assert abs(a - b) < 1e-5 * max(1.0, abs(a)), (l_e, l_g)
    for (k, p), (_, q) in zip(m_e.named_parameters(), m_g.named_parameters()):
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), k
    # (c) torch's clip_grad_norm_ + Adam + the same scheduler, fed the SAME gradient sequence in lock-step.  (Letting a second model
    # walk its own trajectory is ill-posed: after one step the parameters differ in the last bit, the next gradients by ~4e-5, and
    # Adam's m / sqrt(v) turns that into lr-sized differences on the few elements whose gradient is rounding noise --
    # tools/probe_trainer_seam.py.  With identical gradients only fp32 rounding of the update
    # arithmetic is left.)
    m_a = build(cfg, sd)
    o_a = ArenaAdam(m_a, lr=1e-3, capturable=True)
    s_a = B200TrainStep(m_a, o_a, scheduler=sched(o_a), clip_norm=clip)
    m_t = build(cfg, sd)
    named_t = dict(m_t.named_arena_parameters())
    params = list(named_t.values())
    topt = torch.optim.Adam(params, lr=1e-3)
    tsched = sched(topt)
    norms = []
    for x, y in batches:
        s_a.step(x.to(DEV), y.to(DEV))   # (the clip coefficient is applied inside the fused Adam: the arena keeps the raw gradient)
        for k, _ in m_a.named_arena_parameters():
            named_t[k].grad = m_a.arena.g(k).clone()
        norms.append(torch.nn.utils.clip_grad_norm_(params, clip).item())
        topt.step()
        tsched.step()
        for (k, pa), (_, pt) in zip(m_a.named_arena_parameters(), m_t.named_arena_parameters()):
            assert torch.allclose(pa, pt, rtol=1e-5, atol=2e-7), (k, (pa - pt).abs().max().item())
    assert max(norms) > clip  # clipping really happened
    for (k, pa), (_, pe) in zip(m_a.named_arena_parameters(), m_e.named_arena_parameters()):
        assert torch.allclose(pa, pe, rtol=1e-5, atol=1e-7), k  # and the lock-step run IS the eager run of (a)


def test_graphed_step_without_clipping_ignores_an_earlier_clipping_step():
    """A graphed ``B200TrainStep(clip_norm=0)`` on a model and optimizer that a clipping graphed step was built on before does
    not clip: its parameters equal, bit for bit, those of the same run on a fresh model and optimizer."""
    from cflearn_b200.optim import ArenaAdam
    from cflearn_b200.trainer import B200TrainStep

    cfg = vo.vit_config("vit_tiny")
    sd = vo.init_state_dict(cfg, seed=0)
    batches = [vo.synthetic_batch(cfg, 4, seed=20 + i) for i in range(3)]

    def run_unclipped(m, opt):
        step = B200TrainStep(m, opt, clip_norm=0.0, graph=True, batch=4)
        for x, y in batches:
            step.step(x.to(DEV), y.to(DEV))
        torch.cuda.synchronize()
        step.close()

    m = build(cfg, sd)
    opt = ArenaAdam(m, lr=1e-3, capturable=True)
    B200TrainStep(m, opt, clip_norm=0.05, graph=True, batch=4).close()  # its warm-up clips, then restores the state
    run_unclipped(m, opt)
    fresh = build(cfg, sd)
    run_unclipped(fresh, ArenaAdam(fresh, lr=1e-3, capturable=True))
    for (k, p), (_, q) in zip(m.named_parameters(), fresh.named_parameters()):
        assert torch.equal(p, q), k


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 64, 64, 320, 320), (2, 16, 16, 640, 1280)])
def test_unet_res_block_forward_matches_oracle(B, H, W, Cin, Cout):
    """SURVEY.md N3, first composed block: ResidualBlockWithTimeEmbedding forward on the native kernels (GroupNorm+SiLU, 3x3
    implicit-GEMM convolutions, time-embedding Linear, 1x1 shortcut as a GEMM) against oracle/unet_oracle.py::res_block run
    eagerly on this GPU under bf16 autocast and in fp32, at SD-v1.5 shapes (320 ch @ 64x64; the 640 -> 1280 block @ 16x16)."""
    import math

    import unet_oracle as uo
    from cflearn_b200.unet_blocks import res_block_forward

    g = torch.Generator().manual_seed(31)
    tdim = 1280
    shapes = [("b.norm1.weight", (Cin,)), ("b.norm1.bias", (Cin,)), ("b.conv1.weight", (Cout, Cin, 3, 3)), ("b.conv1.bias", (Cout,)),
              ("b.time_embedding.weight", (Cout, tdim)), ("b.time_embedding.bias", (Cout,)), ("b.norm2.weight", (Cout,)), ("b.norm2.bias", (Cout,)),
              ("b.conv2.weight", (Cout, Cout, 3, 3)), ("b.conv2.bias", (Cout,))]
    if Cin != Cout:
        shapes += [("b.shortcut.weight", (Cout, Cin, 1, 1)), ("b.shortcut.bias", (Cout,))]
    sd = {k: v.to(DEV) for k, v in uo.synthetic_state_dict(shapes, seed=2).items()}
    x = torch.randn(B, Cin, H, W, generator=g).to(DEV)
    tn = torch.randn(B, tdim, generator=g).to(DEV)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        xb = x.to(torch.bfloat16)  # the block's input is a bf16 conv output inside the UNet
        tb = tn.to(torch.bfloat16)
        e_out = uo.res_block(sd, "b.", xb, tb)
    f_out = uo.res_block(sd, "b.", x.to(torch.bfloat16).float(), tn.to(torch.bfloat16).float())
    ours = res_block_forward(sd, "b.", xb.permute(0, 2, 3, 1).contiguous(), tb)
    torch.cuda.synchronize()
    ours_nchw = ours.permute(0, 3, 1, 2)
    assert e_out.dtype == torch.bfloat16
    floor = rel(e_out, f_out)
    assert rel(ours_nchw, e_out) < VS_EAGER_FACTOR * floor + SLACK, (rel(ours_nchw, e_out), floor)
    assert rel(ours_nchw, f_out) < VS_FP32_FACTOR * floor + SLACK
    print(f"res_block {Cin}->{Cout} @ {H}x{W}: ours vs eager {rel(ours_nchw, e_out):.2e} (eager vs fp32 {floor:.2e})")
