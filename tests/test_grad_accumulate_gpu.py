"""Gradient accumulation on the GPU: a backward adds to the gradient arenas in place while the parameters hold gradients,
and the trainer seam (``B200TrainStep`` / ``GraphedTrainStep`` with ``grad_accumulate=K``) updates once per K micro-batches.

Every gradient writer of the engines computes ``out = out + t`` with ``t`` the value an overwriting backward would store,
which is eager's ``p.grad += g``: so the accumulated arena equals g1 + g2 + g3, added in fp32 in that order, bit for bit.
The one exception is CLIP's token embedding: its gradient is summed with fp32 atomics (``b200_embedding_bwd``), so each
micro-batch's own gradient already varies in the order of its additions, and the sum can only match within that."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import clip_oracle as co  # noqa: E402
import vit_oracle as vo  # noqa: E402

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import _cabi, registry  # noqa: E402
from cflearn_b200.optim import ArenaAdam, GraphedTrainStep  # noqa: E402
from cflearn_b200.trainer import B200TrainStep  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
MIB = 1 << 20


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


def vit_model(sd, cfg):
    m = registry.build_module("cv_clf", config=dict(in_channels=cfg["in_channels"], num_classes=cfg["num_classes"],
                                                    img_size=cfg["img_size"], latent_dim=cfg["latent_dim"], encoder="vit",
                                                    encoder_config=dict(patch_size=cfg["patch_size"], num_layers=cfg["num_layers"])))
    m.load_state_dict(sd, strict=True)
    return m.to(DEV)


def clip_model(sd, cfg):
    v, t = cfg["vision"], cfg["text"]
    m = registry.build_module("clip", config=dict(
        img_size=v["img_size"], latent_dim=cfg["latent_dim"], in_channels=v["in_channels"], vision_latent_dim=v["latent_dim"],
        vision_patch_size=v["patch_size"], vision_num_heads=v["latent_dim"] // 64, vision_num_layers=v["num_layers"],
        vocab_size=cfg["vocab_size"], context_length=t["context_length"], text_latent_dim=t["latent_dim"],
        text_num_heads=t["latent_dim"] // 64, text_num_layers=t["num_layers"]))
    m.load_state_dict(sd, strict=False)
    return m.to(DEV)


def case(name, batch, n):
    """(model factory, n device batches) for the ViT classifier or CLIP."""
    if name == "vit":
        cfg = vo.vit_config("vit_tiny")
        sd = vo.init_state_dict(cfg, seed=0)
        batches = [vo.synthetic_batch(cfg, batch, seed=40 + i) for i in range(n)]
        make = lambda: vit_model(sd, cfg)  # noqa: E731
    else:
        cfg = co.clip_config("clip_tiny")
        sd = co.init_state_dict(cfg, seed=0)
        batches = [co.synthetic_batch(cfg, batch, seed=40 + i) for i in range(n)]
        make = lambda: clip_model(sd, cfg)  # noqa: E731
    return make, [tuple(t.to(DEV) for t in b) for b in batches]


def assert_sum(m, expected):
    """Every arena equals ``expected`` exactly, but CLIP's token embedding (fp32 atomics: see the module docstring)."""
    for a, want in zip(m.arenas(), expected):
        if "token_embedding.weight" not in a.params:
            assert torch.equal(a.grad, want), (a.grad - want).abs().max().item()
            continue
        for k in a.params:
            got, ref = a.g(k), a.view(want, k)
            if k == "token_embedding.weight":
                assert torch.allclose(got, ref, rtol=1e-5, atol=1e-6 * ref.abs().max().item()), rel(got, ref)
            else:
                assert torch.equal(got, ref), k


@pytest.mark.parametrize("name", ["vit", "clip"])
def test_accumulated_arena_is_the_fp32_sum_of_fresh_backwards(name):
    make, batches = case(name, 6, 3)
    m = make()
    fresh = []
    for b in batches:
        m.zero_grad(set_to_none=True)  # an overwriting backward
        m.train_step(*b)
        fresh.append([a.grad.clone() for a in m.arenas()])
    expected = [(g1 + g2) + g3 for g1, g2, g3 in zip(*fresh)]
    m.zero_grad(set_to_none=True)
    for b in batches:  # the first overwrites, the next two add in place
        m.train_step(*b)
    torch.cuda.synchronize()
    assert_sum(m, expected)
    for a in m.arenas():
        assert all(p.grad.data_ptr() == a.g(k).data_ptr() for k, p in a.params.items())
    # the graphed seam over one window: the arenas are zeroed, the three micro-steps add, the closing one also steps Adam
    # (which reads the gradients but leaves them in place)
    g = make()
    opt = ArenaAdam(g, lr=1e-3, capturable=True)
    seam = B200TrainStep(g, opt, graph=True, batch=6, static_inputs=[torch.zeros_like(t) for t in batches[0]], grad_accumulate=3)
    flags = []
    for b in batches:
        seam.step(*b)
        flags.append(seam.updated)
    torch.cuda.synchronize()
    assert flags == [False, False, True]
    assert_sum(g, expected)
    seam.close()


def test_accumulation_allocates_no_scratch_arena():
    make, batches = case("vit", 8, 2)
    m = make()
    assert not hasattr(m.arena, "grad_scratch")
    m.train_step(*batches[0])
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated()
    m.train_step(*batches[1])  # accumulates
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() - held < MIB, (torch.cuda.memory_allocated() - held) / MIB


def test_lock_step_with_torch_clip_adam_and_scheduler():
    """K = 3 over 9 micro-batches, clipping active, a LambdaLR schedule: our accumulated gradients fed to
    torch.nn.utils.clip_grad_norm_ + torch.optim.Adam + the same scheduler, stepped on the updates only, give the same
    parameters (tolerances of test_model_gpu.py::test_trainer_seam_matches_reference_update_sequence), the same learning
    rate after every micro-batch, and the same number of Adam steps."""
    make, batches = case("vit", 4, 9)
    lam = lambda k: 1.0 + 0.5 * min(k, 3) - 0.2 * max(k - 3, 0)  # noqa: E731
    clip = 0.05
    m_a = make()
    o_a = ArenaAdam(m_a, lr=1e-3, capturable=True)
    s_a = B200TrainStep(m_a, o_a, scheduler=torch.optim.lr_scheduler.LambdaLR(o_a, lam), clip_norm=clip, grad_accumulate=3)
    m_t = make()
    named_t = dict(m_t.named_arena_parameters())
    params = list(named_t.values())
    topt = torch.optim.Adam(params, lr=1e-3)
    tsched = torch.optim.lr_scheduler.LambdaLR(topt, lam)
    norms, updates = [], 0
    for i, (x, y) in enumerate(batches, 1):
        s_a.step(x, y)
        assert s_a.updated == (i % 3 == 0), i
        if s_a.updated:
            updates += 1
            for k, _ in m_a.named_arena_parameters():
                named_t[k].grad = m_a.arena.g(k).clone()
            norms.append(torch.nn.utils.clip_grad_norm_(params, clip).item())
            topt.step()
            tsched.step()
            for (k, pa), (_, pt) in zip(m_a.named_arena_parameters(), m_t.named_arena_parameters()):
                assert torch.allclose(pa, pt, rtol=1e-5, atol=2e-7), (i, k, (pa - pt).abs().max().item())
        assert o_a.lr == topt.param_groups[0]["lr"] == 1e-3 * lam(updates), (i, o_a.lr)
    assert max(norms) > clip  # clipping really happened
    assert int(o_a.step_dev.item()) == updates == 3
    assert all(int(topt.state[p]["step"]) == 3 for p in params)


def test_window_matches_oracle_sum_under_autocast():
    """One K = 2 window against the sum of the oracle's two micro-batch gradients, by test_train_step_parity's criterion."""
    cfg = vo.vit_config("vit_tiny")
    sd = vo.init_state_dict(cfg, seed=0)
    batches = [tuple(t.to(DEV) for t in vo.synthetic_batch(cfg, 4, seed=60 + i)) for i in range(2)]
    m = vit_model(sd, cfg)
    seam = B200TrainStep(m, ArenaAdam(m, lr=1e-3), grad_accumulate=2)
    for x, y in batches:
        seam.step(x, y)
    torch.cuda.synchronize()
    assert seam.updated
    ours = {k: p.grad for k, p in m.named_arena_parameters()}
    sdg = {k: v.to(DEV) for k, v in sd.items()}

    def oracle(autocast):
        out = {}
        for x, y in batches:
            for k, g in vo.train_step(sdg, x, y, cfg, autocast_bf16=autocast)[1].items():
                out[k] = g.float() if k not in out else out[k] + g.float()
        return out

    eager, exact = oracle(True), oracle(False)
    assert set(ours) == set(eager)
    for k in sorted(ours):
        floor = rel(eager[k], exact[k])
        assert rel(ours[k], eager[k]) < 2.0 * floor + 1e-3, (k, rel(ours[k], eager[k]), floor)
        assert rel(ours[k], exact[k]) < 1.5 * floor + 1e-3, (k, rel(ours[k], exact[k]), floor)


@pytest.mark.parametrize("name", ["vit", "clip"])
def test_eager_seam_equals_graphed_seam(name):
    make, batches = case(name, 6, 6)
    lam = lambda k: 1.0 / (1 + k)  # noqa: E731
    tol = dict(rtol=1e-5, atol=1e-7) if name == "vit" else dict(rtol=1e-4, atol=1e-6)  # test_model_gpu.py's per model

    def run(graph):
        m = make()
        opt = ArenaAdam(m, lr=1e-3, capturable=True)
        seam = B200TrainStep(m, opt, scheduler=torch.optim.lr_scheduler.LambdaLR(opt, lam), clip_norm=0.05 if name == "vit" else 0.0,
                             graph=graph, batch=6, static_inputs=[torch.zeros_like(t) for t in batches[0]], grad_accumulate=3)
        out = []
        for b in batches:
            out.append((seam.step(*b).item(), seam.updated, opt.lr))
        torch.cuda.synchronize()
        seam.close()
        return m, out

    m_e, out_e = run(False)
    m_g, out_g = run(True)
    assert [o[1:] for o in out_e] == [o[1:] for o in out_g] == [(i % 3 == 2, 1e-3 * lam((i + 1) // 3)) for i in range(6)]
    for (a, _, _), (b, _, _) in zip(out_e, out_g):
        assert abs(a - b) < tol["rtol"] * max(1.0, abs(a)), (out_e, out_g)
    for (k, p), (_, q) in zip(m_e.named_parameters(), m_g.named_parameters()):
        assert torch.allclose(p, q, **tol), k


def test_launches_k1_unchanged_and_k3_micro_step_has_no_adam():
    make, batches = case("vit", 4, 1)
    m = make()
    opt = ArenaAdam(m, lr=1e-3, capturable=True)
    opt.zero_grad()
    m.train_step(*batches[0])
    opt.step()
    torch.cuda.synchronize()
    n0 = _cabi.launch_count()
    opt.zero_grad()  # the step GraphedTrainStep(K = 1) captures: zero_grad, forward, loss, backward, Adam
    m.train_step(*batches[0])
    n1 = _cabi.launch_count()
    opt.step()
    torch.cuda.synchronize()
    step_launches, adam_launches = _cabi.launch_count() - n0, _cabi.launch_count() - n1
    m1 = make()
    g1 = GraphedTrainStep(m1, ArenaAdam(m1, capturable=True), 4)
    assert g1.launches_per_replay == step_launches and g1.micro_graph is None
    g1.release()
    m3 = make()
    g3 = GraphedTrainStep(m3, ArenaAdam(m3, capturable=True), 4, grad_accumulate=3)
    assert g3.launches_per_replay == step_launches  # closing step: the same launches
    assert g3.launches_per_micro_replay == step_launches - adam_launches  # micro-step: all but Adam's
    g3.release()


def test_graphed_accumulation_does_not_grow_peak_memory():
    """K = 4 keeps two graphs in ONE private pool: its peak allocation and the memory its graphs hold stay within 8 MiB of
    K = 1's (separate pools would hold the step's activations twice)."""
    make, batches = case("vit", 512, 1)

    def measure(K):
        m = make()
        opt = ArenaAdam(m, lr=1e-3, capturable=True)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base, r0 = torch.cuda.memory_allocated(), torch.cuda.memory_reserved()
        gs = GraphedTrainStep(m, opt, 512, grad_accumulate=K)
        for _ in range(2 * K):
            gs.step(*batches[0])
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        peak, held = torch.cuda.max_memory_allocated() - base, torch.cuda.memory_reserved() - r0
        gs.release()
        del gs, opt, m
        torch.cuda.empty_cache()
        return peak / MIB, held / MIB

    (p1, h1), (p4, h4) = measure(1), measure(4)
    print(f"peak MiB K=1 {p1:.1f} K=4 {p4:.1f}; held by the graphs K=1 {h1:.1f} K=4 {h4:.1f}")
    assert p4 <= p1 + 8.0, (p1, p4)
    assert h4 <= h1 + 8.0, (h1, h4)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_accumulation_matches_single_process():
    res = subprocess.run(
        [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
         "--master-port", "29534", os.path.join(ROOT, "tools", "dp_check.py"), "--grad-accumulate", "2"],
        stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert res.returncode == 0 and "dp_check: world 2" in res.stdout and "grad_accumulate 2" in res.stdout, res.stdout[-2000:]
