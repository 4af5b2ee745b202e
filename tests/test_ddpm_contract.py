"""DDPMB200's host surface, checked without a GPU: the noise schedule against tables made by the reference's own code, the gradient arena's bucket layout,
the state_dict, the refusals, the argument contracts of b200_q_sample_pad_bf16 / b200_adamw_step / b200_adamw_step_dev (fake
pointers, never dereferenced: refused calls stop at the argument checks), and the UNet's bucket plan all-reduced over a world-2
gloo group."""
import json
import multiprocessing as mp
import os
import sys

import pytest
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cflearn_b200  # noqa: E402
from cflearn_b200 import _cabi, checkpoint, dp  # noqa: E402
from cflearn_b200.ddpm import DDPMB200, noise_tables  # noqa: E402
from cflearn_b200.optim import ArenaAdam, ArenaAdamW  # noqa: E402
from cflearn_b200.unet import bucket_plan  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
ARG, ALIGN = -1, -2
FAKE = 1 << 20


def _fixture(name):
    d = json.load(open(os.path.join(GOLDEN, name)))
    cfg = {k: tuple(v) if isinstance(v, list) else v for k, v in d["config"].items()}
    return cfg, d


def _ddpm(name, **kw):
    cfg, d = _fixture(name)
    cfg = dict(cfg)
    cin, cout = cfg.pop("in_channels"), cfg.pop("out_channels")
    return DDPMB200(64, cin, cout, use_spatial_transformer=True, **cfg, **kw), d


# ---- the noise schedule ---------------------------------------------------------------------------------------------------------------
# tests/golden/ddpm_noise_tables.pt: the reference's own DDPM._register_noise_schedule / make_beta_schedule
# (diffusion/ddpm.py:599-679, :51-84), imported through oracle/load_reference.py by tools/make_golden_ddpm_tables.py, rounded to
# fp32 as q_sample's .to(net) does.
TABLES = torch.load(os.path.join(GOLDEN, "ddpm_noise_tables.pt"))["cases"]


@pytest.mark.parametrize("case", TABLES, ids=lambda c: "{beta_schedule}-{timesteps}".format(**c["args"])
                         + ("-given" if "given_betas" in c["args"] else ""))
def test_noise_tables_are_the_references(case):
    kw = dict(case["args"])
    given = kw.pop("given_betas", None)
    a, s = noise_tables(given_betas=None if given is None else given.numpy(), **kw)
    assert a.dtype == torch.float32 and s.dtype == torch.float32
    assert torch.equal(a, case["sqrt_alphas_cumprod"]) and torch.equal(s, case["sqrt_one_minus_alphas_cumprod"])


def test_the_fixture_covers_every_schedule():
    assert {c["args"]["beta_schedule"] for c in TABLES if "given_betas" not in c["args"]} == {"linear", "cosine", "sqrt_linear", "sqrt"}
    assert any("given_betas" in c["args"] and c["sqrt_alphas_cumprod"].shape == (250,) for c in TABLES)


def test_unknown_schedule_raises():
    with pytest.raises(ValueError, match="unrecognized schedule"):
        noise_tables(10, None, "quadratic")


# ---- refusals ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,option", [
    (dict(parameterization="x0"), "parameterization"), (dict(parameterization="v"), "parameterization"),
    (dict(learn_log_var=True), "learn_log_var"), (dict(ema_decay=0.999), "ema_decay"), (dict(condition_model="clip"), "condition_model"),
])
def test_ddpm_refusals_name_the_option(kw, option):
    with pytest.raises(NotImplementedError, match=option):
        _ddpm("unet_small64_state_dict_keys.json", **kw)


def test_forward_refuses_a_cpu_latent():
    m, _ = _ddpm("unet_small64_state_dict_keys.json")
    with pytest.raises(cflearn_b200.B200Error, match="CUDA fp32 latent"):
        m.train_step(torch.zeros(1, 4, 8, 8))


# ---- the arena ----------------------------------------------------------------------------------------------------------------------
def _check_layout(m):
    plan = bucket_plan(m.unet)
    names = [n for n, _ in m.unet.named_parameters()]
    keys = [k for _, ks in plan for k in ks]
    assert sorted(keys) == sorted(names) and len(set(keys)) == len(keys)  # every parameter in exactly one bucket
    n_out, n_in = len(m.unet.output_blocks), len(m.unet.input_blocks)
    assert [b for b, _ in plan] == (["head"] + [f"output_blocks.{i}" for i in reversed(range(n_out))] + ["residual"]
                                    + [f"input_blocks.{i}" for i in reversed(range(1, n_in))] + ["stem"])
    assert all(k.startswith(("input_blocks.0.", "time_embedding.")) for k in dict(plan)["stem"])
    A = m.arena
    spans = [A.span(ks) for _, ks in plan]
    assert spans[0][0] == 0 and spans[-1][1] == A.total
    assert all(hi == lo for (_, hi), (lo, _) in zip(spans, spans[1:]))  # contiguous, disjoint, in backward order
    for _, ks in plan:  # inside a bucket: the keys in layout order, each view where its offset says
        offs = [A.offsets[k] for k in ks]
        assert offs == sorted(offs)
    return plan


def test_arena_layout_at_sd_v1_5():
    with torch.device("meta"):
        m, d = _ddpm("unet_sd_v1_5_state_dict_keys.json")
    plan = _check_layout(m)
    assert len(plan) == 26
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == [["unet." + k, s] for k, s in d["keys"]]
    assert sum(p.numel() for p in m.parameters()) == d["num_params"] == 859520964


def test_arena_small_config_views_and_strict_loading():
    m, d = _ddpm("unet_small64_state_dict_keys.json")
    _check_layout(m)
    A = m.arena
    assert A.flat is None and A.grad is None  # nothing allocated until the arena is first used
    A.ensure()
    for k, p in m.unet.named_parameters():
        assert p.data_ptr() == A.flat.data_ptr() + 4 * A.offsets[k], k
        slot = getattr(p, checkpoint.SLOT_ATTR)
        assert slot.arena is A and slot.key == k
    assert A.flat_bf16 is None
    g = torch.Generator().manual_seed(0)
    sd = {"unet." + k: torch.randn(shape, generator=g) for k, shape in d["keys"]}
    m.load_state_dict(sd, strict=True)  # copies into the arena views
    assert all(torch.equal(m.state_dict()[k], v) for k, v in sd.items())
    back, _ = _ddpm("unet_small64_state_dict_keys.json")
    back.load_state_dict(m.state_dict(), strict=True)
    assert list(back.state_dict()) == list(sd)
    m.grad_arena.close()
    assert not any(hasattr(p, checkpoint.SLOT_ATTR) for p in m.parameters())


def test_bucket_counters_fire_once_per_backward():
    fired = []
    b = checkpoint.Bucket("x", 5, fired.append)
    for n in (2, 2, 1):
        b.done(n)
    assert fired == ["x"] and b.left == 0
    b.done(1)  # a gradient written twice: no second hand-over, and the count shows it
    assert fired == ["x"] and b.left == -1
    b.reset()
    assert b.left == 5


def _complete(m, skip=()):
    for name, keys in bucket_plan(m.unet):
        n = sum(m.unet.get_parameter(k).requires_grad for k in keys)
        if name not in skip and n:
            m.grad_arena._buckets[name].done(n)


def test_check_refuses_a_skipped_or_repeated_exchange():
    m, _ = _ddpm("unet_small64_state_dict_keys.json")
    ga = m.grad_arena
    ga.begin()
    _complete(m)
    ga.check()
    ga.begin()
    _complete(m, skip={"residual"})
    with pytest.raises(cflearn_b200.B200Error, match="residual"):
        ga.check()
    ga.begin()
    _complete(m)
    _complete(m)  # two backwards after one forward
    with pytest.raises(cflearn_b200.B200Error, match="not completed exactly once"):
        ga.check()
    # a frozen parameter's op writes no gradient: its bucket waits only for the trainable ones
    m.unet.head[2].weight.requires_grad_(False)
    ga.begin()
    _complete(m)
    ga.check()
    assert ga._buckets["head"].size == len(dict(bucket_plan(m.unet))["head"]) - 1


def test_optimizers_and_dp_accept_the_module_through_its_grad_arena():
    m, _ = _ddpm("unet_small64_state_dict_keys.json")
    opt = ArenaAdamW(m, lr=1e-4)
    assert opt.weight_decay == 0.01 and opt.decoupled and not ArenaAdam.decoupled
    assert opt.arenas() == [m.arena]
    dp.detach_reducers(m)
    assert m.grad_arena.reducer is None
    with dp.no_sync(m):
        assert m.grad_arena.reducer is None


# ---- the three entries' argument contracts ----------------------------------------------------------------------------------------------
def _status(name, *args):
    rc = getattr(_cabi.lib(), name)(*args)
    return rc, _cabi.last_error()


@pytest.mark.parametrize("kw,code,text", [
    (dict(B=0), ARG, "non-positive size"), (dict(C=0), ARG, "non-positive size"), (dict(H=0), ARG, "non-positive size"),
    (dict(T=0), ARG, "non-positive size"), (dict(Cp=60), ARG, "multiple of 8"), (dict(C=65), ARG, "at most Cp"),
    (dict(cl=2), ARG, "flags"), (dict(B=1, C=1, H=46341, W=46341, Cp=8), ARG, "H * W"),
    (dict(B=1 << 22, H=1 << 10, W=1 << 10), ARG, "too many"),
    (dict(x0=None), ARG, "null pointer"), (dict(noise=None), ARG, "null pointer"), (dict(t=None), ARG, "null pointer"),
    (dict(a=None), ARG, "null pointer"), (dict(s=None), ARG, "null pointer"), (dict(bad=None), ARG, "null pointer"),
    (dict(out=None), ARG, "null pointer"), (dict(x0=FAKE + 2), ALIGN, "element size"), (dict(noise=FAKE + 2), ALIGN, "element size"),
    (dict(t=FAKE + 4), ALIGN, "element size"), (dict(a=FAKE + 1), ALIGN, "element size"), (dict(bad=FAKE + 2), ALIGN, "element size"),
    (dict(out=FAKE + 8), ALIGN, "16-byte aligned"),
])
def test_q_sample_pad_refusals(kw, code, text):
    a = dict(x0=FAKE, noise=FAKE, cl=0, t=FAKE, a=FAKE, s=FAKE, T=1000, bad=FAKE, out=FAKE, B=2, C=4, H=8, W=8, Cp=64)
    a.update(kw)
    rc, msg = _status("b200_q_sample_pad_bf16", a["x0"], a["noise"], a["cl"], a["t"], a["a"], a["s"], a["T"], a["bad"], a["out"], a["B"],
                      a["C"], a["H"], a["W"], a["Cp"], None)
    assert rc == code and text in msg and "q_sample_pad" in msg, (rc, msg)


@pytest.mark.parametrize("kw,code,text", [
    (dict(n=0), ARG, "multiple of 4"), (dict(n=6), ARG, "multiple of 4"), (dict(step=0), ARG, "step >= 1"),
    (dict(p=None), ARG, "null pointer"), (dict(g=None), ARG, "null pointer"), (dict(m=None), ARG, "null pointer"),
    (dict(v=None), ARG, "null pointer"), (dict(p=FAKE + 8), ALIGN, "16-byte"), (dict(v=FAKE + 4), ALIGN, "16-byte"),
    (dict(sd=FAKE + 2), ALIGN, "step_dev"),
])
def test_adamw_step_refusals(kw, code, text):
    a = dict(p=FAKE, g=FAKE, m=FAKE, v=FAKE, n=4096, step=1, sd=None)
    a.update(kw)
    rc, msg = _status("b200_adamw_step", a["p"], a["g"], a["m"], a["v"], a["n"], 1e-3, 0.9, 0.999, 1e-8, 1e-2, a["step"], a["sd"], None)
    assert rc == code and text in msg and "adamw_step" in msg, (rc, msg)


@pytest.mark.parametrize("kw,code,text", [
    (dict(n=-4), ARG, "multiple of 4"), (dict(n=10), ARG, "multiple of 4"), (dict(p=None), ARG, "null pointer"),
    (dict(h=None), ARG, "null pointer"), (dict(sd=None), ARG, "null pointer"), (dict(g=FAKE + 4), ALIGN, "16-byte"),
    (dict(h=FAKE + 2), ALIGN, "hyper_dev"), (dict(sd=FAKE + 1), ALIGN, "hyper_dev / step_dev"),
])
def test_adamw_step_dev_refusals(kw, code, text):
    a = dict(p=FAKE, g=FAKE, m=FAKE, v=FAKE, n=4096, h=FAKE, sd=FAKE)
    a.update(kw)
    rc, msg = _status("b200_adamw_step_dev", a["p"], a["g"], a["m"], a["v"], a["n"], a["h"], a["sd"], 1, None)
    assert rc == code and text in msg and "adamw_step_dev" in msg, (rc, msg)


# ---- the bucket plan over a world-2 gloo group ------------------------------------------------------------------------------------------
def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.manual_seed(rank)  # different replicas until the broadcast
        m, _ = _ddpm("unet_small64_state_dict_keys.json")
        dp.broadcast_parameters(m)
        red = dp.GradBucketReducer(m.arena, m.grad_arena.buckets())
        m.grad_arena.reducer = red
        # every parameter's gradient as its backward would leave it: rank r writes (r + 1) x its flat index, bucket by bucket
        idx = torch.arange(m.arena.total, dtype=torch.float32)
        for name, keys in bucket_plan(m.unet):
            lo, hi = m.arena.span(keys)
            m.arena.grad[lo:hi] = idx[lo:hi] * (rank + 1)
            m.grad_arena._buckets[name].done(len(keys))
        red.finish()
        q.put((rank, m.arena.flat.numpy().copy(), m.arena.grad.numpy().copy()))  # by value: the worker exits
    finally:
        dist.destroy_process_group()


def test_world2_gloo_grad_arena_buckets_average_the_arena():
    world, port = 2, 29581
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, f0, g0), (_, f1, g1) = [(r, torch.from_numpy(f), torch.from_numpy(g)) for r, f, g in sorted(results, key=lambda t: t[0])]
    assert torch.equal(f0, f1)
    expect = torch.arange(g0.numel(), dtype=torch.float32) * 1.5
    assert torch.equal(g0, g1) and torch.allclose(g0, expect)
