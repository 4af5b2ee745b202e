"""CPU tests of the trainer seam's gradient accumulation cadence (``B200TrainStep(..., grad_accumulate=K)``), with stand-ins
for the model, optimizer, scheduler and communicator that record what the seam calls.  The reference increments its step
counter before each step and updates when it is a multiple of K (cflearn/trainer.py:334, schema.py:1276-1290): with K = 3
backward runs on every micro-batch, and clipping, the optimizer, the scheduler and the gradient exchange on micro-batches
3, 6, 9, ... only."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import dp  # noqa: E402
from cflearn_b200.arena import ParamArena  # noqa: E402
from cflearn_b200.optim import GraphedTrainStep  # noqa: E402
from cflearn_b200.trainer import B200TrainStep  # noqa: E402


class _Comm:
    world = 2
    ctas = 0


class _Site:
    """An exchange site: its arena, its buckets and the reducer ``dp`` puts on it."""

    reducer = None
    shrink_next = 0

    def __init__(self):
        self.arena = ParamArena([("w", (4,))])
        self.arena.attach({"w": torch.nn.Parameter(torch.zeros(4))})

    def buckets(self):
        return {"stem": [["w"]]}


class _Model:
    """CLIP-shaped: an exchange site whose backward runs the bucket reducer, and loose parameters all-reduced through
    ``comm``."""

    def __init__(self, log):
        self.log, self.site, self.comm = log, _Site(), None

    def arenas(self):
        return [self.site.arena]

    def exchanges(self):
        return [self.site]

    def train_step(self, x):
        self.log.append(("backward", int(x)))
        if self.site.reducer is not None:
            self.log.append(("bucket_exchange", int(x)))
        if self.comm is not None:
            self.log.append(("glue_exchange", int(x)))
        return torch.tensor(float(x))


class _Opt:
    capturable = True

    def __init__(self, log):
        self.log = log

    def zero_grad(self):
        self.log.append(("zero_grad",))

    def clip_grad_norm_(self, max_norm):
        self.log.append(("clip",))

    def step(self):
        self.log.append(("step",))


class _Sched:
    def __init__(self, log):
        self.log = log

    def step(self):
        self.log.append(("sched",))


def _run(K, n, comm=None):
    log = []
    model = _Model(log)
    seam = B200TrainStep(model, _Opt(log), scheduler=_Sched(log), clip_norm=1.0, comm=comm, grad_accumulate=K)
    updated = []
    for i in range(1, n + 1):
        log.append(("call", i))
        assert seam.step(torch.tensor(i)).item() == i  # each call returns its own micro-batch's loss
        updated.append(seam.updated)
    return log, updated, model


def _calls_of(log):
    """{call index: [what ran during it]}"""
    out, cur = {}, None
    for e in log:
        if e[0] == "call":
            cur = out.setdefault(e[1], [])
        else:
            cur.append(e[0])
    return out


def test_k3_updates_clips_schedules_and_exchanges_every_site_on_every_third_micro_batch():
    log, updated, model = _run(3, 10, comm=_Comm())
    calls = _calls_of(log)
    assert [i for i, u in enumerate(updated, 1) if u] == [3, 6, 9]
    for i in range(1, 11):
        c = calls[i]
        assert c.count("backward") == 1, (i, c)
        update = i % 3 == 0
        for what in ("clip", "step", "sched", "bucket_exchange", "glue_exchange"):
            assert c.count(what) == int(update), (i, what, c)
        assert c.count("zero_grad") == int(i % 3 == 1), (i, c)  # once per window, before its first backward
        if update:
            assert c == ["backward", "bucket_exchange", "glue_exchange", "clip", "step", "sched"], c
    # the exchange is switched off only for the micro-steps: the reducer and the communicator are back afterwards
    assert model.site.reducer is not None and model.comm is not None


def test_k1_is_one_update_per_call_with_exchange_sites():
    log, updated, _ = _run(1, 3)
    assert updated == [True, True, True]
    calls = _calls_of(log)
    for i in range(1, 4):
        assert calls[i] == ["zero_grad", "backward", "clip", "step", "sched"], calls[i]
    log, _, _ = _run(1, 2, comm=_Comm())
    assert _calls_of(log)[2] == ["zero_grad", "backward", "bucket_exchange", "glue_exchange", "clip", "step", "sched"]


def test_no_sync_restores_every_exchange_site_after_an_error():
    model = _Model([])
    dp.attach_native_reducers(model, _Comm())
    red, comm = model.site.reducer, model.comm
    with pytest.raises(RuntimeError):
        with dp.no_sync(model):
            assert model.site.reducer is None and model.comm is None
            raise RuntimeError("backward failed")
    assert model.site.reducer is red and model.comm is comm


@pytest.mark.parametrize("K", [0, -1])
def test_grad_accumulate_below_one_is_refused(K):
    with pytest.raises(ValueError, match="grad_accumulate"):
        B200TrainStep(_Model([]), _Opt([]), grad_accumulate=K)
    with pytest.raises(ValueError, match="grad_accumulate"):
        GraphedTrainStep(_Model([]), _Opt([]), 4, grad_accumulate=K)
