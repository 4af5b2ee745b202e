"""The trainer seam: what replaces ``accelerator.prepare`` + the per-step update of the reference for the fused native modules.

In the reference one optimisation step is (``IDLModel.train``, cflearn/schema.py:1174-1294; ``get_update_fn``, :977-986):

    with autocast:  forward, loss                      schema.py:1260-1276
    accelerator.backward(loss)                         schema.py:980   (DDP's bucketed all-reduce hides in here)
    trainer.clip_norm_step()                           schema.py:982   (clip_grad_norm_ when clip_norm > 0)
    optimizer.step(); optimizer.zero_grad()            schema.py:983-984
    scheduler.step()                                   trainer.py (per step, after the optimizer)

``B200TrainStep`` runs the same sequence on a ``VanillaClassifierB200`` / ``CLIPB200``: the module's own fused
``train_step`` (forward + loss + backward, bucketed all-reduce on the native communicator inside backward), device-side
gradient clipping, the fused multi-arena Adam, and any ``torch.optim.lr_scheduler`` -- including the reference's default
``WarmupScheduler`` (cflearn/schedulers.py:126-171; pipeline/blocks/basic.py:334-352) -- driving the learning rate through
``optimizer.param_groups``.  With ``graph=True`` everything up to and including Adam is ONE CUDA graph; the scheduler's new
learning rate reaches the captured kernels through 24 bytes of device memory, never by re-capturing.

``grad_accumulate=K`` follows the reference's ``TrainerConfig.grad_accumulate`` (schema.py:1276-1290, 1888): backward runs
on every micro-batch and the update (clip, optimizer, scheduler) only on every K-th call, counting from the first; the
loss is not divided by K, so the update sees the sum of the K micro-batch gradients.  The gradients add up in place in
the arenas.  With a communicator they are exchanged once per window, by its last backward: that gives avg_r(sum_k g)
where DDP without ``no_sync`` gives sum_k avg_r(g) -- equal but for the order of the fp32 additions, and K - 1 fewer
exchanges per window.
"""
from __future__ import annotations

import contextlib
from typing import Any, List, Optional

import torch
from torch import Tensor

from . import dp
from .optim import ArenaAdam, GraphedTrainStep


class B200TrainStep:
    def __init__(self, model: Any, optimizer: ArenaAdam, *, scheduler: Any = None, clip_norm: float = 0.0, comm: Any = None,
                 graph: bool = False, batch: Optional[int] = None, static_inputs: Optional[List[Tensor]] = None, flat: bool = False,
                 grad_accumulate: int = 1):
        if grad_accumulate < 1:
            raise ValueError(f"grad_accumulate must be >= 1, got {grad_accumulate}")
        self.model, self.optimizer, self.scheduler = model, optimizer, scheduler
        self.clip_norm = float(clip_norm)
        self.comm = comm
        self.accumulate = int(grad_accumulate)
        self.steps = 0
        self.updated = False  # whether the last ``step`` ran the optimizer
        self._graph: Optional[GraphedTrainStep] = None
        if self.clip_norm > 0.0 and not optimizer.capturable:
            raise ValueError("clip_norm > 0 needs ArenaAdam(capturable=True)")
        if graph:
            if self.clip_norm > 0.0:
                # the clip coefficient is computed between backward and Adam: both live inside the captured step
                model.clip_norm_hook = lambda: optimizer.clip_grad_norm_(self.clip_norm)
            if batch is None and static_inputs is None:
                raise ValueError("graph=True needs the batch size (or the static input tensors)")
            self._graph = GraphedTrainStep(model, optimizer, batch or static_inputs[0].shape[0], comm=comm, inputs=static_inputs,
                                           flat=flat,  # flat: ONE all-reduce behind the graph instead of in-graph buckets
                                           grad_accumulate=self.accumulate)
        elif comm is not None and comm.world > 1:
            dp.attach_native_reducers(model, comm)

    def close(self) -> None:
        """Destroy the captured graph (must happen before the communicator it captured is closed)."""
        if self._graph is not None:
            self._graph.release()
            self._graph = None

    def step(self, *batch: Tensor) -> Tensor:
        """One micro-batch on ``batch`` (device tensors or pinned host tensors); returns its loss (device scalar).  Every
        ``grad_accumulate``-th call also updates the parameters; ``updated`` says whether this one did."""
        if self._graph is not None:
            loss = self._graph.step(*batch)
            self.updated = self._graph.updated
        else:
            first, self.updated = self.steps % self.accumulate == 0, (self.steps + 1) % self.accumulate == 0
            if first:
                self.optimizer.zero_grad()                  # schema.py:984 (moved to the front: the window's first backward overwrites the arena)
            with contextlib.nullcontext() if self.updated else dp.no_sync(self.model):
                loss = self.model.train_step(*batch)        # autocast forward + loss + accelerator.backward   schema.py:1266-1276,980
            if self.updated:
                if self.clip_norm > 0.0:
                    self.optimizer.clip_grad_norm_(self.clip_norm)  # trainer.clip_norm_step()                 schema.py:982
                self.optimizer.step()                       # schema.py:983
        if self.updated and self.scheduler is not None:
            self.scheduler.step()                           # writes optimizer.param_groups[0]["lr"]; reaches the device on the next step
        self.steps += 1
        return loss
