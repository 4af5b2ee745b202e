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
import math
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import torch
from torch import Tensor

from . import dp, ops
from ._cabi import B200Error
from .optim import ArenaAdam, GraphedTrainStep
from .vit import PREDICTIONS_KEY


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
            if batch is None and static_inputs is None:
                raise ValueError("graph=True needs the batch size (or the static input tensors)")
            self._graph = GraphedTrainStep(model, optimizer, batch or static_inputs[0].shape[0], comm=comm, inputs=static_inputs,
                                           flat=flat,  # flat: ONE all-reduce behind the graph instead of in-graph buckets
                                           grad_accumulate=self.accumulate, clip_norm=self.clip_norm)
        else:
            if self.clip_norm <= 0.0:
                optimizer.reset_grad_scale()
            if comm is not None and comm.world > 1:
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


# ---------------------------------------------------------------------------------------------------------------------
# evaluation
# ---------------------------------------------------------------------------------------------------------------------
def label_predictions(logits: Tensor, threshold: float = 0.5) -> Tensor:
    """The class each row of ``logits`` [B, C] predicts, by the rule of the reference's ``acc`` metric (``Accuracy.forward``,
    cflearn/metrics.py:34-52, through cftool's ``get_label_predictions``), as int64 [B]:
      - C > 2: the arg-max, with numpy's rules: the first index among ties, the first NaN in a row holding one;
      - C = 2: 1 where the fp32 difference ``l1 - l0`` exceeds ``log(threshold / (1 - threshold))``, else 0 (a NaN is 0);
      - C = 1: 1 where ``l0`` exceeds that logit threshold.
    bf16 values widen to fp32 exactly, so this is the reference's rule on its numpy copy of the same logits."""
    C = logits.shape[1]
    if C > 2:
        return torch.argmax(logits, 1)  # ATen's arg-max: NaN above every number, lower index first among equals
    z = logits[:, 1].float() - logits[:, 0].float() if C == 2 else logits[:, 0].float()
    return (z > math.log(threshold / (1.0 - threshold))).long()


def accumulate_batch(sums: Tensor, loss: Tensor, correct: Tensor, rows: Tensor, bad: Tensor) -> None:
    """``sums`` (float64 [3]) += (the batch's loss, its accuracy ``correct / rows``, its bad-label flag).  ``rows`` is a
    float64 tensor on ``sums``' device: divided by a host scalar, a CUDA division multiplies by the reciprocal instead,
    which is not numpy's correctly rounded quotient."""
    sums.add_(torch.stack([loss.reshape(()).double(), correct.reshape(()).double() / rows, bad.reshape(()).double()]))


def summarize(sums: List[float], batches: int) -> Dict[str, float]:
    """What ``DLInference.get_outputs`` reports for ``batches`` batches (cflearn/inference.py:175-198): each value's mean
    over the batches, ``sum(values) / len(values)`` -- the float64 sums in ``sums`` were added in batch order, as
    Python's ``sum`` adds.  Raises ``ValueError`` if a batch held a label outside [0, num_classes)."""
    loss_sum, acc_sum, bad = sums
    if bad != 0.0:
        raise ValueError("B200EvalStep: a label of an evaluated batch was outside [0, num_classes)")
    return {"loss": loss_sum / batches, "acc": acc_sum / batches}


class B200EvalStep:
    """The reference's validation pass (``IDLModel.evaluate`` -> ``DLInference.get_outputs`` with the loss as a metric,
    cflearn/schema.py:1296-1327) for a ``VanillaClassifierB200``, with the per-batch metric reduced on the device.

    ``step(x, y)`` runs the forward-only stack and the head (no activations kept), the fused cross-entropy (bit for bit the
    training loss) and the ``acc`` count (``label_predictions(logits) == labels``), and adds the batch's loss and accuracy
    to float64 accumulators on the device.  ``x``: fp32 [B, C, S, S] or RAW uint8 [B, S, S, C] (``model.set_input_pipeline``),
    ``y``: integer labels [B] or [B, 1], both on the GPU.  With ``graph=True`` a full batch of ``batch`` rows is one CUDA-graph
    replay (captured at the first such batch, again if the input dtype, the input pipeline or the parameter arena changes);
    a smaller batch -- a loader's last -- runs the same ops eagerly.  ``result()`` reads the accumulators once, returns
    ``{"loss": ..., "acc": ...}`` as ``get_outputs`` aggregates them (the mean over batches of per-batch values), and
    resets them.  ``metrics``: the reference's metric names; only ``"acc"`` (with its ``threshold``) is native."""

    def __init__(self, model: Any, *, batch: int, graph: bool = True, metrics: Union[str, Sequence[str]] = "acc",
                 threshold: float = 0.5):
        from .vit import VanillaClassifierB200

        for name in [metrics] if isinstance(metrics, str) else list(metrics):
            if name != "acc":
                raise NotImplementedError(f"B200EvalStep: metric {name!r} has no native implementation (native: 'acc' and the loss)")
        if not isinstance(model, VanillaClassifierB200):
            raise NotImplementedError(f"B200EvalStep evaluates VanillaClassifierB200, got {type(model).__name__}")
        if batch < 1:
            raise ValueError(f"batch must be >= 1, got {batch}")
        if not 0.0 < threshold < 1.0:
            raise ValueError(f"threshold must lie in (0, 1), got {threshold}")
        self.model, self.batch, self.graph, self.threshold = model, int(batch), bool(graph), float(threshold)
        self.batches = 0  # batches accumulated since the last result()
        self._sums: Optional[Tensor] = None
        self._graph: Optional[torch.cuda.CUDAGraph] = None
        self._key: Optional[Tuple[Any, ...]] = None
        self._x: Optional[Tensor] = None
        self._y: Optional[Tensor] = None
        self._rows: Optional[Tensor] = None

    def _check(self, x: Tensor, y: Tensor) -> Tensor:
        g = self.model.geo
        n = x.shape[0] if x.dim() == 4 else 0
        want = (n, g.img, g.img, g.cin) if x.dtype == torch.uint8 else (n, g.cin, g.img, g.img)
        if tuple(x.shape) != want or not 1 <= n <= self.batch or not (x.dtype == torch.uint8 or x.is_floating_point()):
            raise ValueError(f"B200EvalStep: x must be float [n, {g.cin}, {g.img}, {g.img}] or uint8 [n, {g.img}, {g.img}, {g.cin}] "
                             f"with 1 <= n <= {self.batch}, got {x.dtype} {list(x.shape)}")
        if y.dim() not in (1, 2) or y.shape[0] != n or y.numel() != n or y.is_floating_point() or y.is_complex() or y.dtype == torch.bool:
            raise ValueError(f"B200EvalStep: y must be integer labels [{n}] or [{n}, 1], got {y.dtype} {list(y.shape)}")
        if not x.is_cuda or not y.is_cuda or not next(iter(self.model.arena.params.values())).is_cuda:
            raise B200Error("B200EvalStep runs on CUDA only: the model, x and y must be on the GPU (there is no CPU fallback)")
        return y.reshape(-1).long()

    def _body(self, x: Tensor, labels: Tensor, sums: Tensor, rows: Tensor) -> None:
        with torch.no_grad():
            logits = self.model(x)[PREDICTIONS_KEY]
            loss, _, _, bad = ops.softmax_xent(logits, labels, need_grad=False)
            correct = (label_predictions(logits, self.threshold) == labels).sum()
            accumulate_batch(sums, loss, correct, rows, bad)

    def _capture(self, x: Tensor, key: Tuple[Any, ...]) -> None:
        self.close()
        dev = x.device
        self._x = torch.zeros(x.shape, dtype=torch.uint8 if x.dtype == torch.uint8 else torch.float32, device=dev)
        self._y = torch.zeros(self.batch, dtype=torch.int64, device=dev)
        rows = self._rows = torch.full((), float(self.batch), dtype=torch.float64, device=dev)  # read by every replay: kept alive
        # one eager pass on a side stream first (lazy initialisation stays out of the capture), into throw-away sums
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self._body(self._x, self._y, torch.zeros_like(self._sums), rows)
        torch.cuda.current_stream().wait_stream(s)
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph, capture_error_mode="thread_local"):
            self._body(self._x, self._y, self._sums, rows)
        self._key = key

    def step(self, x: Tensor, y: Tensor) -> None:
        """Evaluate one batch; nothing is read back to the host."""
        labels = self._check(x, y)
        if self._sums is None:
            self._sums = torch.zeros(3, dtype=torch.float64, device=x.device)
        if self.graph and x.shape[0] == self.batch:
            self.model.arena.ensure()
            key = (x.dtype == torch.uint8, self.model.arena.flat.data_ptr(), repr(self.model.engine.input_pipeline))
            if self._graph is None or key != self._key:
                self._capture(x, key)
            self._x.copy_(x, non_blocking=True)
            self._y.copy_(labels, non_blocking=True)
            self._graph.replay()
        else:
            self._body(x, labels, self._sums, torch.full((), float(x.shape[0]), dtype=torch.float64, device=x.device))
        self.batches += 1

    def result(self) -> Dict[str, float]:
        """``{"loss", "acc"}`` over the batches since the last call (one read from the device), then a reset."""
        if self.batches == 0 or self._sums is None:
            raise ValueError("B200EvalStep.result: no batch was evaluated since the last result()")
        sums, batches = self._sums.tolist(), self.batches
        self._sums.zero_()
        self.batches = 0
        return summarize(sums, batches)

    def close(self) -> None:
        """Destroy the captured graph (a later full batch captures a new one)."""
        if self._graph is not None:
            torch.cuda.synchronize()
            self._graph.reset()
            self._graph = None
