"""Fused Adam over the flat parameter / gradient arenas, and a CUDA-graph wrapper for the whole training step.

``ArenaAdam`` mirrors ``torch.optim.Adam`` (the reference's default optimizer ``"adam"``, cflearn/optimizers.py:29-32,
built by BuildOptimizersBlock at cflearn/pipeline/blocks/basic.py:385-558 and stepped in cflearn/schema.py:983-984):
one kernel per step instead of one per tensor.  With ``capturable=True`` the step counter AND every hyper-parameter
live on the device, so the update can be replayed from a CUDA graph while a scheduler keeps changing the learning rate
(``param_groups[0]["lr"]`` is what ``torch.optim.lr_scheduler`` classes write; the reference's default scheduler is
``warmup``, basic.py:334-352).

``GraphedTrainStep`` captures ``zero_grad -> forward -> cross-entropy -> backward -> bucketed gradient all-reduce ->
Adam`` (IDLModel.train, cflearn/schema.py:1174-1294, minus its per-step host work) into ONE CUDA graph.  With more
than one rank the all-reduces are nodes of the same graph: each transformer block's bucket is reduced on a forked
communication stream through the library's own NCCL communicator (``dp.NativeComm``) while the backward of the
earlier blocks is still running.  With gradient accumulation over K micro-batches it captures two graphs in one memory
pool: a micro-step (forward, loss, backward adding to the gradient arenas) and the window's closing step (the same, then
the exchange, clipping and Adam).
"""
from __future__ import annotations

import contextlib
from typing import Any, Dict, List, Optional

import torch
from torch import Tensor

from . import ops


class ArenaAdam(torch.optim.Optimizer):
    """A real ``torch.optim.Optimizer`` (so ``torch.optim.lr_scheduler`` classes -- and the reference's own ``WarmupScheduler``,
    cflearn/schedulers.py:126-171 -- accept it), with ONE parameter group holding every parameter of the module's arenas."""

    decoupled = False  # weight decay as an L2 term in the gradient (torch.optim.Adam)

    def __init__(self, module: Any, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0,
                 capturable: bool = False):
        self.module = module
        self.capturable = capturable
        super().__init__(list(module.parameters()), dict(lr=float(lr), betas=tuple(betas), eps=float(eps), weight_decay=float(weight_decay),
                                                         grad_scale=1.0))
        self.step_count = 0
        self.step_dev: Optional[Tensor] = None
        self.hyper_dev: Optional[Tensor] = None
        self._hyper_host: Optional[Tensor] = None
        self._hyper_events: List[Any] = []
        self._hyper_slot = -1
        self._hyper_sent: Optional[tuple] = None
        self._clip_dev: Optional[Tensor] = None  # when set: grad_scale lives on the device only (clip_grad_norm_)
        # one (exp_avg, exp_avg_sq) pair per parameter arena: a ViT / classifier has one arena, CLIP three (vision tower,
        # text tower, and the loose parameters: logit_scale, token embedding, text projection)
        self.exp_avgs: List[Tensor] = []
        self.exp_avg_sqs: List[Tensor] = []

    def arenas(self) -> List[Any]:
        return self.module.arenas()

    @property
    def exp_avg(self) -> Optional[Tensor]:
        return self.exp_avgs[0] if self.exp_avgs else None

    @property
    def exp_avg_sq(self) -> Optional[Tensor]:
        return self.exp_avg_sqs[0] if self.exp_avg_sqs else None

    # ---- hyper-parameters ---------------------------------------------------------------------------------------
    @property
    def lr(self) -> float:
        return self.param_groups[0]["lr"]

    @lr.setter
    def lr(self, value: float) -> None:
        self.param_groups[0]["lr"] = float(value)

    def set_lr(self, value: float) -> None:
        self.lr = value

    @property
    def betas(self):
        return self.param_groups[0]["betas"]

    @property
    def eps(self) -> float:
        return self.param_groups[0]["eps"]

    @property
    def weight_decay(self) -> float:
        return self.param_groups[0]["weight_decay"]

    def _hyper_tuple(self) -> tuple:
        g = self.param_groups[0]
        return (float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]), float(g["weight_decay"]),
                float(g.get("grad_scale", 1.0)))

    def sync_hyper(self) -> None:
        """Push the current ``param_groups`` values to the device buffer the captured kernels read (24 bytes, only when
        something changed; pinned source, asynchronous on the current stream, ordered before the next replay)."""
        if self.hyper_dev is None:
            return
        cur = self._hyper_tuple()
        if cur == self._hyper_sent:
            return
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("ArenaAdam.sync_hyper() must run outside the capture (it is a host-to-device copy of new values)")
        # the copy is asynchronous: a pinned row may only be rewritten once the copy that read it has run (the host can be
        # many replays ahead of the device), so the rows form a ring and each carries the event of its last copy
        slot = self._hyper_slot = (self._hyper_slot + 1) % self._hyper_host.shape[0]
        if self._hyper_events[slot] is not None:
            self._hyper_events[slot].synchronize()
        row = self._hyper_host[slot]
        row.copy_(torch.tensor(cur, dtype=torch.float32))
        n = 5 if self._clip_dev is not None else 6  # with clipping on, slot 5 (grad_scale) is written on the device every step
        self.hyper_dev[:n].copy_(row[:n], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._hyper_events[slot] = ev
        self._hyper_sent = cur

    # ---- state --------------------------------------------------------------------------------------------------
    def _state(self) -> None:
        arenas = self.arenas()
        for a in arenas:
            a.ensure()
        dev = arenas[0].flat.device
        if not self.exp_avgs or self.exp_avgs[0].device != dev or len(self.exp_avgs) != len(arenas):
            self.exp_avgs = [torch.zeros_like(a.flat) for a in arenas]
            self.exp_avg_sqs = [torch.zeros_like(a.flat) for a in arenas]
            if self.capturable:
                self.step_dev = torch.full((1,), self.step_count, dtype=torch.int32, device=dev)
                self.hyper_dev = torch.zeros(6, dtype=torch.float32, device=dev)
                self._hyper_host = torch.zeros(8, 6, dtype=torch.float32).pin_memory()
                self._hyper_events = [None] * 8
                self._hyper_slot = -1
                self._hyper_sent = None
        if self.capturable and not torch.cuda.is_current_stream_capturing():
            self.sync_hyper()

    def state_tensors(self) -> List[Tensor]:
        """Everything a step mutates besides the gradients: parameters, moments, the device step counter."""
        self._state()
        out = [a.flat for a in self.arenas()] + self.exp_avgs + self.exp_avg_sqs
        if self.step_dev is not None:
            out.append(self.step_dev)
        return out

    @torch.no_grad()
    def step(self, closure: Any = None) -> None:  # type: ignore[override]
        """One Adam update of every arena (one launch per arena; the step counter advances once)."""
        self._state()
        if not self.capturable:
            self.step_count += 1
            lr, b1, b2, eps, wd, gs = self._hyper_tuple()
            if gs != 1.0:
                raise ValueError("grad_scale needs ArenaAdam(capturable=True)")
        for idx, a in enumerate(self.arenas()):
            if self.capturable:
                ops.adam_step(a.flat, a.grad, self.exp_avgs[idx], self.exp_avg_sqs[idx], hyper_dev=self.hyper_dev, step_dev=self.step_dev,
                              increment=idx == 0, decoupled=self.decoupled)
            else:
                ops.adam_step(a.flat, a.grad, self.exp_avgs[idx], self.exp_avg_sqs[idx], hyper=(lr, b1, b2, eps, wd), step=self.step_count,
                              decoupled=self.decoupled)

    def zero_grad(self, set_to_none: bool = True) -> None:
        if set_to_none:
            for p in self.module.parameters():
                p.grad = None

    def clip_grad_norm_(self, max_norm: float) -> Tensor:
        """``trainer.clip_norm_step()`` (cflearn/schema.py:981; torch.nn.utils.clip_grad_norm_ over all parameters) without a
        host round trip: the global L2 norm of the flat gradient arenas is taken on the device and the coefficient
        ``min(1, max_norm / (norm + 1e-6))`` goes straight into the ``grad_scale`` slot the fused Adam kernel multiplies the
        gradient by -- capturable in the step's CUDA graph.  Returns the norm (device scalar)."""
        if not self.capturable:
            raise ValueError("clip_grad_norm_ needs ArenaAdam(capturable=True) (the coefficient stays on the device)")
        self._state()
        sq = None
        for a in self.arenas():
            t = torch.linalg.vector_norm(a.grad) ** 2
            sq = t if sq is None else sq + t
        norm = sq.sqrt()
        self._clip_dev = (float(max_norm) / (norm + 1e-6)).clamp(max=1.0)
        self.hyper_dev[5:6].copy_(self._clip_dev.reshape(1))
        return norm

    def reset_grad_scale(self) -> None:
        """For steps that do not clip after steps that did: ``clip_grad_norm_`` left its last coefficient in the device's
        ``grad_scale`` slot, so hand the slot back to the host's value (1), which the next ``sync_hyper`` writes."""
        if self._clip_dev is not None:
            self._clip_dev = None
            self._hyper_sent = None

    def state_dict(self) -> Dict[str, Any]:
        step = int(self.step_dev.item()) if self.step_dev is not None else self.step_count
        g = self.param_groups[0]
        return {"step": step, "exp_avg": list(self.exp_avgs), "exp_avg_sq": list(self.exp_avg_sqs), "lr": g["lr"],
                "betas": g["betas"], "eps": g["eps"], "weight_decay": g["weight_decay"]}

    def load_state_dict(self, sd: Dict[str, Any]) -> None:
        self._state()
        g = self.param_groups[0]
        for k in ("lr", "betas", "eps", "weight_decay"):
            if k in sd:
                g[k] = tuple(sd[k]) if k == "betas" else float(sd[k])
        with torch.no_grad():
            for name, mine in (("exp_avg", self.exp_avgs), ("exp_avg_sq", self.exp_avg_sqs)):
                src = sd.get(name)
                src = [src] if isinstance(src, Tensor) else src
                for i, t in enumerate(mine):
                    if src is not None and i < len(src) and src[i] is not None:
                        t.copy_(src[i].to(t.device))
                    else:
                        t.zero_()
            self.step_count = int(sd.get("step", 0))
            if self.step_dev is not None:
                self.step_dev.fill_(self.step_count)
        if self.capturable:
            self.sync_hyper()


class ArenaAdamW(ArenaAdam):
    """``torch.optim.AdamW`` (the zoo's DDPM optimizer ``"adamw"``, cflearn/optimizers.py:31; weight decay 0.01 by default) on
    the arenas: the same fused kernels with decoupled decay, p <- p (1 - lr weight_decay) before the Adam update."""

    decoupled = True

    def __init__(self, module: Any, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2,
                 capturable: bool = False):
        super().__init__(module, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, capturable=capturable)


class GraphedTrainStep:
    """Whole training step of a B200 module (an ``arena.ArenaModule``: ``VanillaClassifierB200``, ``CLIPB200``, ``DDPMB200``)
    as one CUDA graph with static input / loss buffers.

    ``step(*inputs)`` copies the batch into the static buffers (device->device or pinned-host->device, on the current
    stream), replays the graph and returns the static loss tensor (fp32 scalar, on the device).  The warm-up runs needed
    before the capture leave NO trace: parameters, Adam moments and the step counter are restored.

    Data parallel (``comm``: a ``dp.NativeComm``): the graph also holds the gradient exchange -- the model's bucket
    reducers launch ``ncclAllReduce`` per transformer block on a forked stream as soon as that block's gradients are
    complete -- and the Adam update behind the join.  ``inputs``: the static input tensors (default: an image batch
    [batch, C, S, S] fp32 and int64 labels [batch, 1] for the classifier).  ``clip_norm > 0``: the exchanged gradients are
    clipped to that global L2 norm before Adam (``ArenaAdam.clip_grad_norm_``, in the graph).

    ``grad_accumulate=K``: one optimizer update per K calls of ``step`` (the reference's ``TrainerConfig.grad_accumulate``).
    Every call runs forward, loss and a backward that adds to the gradient arenas, which are zeroed (one ``fill`` launch per
    arena) before a window's first call; the K-th call also exchanges the summed gradients, clips them and steps Adam.
    ``updated`` says whether the last call did.  K = 1 is the single graph described above."""

    def __init__(self, model: Any, optimizer: ArenaAdam, batch: int, warmup: int = 2, comm: Any = None, flat: bool = False,
                 inputs: Optional[List[Tensor]] = None, grad_accumulate: int = 1, clip_norm: float = 0.0):
        if grad_accumulate < 1:
            raise ValueError(f"grad_accumulate must be >= 1, got {grad_accumulate}")
        if not optimizer.capturable:
            raise ValueError("GraphedTrainStep needs ArenaAdam(capturable=True)")
        from . import _cabi, dp

        self.world = 1 if comm is None else comm.world
        self.comm = comm
        self.accumulate = int(grad_accumulate)
        self.clip_norm = float(clip_norm)
        self.micro = 0  # calls of the current window so far
        self.updated = False
        # flat=True (A/B switch): the graph stops after backward; ONE all-reduce per gradient arena and Adam are
        # enqueued behind every replay -- the un-overlapped schedule
        self.flat = bool(flat) and self.world > 1
        self.model, self.optimizer = model, optimizer
        arenas = optimizer.arenas()
        for a in arenas:
            a.ensure()
        dev = arenas[0].flat.device
        if self.clip_norm <= 0.0:
            optimizer.reset_grad_scale()
        if self.flat or self.world == 1:
            dp.detach_reducers(model)
        else:
            dp.attach_native_reducers(model, comm)
        if inputs is None:
            g = model.geo
            inputs = [torch.zeros((batch, g.cin, g.img, g.img), dtype=torch.float32, device=dev),
                      torch.zeros((batch, 1), dtype=torch.int64, device=dev)]
        self.inputs = inputs
        self.x, self.labels = inputs[0], inputs[-1]
        self.loss = torch.zeros((), dtype=torch.float32, device=dev)
        self.bad_label = torch.zeros(1, dtype=torch.int32, device=dev)
        if self.accumulate > 1:  # every backward from here on adds to the arenas, the captured ones included
            for a in arenas:
                a.publish_grads(list(a.params))
        # warm up on a side stream (allocator pools, workspaces, lazy function attributes, NCCL connections), then
        # capture.  Warm-up steps run real Adam updates on an all-zero batch, so everything they touch is put back.
        state = optimizer.state_tensors()
        snap = [t.clone() for t in state]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                if self.accumulate > 1:
                    self._eager(update=False)
                self._eager()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        # one pool for both graphs: they never run at the same time, so the micro-step's activations reuse the closing step's
        pool = torch.cuda.graph_pool_handle()
        self.micro_graph: Optional[torch.cuda.CUDAGraph] = None
        self.launches_per_micro_replay: Optional[int] = None
        if self.accumulate > 1:
            self.micro_graph = torch.cuda.CUDAGraph()
            n0 = _cabi.launch_count()
            with torch.cuda.graph(self.micro_graph, pool=pool, capture_error_mode="thread_local"):
                self._eager(update=False)
            self.launches_per_micro_replay = _cabi.launch_count() - n0
        self.graph = torch.cuda.CUDAGraph()
        n0 = _cabi.launch_count()
        # thread_local: only THIS thread is held to the capture rules -- a torch.distributed watchdog thread polling its own
        # events (the process group that bootstrapped the communicator) must not invalidate the capture
        with torch.cuda.graph(self.graph, pool=pool, capture_error_mode="thread_local"):
            self._eager()
        self.launches_per_replay = _cabi.launch_count() - n0  # b200 kernels inside one replay of the (closing) graph
        with torch.no_grad():
            for dst, src in zip(state, snap):
                dst.copy_(src)
        if optimizer.step_dev is not None:
            optimizer.step_count = int(optimizer.step_dev.item())
        torch.cuda.synchronize()

    def _eager(self, update: bool = True) -> None:
        """One step; ``update=False``: a micro-step of a window, which only adds its gradients to the arenas."""
        from . import dp

        if self.accumulate == 1:
            self.optimizer.zero_grad()
        with contextlib.nullcontext() if update else dp.no_sync(self.model):
            loss = self.model.train_step(*self.inputs)  # DP: the reducers all-reduce bucket by bucket inside backward
        if update and not self.flat:
            if self.clip_norm > 0.0:
                self.optimizer.clip_grad_norm_(self.clip_norm)  # device-side clip coefficient: captured with the step
            self.optimizer.step()
        self.loss.copy_(loss)
        if self.model.last_bad_flag is not None:
            self.bad_label.copy_(self.model.last_bad_flag)

    def step(self, *inputs: Tensor) -> Tensor:
        self.optimizer.sync_hyper()  # lr schedule: 24 bytes host->device when (and only when) a value changed
        for dst, src in zip(self.inputs, inputs):
            dst.copy_(src.reshape(dst.shape), non_blocking=True)
        if self.accumulate > 1 and self.micro == 0:
            for a in self.optimizer.arenas():
                ops.fill_f32(a.grad, 0.0)
        self.micro = (self.micro + 1) % self.accumulate
        self.updated = self.micro == 0
        if not self.updated:
            self.micro_graph.replay()
            return self.loss
        self.graph.replay()
        if self.flat:
            for a in self.optimizer.arenas():
                self.comm.allreduce_(a.grad, average=True)
            if self.clip_norm > 0.0:
                self.optimizer.clip_grad_norm_(self.clip_norm)  # (clipping sees the AVERAGED gradients, as under DDP)
            self.optimizer.step()
        return self.loss

    def release(self) -> None:
        """Destroy the captured graph.  REQUIRED before ``comm.close()`` when the graph holds NCCL kernels: ``ncclCommDestroy``
        waits for every CUDA graph that captured the communicator to be destroyed (it hung the 2-GPU bench at exit until the
        graph was dropped first)."""
        if self.graph is not None:
            torch.cuda.synchronize()
            self.graph.reset()
            self.graph = None
            if self.micro_graph is not None:
                self.micro_graph.reset()
                self.micro_graph = None

    def check_labels(self) -> None:
        """Synchronises and raises ``ValueError`` if the last replay saw a label outside [0, num_classes)."""
        if int(self.bad_label.item()) != 0:
            raise ValueError("cross_entropy: a label of the last step was outside [0, num_classes)")
