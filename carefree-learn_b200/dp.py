"""Data-parallel gradient exchange: bucketed NCCL all-reduce of the flat gradient arena, overlapped with backward.

Replaces what ``accelerator.prepare`` sets up in the reference (cflearn/trainer.py:226-229,266-273 -> torch DDP ->
NCCL; launched one process per GPU by cflearn/api/api.py:269-294).  Rank / world size come from the same environment
variables the reference reads (cflearn/toolkit.py:1917-1922: RANK, WORLD_SIZE, LOCAL_RANK).

The engine's backward produces gradients block by block, last block first.  The arena is laid out in forward order,
so each transformer block is one contiguous bucket (~28 MB fp32 for ViT-B/16, DDP's default is 25 MB).  As soon as a
block's last wgrad kernel has been queued, ``ready(i)`` records an event on the compute stream and launches
``all_reduce(AVG)`` for that slice on a dedicated communication stream; ``finish()`` makes the compute stream wait for
the last bucket.  Gradient averaging therefore equals the gradient of the global-batch mean loss (SURVEY.md
finding 3: the reference defines multi-GPU parity only mathematically).
"""
from __future__ import annotations

import contextlib
import ctypes
import os
from typing import Any, Dict, List, Optional, Tuple, Union

import torch
import torch.distributed as dist

from . import _cabi

BucketKey = Union[int, str]


def ddp_info() -> Optional[Tuple[int, int, int]]:
    """(rank, world_size, local_rank) or None -- same contract as cflearn/toolkit.py:1902-1922 get_ddp_info."""
    if "RANK" not in os.environ or "WORLD_SIZE" not in os.environ:
        return None
    return int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))


def shard_indices(n: int, rank: int, world: int) -> range:
    """DistributedSampler's rule without shuffling (cflearn/data/pytorch/api.py:62-71): rank r takes r, r+W, ..."""
    return range(rank, n, world)


class GradBucketReducer:
    """Bucketed gradient averaging over ``torch.distributed``.  ``buckets`` (an exchange site's ``buckets()``): for each point
    of backward that calls ``ready``, the parameter keys of each arena span complete there."""

    def __init__(self, arena, buckets: Dict[BucketKey, List[List[str]]], process_group=None):
        self.arena = arena
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.buckets: Dict[BucketKey, List[Tuple[int, int]]] = {
            point: [arena.span(keys) for keys in runs] for point, runs in buckets.items()}
        self.comm_stream: Optional[torch.cuda.Stream] = None
        self._pending: List = []
        self._forked = False

    def _stream(self) -> torch.cuda.Stream:
        if self.comm_stream is None:
            self.comm_stream = torch.cuda.Stream()
        return self.comm_stream

    def ready(self, key: BucketKey, grad: Optional[torch.Tensor] = None) -> None:
        """Bucket ``key`` of the gradient arena ``grad`` (default: the arena's own) is complete on the current stream:
        start reducing it."""
        if self.world == 1:
            return
        if grad is None:
            grad = self.arena.grad
        views = [grad[lo:hi] for lo, hi in self.buckets[key]]
        if not grad.is_cuda:  # gloo path (host-side logic tests): same protocol, SUM then divide in finish()
            for v in views:
                self._pending.append((dist.all_reduce(v, op=dist.ReduceOp.SUM, group=self.group, async_op=True), v))
            return
        cs = self._stream()
        cs.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(cs):
            for v in views:
                self._allreduce(v)
        self._forked = True

    def _allreduce(self, view: torch.Tensor) -> None:
        """In-place average of ``view`` over the ranks, enqueued on the communication stream."""
        work = dist.all_reduce(view, op=dist.ReduceOp.AVG, group=self.group, async_op=True)
        self._pending.append((work, None))

    def finish(self) -> None:
        """The compute stream waits for every bucket started since the last ``finish`` (gloo: the host waits, then averages)."""
        for work, host_view in self._pending:
            work.wait()  # on CUDA this only orders streams, it does not block the host
            if host_view is not None:
                host_view.div_(self.world)
        self._pending.clear()
        if self._forked:
            torch.cuda.current_stream().wait_stream(self._stream())
            self._forked = False


class NativeComm:
    """The library's own NCCL communicator (C-ABI ``b200_comm_*``, csrc/comm.cu): one per process / GPU.

    Unlike ``torch.distributed``'s ProcessGroup, its all-reduce is a plain stream operation -- no Work object, no
    watchdog thread -- so it can be captured into the CUDA graph of the training step and forked onto a side stream.
    The 128-byte NCCL unique id is created by rank 0 and handed to the other ranks through whatever process group
    already exists (``bootstrap_group``; gloo or nccl), exactly once."""

    def __init__(self, rank: int, world: int, device: torch.device, bootstrap_group: Any = None, max_ctas: Optional[int] = None):
        if not dist.is_initialized():
            raise RuntimeError("NativeComm needs an initialised torch.distributed group to ship the NCCL unique id")
        # NCCL kernels and the persistent kernels of the backward share the SMs: cap the channels NCCL may use so that the
        # step can leave exactly that many SMs free for the GEMM that starts while a bucket is in flight (B200_COMM_CTAS,
        # default 16; ncclConfig_t.maxCTAs of THIS communicator only: torch.distributed's own communicator keeps NCCL's defaults)
        # ``max_ctas=0``: NCCL's own default (for an all-reduce that is NOT overlapped with compute: nothing to leave room for)
        self.ctas = int(os.environ.get("B200_COMM_CTAS", "16")) if max_ctas is None else int(max_ctas)
        self.rank, self.world, self.device = rank, world, device
        lib = _cabi.lib()
        buf = ctypes.create_string_buffer(128)
        if rank == 0:
            _cabi.check(lib.b200_comm_unique_id(buf), "b200_comm_unique_id")
        backend = dist.get_backend(bootstrap_group)
        t = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
        if backend == "nccl":
            t = t.to(device)
        dist.broadcast(t, src=0, group=bootstrap_group)
        raw = bytes(t.cpu().numpy().tobytes())
        handle = ctypes.c_void_p()
        with torch.cuda.device(device):
            _cabi.check(lib.b200_comm_init(raw, rank, world, self.ctas, ctypes.byref(handle)), "b200_comm_init")
        self._h = handle
        self.nccl_version = int(lib.b200_comm_nccl_version())

    def allreduce_(self, t: torch.Tensor, *, average: bool = True) -> None:
        """In-place fp32 all-reduce of a contiguous tensor on the CURRENT stream."""
        if t.dtype != torch.float32 or not t.is_contiguous() or not t.is_cuda:
            raise _cabi.B200Error("NativeComm.allreduce_: contiguous fp32 CUDA tensor required")
        _cabi.call("b200_comm_allreduce_bucket", self._h, t.data_ptr(), t.numel(), int(average), torch.cuda.current_stream().cuda_stream)

    def check(self) -> None:
        """Raises if NCCL recorded an asynchronous error on the communicator (dead peer, failed transport): the caller
        aborts instead of waiting on a collective that will never finish."""
        _cabi.call("b200_comm_async_error", self._h)

    def close(self, abort: bool = False) -> None:
        """``ncclCommDestroy`` (``abort``: ``ncclCommAbort``).  Every CUDA graph that captured this communicator must have been
        destroyed first (``GraphedTrainStep.release()``): NCCL waits for them."""
        if self._h is not None and self._h.value:
            _cabi.lib().b200_comm_finalize(self._h, int(abort))
            self._h = None


class TorchComm:
    """``torch.distributed`` behind the ``NativeComm`` interface (flat, un-captured all-reduces only): the round-1 schedule,
    kept as the conservative fallback of ``bench.py --dp-mode torch``."""

    def __init__(self, rank: int, world: int, device: torch.device, group: Any = None):
        self.rank, self.world, self.device, self.group = rank, world, device, group
        self.ctas = 0
        self.nccl_version = 0

    def allreduce_(self, t: torch.Tensor, *, average: bool = True) -> None:
        dist.all_reduce(t, op=dist.ReduceOp.AVG if average else dist.ReduceOp.SUM, group=self.group)

    def check(self) -> None:
        pass

    def close(self, abort: bool = False) -> None:
        pass


class NativeBucketReducer(GradBucketReducer):
    """Same bucket protocol as ``GradBucketReducer`` over a ``NativeComm``: works eagerly AND under stream capture.

    ``ready(key)`` forks the communication stream off the compute stream and enqueues the bucket's all-reduce there;
    ``finish()`` joins.  The persistent kernels assign their tiles to CTAs statically, so a CTA that cannot start because
    NCCL holds its SM stretches its kernel by the whole duration of the all-reduce: the GEMM launched right behind a
    bucket runs on ``SMs - comm.ctas`` CTAs (``engine.shrink_next``)."""

    def __init__(self, arena, buckets: Dict[BucketKey, List[List[str]]], comm: NativeComm, engine: Any = None):
        super().__init__(arena, buckets, process_group=None)
        self.comm = comm
        self.world = comm.world
        self.engine = engine

    def _allreduce(self, view: torch.Tensor) -> None:
        self.comm.allreduce_(view, average=True)

    def ready(self, key: BucketKey, grad: Optional[torch.Tensor] = None) -> None:
        super().ready(key, grad)
        if self.world > 1 and self.engine is not None and key != "stem":
            self.engine.shrink_next = self.comm.ctas  # the next block's FF2 input-gradient GEMM

    def _stream(self) -> torch.cuda.Stream:
        if self.comm_stream is None:
            # high priority: at a kernel boundary the NCCL CTAs are placed before the next GEMM's
            self.comm_stream = torch.cuda.Stream(priority=-1)
        return self.comm_stream


def attach_native_reducers(module, comm: NativeComm) -> List[NativeBucketReducer]:
    """Overlapped, capturable gradient averaging: a bucket reducer on every exchange site of ``module``
    (``arena.ArenaModule.exchanges``), and ``module.comm`` for the gradients no site covers (CLIP's loose parameters, which
    its ``train_step`` all-reduces itself)."""
    reds = []
    for site in module.exchanges():
        red = site.reducer
        if not isinstance(red, NativeBucketReducer) or red.comm is not comm:
            site.arena.ensure()
            red = site.reducer = NativeBucketReducer(site.arena, site.buckets(), comm, site)
        reds.append(red)
    module.comm = comm
    return reds


def detach_reducers(module) -> None:
    """No gradient exchange: every site's reducer and ``module.comm`` cleared."""
    for site in module.exchanges():
        site.reducer = None
    module.comm = None


@contextlib.contextmanager
def no_sync(module):
    """Backward without the gradient exchange, like DDP's ``no_sync``: inside, the bucket reducers and a module's all-reduce
    of its loose parameters (``module.comm``) are switched off.  Gradient accumulation runs every micro-batch of a window
    but the last inside it, so the window's sum is exchanged once, by its last backward."""
    sites = module.exchanges()
    reducers = [site.reducer for site in sites]
    comm = module.comm
    try:
        detach_reducers(module)
        yield
    finally:
        for site, red in zip(sites, reducers):
            site.reducer = red
        module.comm = comm


def attach_reducer(module, process_group=None) -> List[GradBucketReducer]:
    """Overlapped gradient averaging over ``torch.distributed``: a bucket reducer on every exchange site of ``module``."""
    reds = []
    for site in module.exchanges():
        site.arena.ensure()
        site.reducer = GradBucketReducer(site.arena, site.buckets(), process_group)
        reds.append(site.reducer)
    return reds


def broadcast_parameters(module, src: int = 0, process_group=None) -> None:
    """Identical replicas at start (what DDP's constructor does): one broadcast per flat fp32 arena."""
    for a in module.arenas():
        a.ensure()
        dist.broadcast(a.flat, src=src, group=process_group)
