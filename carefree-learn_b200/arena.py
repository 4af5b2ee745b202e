"""The flat parameter arena every native model trains on, and the contract between a model and the trainer seam.

``ParamArena`` holds a model's parameters in one flat fp32 tensor (each ``nn.Parameter`` is a view), an optional bf16 shadow,
and one flat fp32 gradient tensor: one Adam launch, one cast and one all-reduce per arena instead of one per parameter.

``ArenaModule`` is the base class of every trainable native model.  Its docstring is the contract the trainer seam
(``optim.ArenaAdam``, ``optim.GraphedTrainStep``, ``trainer.B200TrainStep`` and ``dp``) reads, and all it reads.
"""
from __future__ import annotations

import math
from typing import Any, Dict, List, Optional, Tuple

import torch
import torch.nn as nn
from torch import Tensor

from . import ops

_ALIGN = 64  # elements; keeps every view 16-byte aligned in both the fp32 and the bf16 arena


def _padded(shape: Tuple[int, ...]) -> int:
    return (math.prod(shape) + _ALIGN - 1) // _ALIGN * _ALIGN


class ParamArena:
    """Flat fp32 parameters + bf16 shadow + flat fp32 gradients, addressed by reference ``state_dict`` key.  ``bf16_shadow=False``:
    no shadow (a module whose ops cast their own weights)."""

    def __init__(self, spec: List[Tuple[str, Tuple[int, ...]]], bf16_shadow: bool = True):
        self.spec = list(spec)
        self.bf16_shadow = bf16_shadow
        self.offsets: Dict[str, int] = {}
        off = 0
        for key, shape in self.spec:
            self.offsets[key] = off
            off += _padded(shape)
        self.total = off
        self.shapes = dict(self.spec)
        self.flat: Optional[Tensor] = None
        self.flat_bf16: Optional[Tensor] = None
        self.grad: Optional[Tensor] = None
        self.params: Dict[str, nn.Parameter] = {}
        self._bf16_version = -1

    def view(self, flat: Tensor, key: str) -> Tensor:
        off = self.offsets[key]
        shape = self.shapes[key]
        return flat[off : off + math.prod(shape)].view(shape)

    def attach(self, params: Dict[str, nn.Parameter]) -> None:
        self.params = params
        self.rebuild()

    def rebuild(self) -> None:
        """(Re)create the arenas on the parameters' current device and re-point every parameter into them."""
        first = next(iter(self.params.values()))
        dev = first.device
        flat = torch.zeros(self.total, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for key, p in self.params.items():
                v = self.view(flat, key)
                v.copy_(p.data.to(torch.float32))
                p.data = v
        self.flat = flat
        self.flat_bf16 = torch.zeros(self.total, dtype=torch.bfloat16, device=dev) if dev.type == "cuda" and self.bf16_shadow else None
        self.grad = torch.zeros(self.total, dtype=torch.float32, device=dev)
        self._bf16_version = -1

    def ensure(self) -> None:
        """Cheap aliasing check: ``module.to(device)`` / ``load_state_dict(assign=True)`` break the views.  An arena whose
        parameters were given but not yet attached (``flat`` None) is built here, on their device."""
        if self.flat is None:
            self.rebuild()
            return
        base = self.flat.data_ptr()
        ok = True
        for key, p in self.params.items():
            if p.data_ptr() != base + 4 * self.offsets[key] or p.device != self.flat.device:
                ok = False
                break
        if not ok:
            self.rebuild()

    def refresh_bf16(self) -> None:
        """fp32 -> bf16 shadow of ALL parameters in one launch (what autocast's per-op weight casts amount to)."""
        assert self.flat is not None and self.flat_bf16 is not None
        ops.cast_bf16(self.flat, self.flat_bf16)

    def w(self, key: str) -> Tensor:  # bf16 view
        return self.view(self.flat_bf16, key)

    def p(self, key: str) -> Tensor:  # fp32 view
        return self.view(self.flat, key)

    def g(self, key: str, arena: Optional[Tensor] = None) -> Tensor:  # fp32 grad view
        return self.view(self.grad if arena is None else arena, key)

    def span(self, keys: List[str]) -> Tuple[int, int]:
        """[lo, hi) of the arena holding ``keys``, which are consecutive in the layout (one all-reduce bucket)."""
        return self.offsets[keys[0]], self.offsets[keys[-1]] + _padded(self.shapes[keys[-1]])

    def claim_grads(self, keys: List[str]) -> bool:
        """Before a backward over ``keys``: whether it adds to the gradient arena in place (``True``: eager's ``p.grad += g``)
        or overwrites it.  It overwrites while no parameter holds a gradient.  Once one does (gradient accumulation), every
        ``p.grad`` that is not yet its arena view is folded in first -- a missing one as zeros, any other tensor copied -- so
        that the arena holds every gradient the backward adds to.  After ``publish_grads`` the gradients are live (each
        ``p.grad`` its arena view) and the next backward accumulates with no extra pass."""
        if all(self.params[k].grad is None for k in keys):
            return False
        with torch.no_grad():
            for key in keys:
                p, v = self.params[key], self.view(self.grad, key)
                if p.grad is None:
                    ops.fill_f32(v, 0.0)
                elif p.grad.data_ptr() != v.data_ptr():
                    v.copy_(p.grad)
        return True

    def publish_grads(self, keys: List[str]) -> None:
        """Make each ``p.grad`` of ``keys`` its view of the gradient arena (no copies)."""
        for key in keys:
            p = self.params[key]
            v = self.view(self.grad, key)
            if p.grad is None or p.grad.data_ptr() != v.data_ptr():
                p.grad = v


def register_dotted(root: nn.Module, key: str, param: nn.Parameter) -> None:
    """Register ``param`` under the dotted ``state_dict`` key ``key`` of ``root``, creating empty intermediate modules."""
    parts = key.split(".")
    mod = root
    for name in parts[:-1]:
        child = mod._modules.get(name)
        if child is None:
            child = nn.Module()
            mod.add_module(name, child)
        mod = child
    mod.register_parameter(parts[-1], param)


class ArenaModule(nn.Module):
    """A trainable native model, as the trainer seam sees it.  The seam reads these names and nothing else:

    ``arenas() -> List[ParamArena]``
        Every parameter arena of the model; each parameter is in exactly one.  ``ArenaAdam`` steps them,
        ``dp.broadcast_parameters`` broadcasts them and the flat exchange (``GraphedTrainStep(flat=True)``) all-reduces
        their gradients.  Default: ``[self.arena]``.
    ``exchanges() -> list``
        The sites of the bucketed gradient exchange, in no particular order.  A site has ``arena`` (a ``ParamArena`` of
        ``arenas()``), ``buckets()`` (the dict ``dp.GradBucketReducer`` takes: for each point of backward that calls
        ``reducer.ready(point)``, the keys of each arena run complete there), ``reducer`` (the bucket reducer, or None; only
        ``dp`` sets it) and a writable ``shrink_next`` (SMs to leave to an in-flight all-reduce).  Default: ``[self.engine]``.
        A model without bucketed exchange raises ``NotImplementedError``.
    ``comm``
        The communicator for the gradients of ``arenas()`` that no exchange site covers, all-reduced by ``train_step``
        itself when it is set (CLIP's loose parameters).  Only ``dp`` sets it.
    ``last_bad_flag``
        The device flag (int32 [1]) the last ``train_step``'s loss or noising wrote for an out-of-range input, or None.
    ``train_step(*batch) -> loss``
        Forward, loss and backward into the gradient arenas (exchanged on the way when reducers are attached); returns
        the loss as a device scalar (``FCNNB200``: the loss and the predictions)."""

    comm: Any = None
    last_bad_flag: Optional[Tensor] = None

    def arenas(self) -> List[ParamArena]:
        return [self.arena]

    def exchanges(self) -> List[Any]:
        return [self.engine]
