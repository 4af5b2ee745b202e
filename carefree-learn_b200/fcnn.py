"""Drop-in for the reference's ``FCNN`` (cflearn/modules/ml/fcnn.py:12-59, registry name ``"fcnn"``) on sm_90a.

BASELINE.json configs[0] is the reference's CPU case: a 10 -> 32 -> 32 -> 1 network (fcnn.py:29-31) trained with
``multi_task[mae, mse]`` on batches of 128 (examples/ml/simple/toy.py).  The whole step -- forward, loss, backward and
per-block gradient partials -- is ONE launch of ``b200_fcnn_step`` (csrc/mlp.cu), fp32 like the reference.
Constructor keywords, ``state_dict`` keys (``net.{i}.linear.linear.{weight,bias}``, ``net.{n}.{weight,bias}``) and the
plain-tensor ``forward`` signature are the reference's; options the fused kernel does not implement raise instead of
silently differing.  Initialisation follows the reference: xavier_normal weights / zero bias in every ``Mapping``
(core/mappings.py:46, core/customs.py:64-67), torch's default ``nn.Linear`` init for the output layer (fcnn.py:54).
"""
from __future__ import annotations

import math
from typing import Any, List, Optional, Tuple

import torch
import torch.nn as nn
from torch import Tensor

from . import ops
from .arena import ArenaModule, ParamArena, register_dotted


def _spec(input_dim: int, output_dim: int, hidden_units: List[int], bias: bool) -> List[Tuple[str, Tuple[int, ...]]]:
    dims = [input_dim] + list(hidden_units)
    out: List[Tuple[str, Tuple[int, ...]]] = []
    for i in range(len(dims) - 1):
        out.append((f"net.{i}.linear.linear.weight", (dims[i + 1], dims[i])))
        if bias:
            out.append((f"net.{i}.linear.linear.bias", (dims[i + 1],)))
    n = len(dims) - 1
    out.append((f"net.{n}.weight", (output_dim, dims[-1])))
    if bias:
        out.append((f"net.{n}.bias", (output_dim,)))
    return out


class _FCNNFn(torch.autograd.Function):
    """predictions = fcnn(x); backward re-runs the fused kernel with the incoming output gradient (the network is
    ~1.4 k parameters: recomputing the forward is cheaper than saving activations)."""

    @staticmethod
    def forward(ctx: Any, module: "FCNNB200", x: Tensor, *params: Tensor) -> Tensor:
        ctx.module = module
        ctx.save_for_backward(x)
        return module._launch(x)[0]

    @staticmethod
    def backward(ctx: Any, dpred: Tensor) -> Tuple[Any, ...]:
        module = ctx.module
        (x,) = ctx.saved_tensors
        G = torch.empty_like(module.arena.flat)
        module._launch(x, dpred=dpred.contiguous().float(), grads=G)
        grads = tuple(module.arena.view(G, k) for k, _ in module.arena.spec)
        return (None, None) + grads


class FCNNB200(ArenaModule):
    def __init__(self, input_dim: int, output_dim: int, hidden_units: Optional[List[int]] = None, *,
                 mapping_type: str = "basic", bias: bool = True, activation: str = "ReLU", batch_norm: bool = False,
                 dropout: float = 0.0, rank: Optional[int] = None, rank_ratio: Optional[float] = None):
        super().__init__()
        if hidden_units is None:  # fcnn.py:29-31
            hidden_units = 2 * [max(32, min(1024, 2 * input_dim))]
        if mapping_type != "basic":
            raise NotImplementedError(f"mapping type `{mapping_type}` is not implemented by the fused FCNN (only `basic`)")
        if activation != "ReLU" or batch_norm or 0.0 < dropout < 1.0 or rank is not None or rank_ratio is not None:
            raise NotImplementedError("the fused FCNN implements the reference defaults only: ReLU, no batch norm, "
                                      "no dropout, full-rank Linear")
        if len(hidden_units) + 1 > 8:
            raise NotImplementedError("the fused FCNN supports at most 8 Linear layers")
        self.input_dim, self.output_dim, self.hidden_units, self.has_bias = input_dim, output_dim, list(hidden_units), bias
        self.dims = [input_dim] + self.hidden_units + [output_dim]
        spec = _spec(input_dim, output_dim, self.hidden_units, bias)
        self.arena = ParamArena(spec)
        params = {}
        n = len(self.hidden_units)
        for key, shape in spec:
            t = torch.zeros(shape)
            if key.endswith("weight"):
                if key.startswith(f"net.{n}."):
                    nn.init.kaiming_uniform_(t, a=math.sqrt(5))  # nn.Linear.reset_parameters
                else:
                    nn.init.xavier_normal_(t)  # Linear(init_method="xavier_normal"), customs.py:64-67
            elif key.startswith(f"net.{n}."):
                bound = 1.0 / math.sqrt(self.dims[-2])
                nn.init.uniform_(t, -bound, bound)
            p = nn.Parameter(t)
            register_dotted(self, key, p)
            params[key] = p
        self.arena.attach(params)
        self._woff = [self.arena.offsets[k] for k, _ in spec if k.endswith("weight")]
        self._boff = [self.arena.offsets[k] for k, _ in spec if k.endswith("bias")] if bias else [-1] * (n + 1)

    def exchanges(self) -> List[Any]:
        raise NotImplementedError("FCNNB200 has no bucketed gradient exchange: its whole backward is one fused launch")

    # ---- kernel launch ------------------------------------------------------------------------------------------
    def _launch(self, x: Tensor, *, y: Optional[Tensor] = None, dpred: Optional[Tensor] = None, grads: Optional[Tensor] = None,
                loss_weights: Tuple[float, float] = (1.0, 1.0)) -> Tuple[Tensor, Optional[Tensor]]:
        if x.dim() != 2 or x.shape[1] != self.input_dim:
            raise ValueError(f"expected input [B, {self.input_dim}], got {tuple(x.shape)}")
        self.arena.ensure()
        if y is not None:
            y = y.reshape(x.shape[0], self.output_dim).contiguous().float()
        return ops.fcnn_step(x.contiguous().float(), self.arena.flat, self.dims, self._woff, self._boff, y=y, dpred=dpred, grads=grads,
                             loss_weights=loss_weights)

    # ---- reference surface --------------------------------------------------------------------------------------
    def forward(self, net: Tensor) -> Tensor:  # fcnn.py:58-59
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            return _FCNNFn.apply(self, net, *[self.arena.params[k] for k, _ in self.arena.spec])
        return self._launch(net)[0]

    def train_step(self, x: Tensor, y: Tensor, *, loss_weights: Tuple[float, float] = (1.0, 1.0)) -> Tuple[Tensor, Tensor]:
        """Forward + ``multi_task[mae, mse]`` loss + backward in one launch; sets ``.grad`` of every parameter (views of
        the gradient arena, overwritten every call) and returns (loss, predictions)."""
        self.arena.ensure()  # may re-create the gradient arena
        pred, loss = self._launch(x, y=y, grads=self.arena.grad, loss_weights=loss_weights)
        self.arena.publish_grads(list(self.arena.params))
        return loss, pred
