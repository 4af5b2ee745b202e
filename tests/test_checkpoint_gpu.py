"""use_checkpoint in the SD-UNet blocks: ResidualBlockWithTimeEmbeddingB200, SpatialTransformerBlockB200 and SpatialTransformerB200
keep only their (blocks') inputs for backward and rerun the forward there.  The forward kernels are deterministic, so the output
and every gradient must equal the stored path's bit for bit (torch.equal); autograd must hold the inputs alone, and backward must
add exactly one forward's launches.  Needs an H100 (pytest -m gpu)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import _cabi  # noqa: E402
from cflearn_b200.spatial_transformer import BLOCK_PARAMS, SpatialTransformerB200, SpatialTransformerBlockB200  # noqa: E402
from cflearn_b200.unet_blocks import ResidualBlockWithTimeEmbeddingB200 as ResBlock  # noqa: E402

DEV = "cuda"
CL = torch.channels_last
B, TDIM, CONTEXT, CONTEXT_DIM, HEADS = 2, 1280, 77, 768, 8


# ---- cases: a module with synthetic weights (conv2 / from_latent not zero), its inputs and an upstream gradient -----------------
def _load(m, seed):
    import unet_oracle as uo

    m.load_state_dict(uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=seed), strict=True)
    return m.to(DEV)


def _res_block(Cin, Cout, side, with_time=True, fmt=CL, seed=0):
    m = _load(ResBlock(Cin, Cout, norm_eps=1e-5, time_embedding_channels=TDIM), seed=Cin + Cout + side + seed)
    g = torch.Generator().manual_seed(side + seed)
    net = torch.randn(B, Cin, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=fmt)
    tn = torch.randn(B, TDIM, generator=g).to(DEV).to(torch.bfloat16)
    up = torch.randn(B, Cout, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=CL)
    return m, [net, tn if with_time else None], up


def _block(C, side, seed=0):
    m = _load(SpatialTransformerBlockB200(C, HEADS, C // HEADS, context_dim=CONTEXT_DIM), seed=C + seed)
    g = torch.Generator().manual_seed(side + seed)
    net = torch.randn(B, side * side, C, generator=g).to(DEV).to(torch.bfloat16)
    context = torch.randn(B, CONTEXT, CONTEXT_DIM, generator=g).to(DEV)
    up = torch.randn(B, side * side, C, generator=g).to(DEV).to(torch.bfloat16)
    return m, [net, context], up


def _transformer(C, side, layers, fmt=CL, seed=0):
    m = _load(SpatialTransformerB200(C, HEADS, C // HEADS, num_layers=layers, context_dim=CONTEXT_DIM), seed=C + side + seed)
    g = torch.Generator().manual_seed(side + seed)
    net = torch.randn(B, C, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=fmt)
    context = torch.randn(B, CONTEXT, CONTEXT_DIM, generator=g).to(DEV)
    up = torch.randn(B, C, side, side, generator=g).to(DEV).to(torch.bfloat16).contiguous(memory_format=CL)
    return m, [net, context], up


SMALL = {"res_block": lambda seed=0: _res_block(320, 640, 16, seed=seed), "block": lambda seed=0: _block(320, 16, seed=seed),
         "transformer": lambda seed=0: _transformer(320, 16, 2, seed=seed)}


def _set_checkpoint(m, flag):
    for mod in m.modules():
        if hasattr(mod, "use_checkpoint"):
            mod.use_checkpoint = flag


def _leaves(inputs):
    return [None if t is None else t.detach().clone().requires_grad_(True) for t in inputs]


def _grads(m, leaves):
    res = {f"input{i}": x.grad for i, x in enumerate(leaves) if x is not None}
    res.update({k: p.grad for k, p in m.named_parameters()})
    return res


def _run(m, inputs, ups, flag, retain=False):
    """Forward + backward with use_checkpoint=flag on fresh leaves, one backward per upstream gradient in ``ups`` (the later
    ones through the same graph with retain, else through a new forward each).  Returns the last output and the gradients."""
    _set_checkpoint(m, flag)
    m.zero_grad(set_to_none=True)
    leaves = _leaves(inputs)
    y = m(*leaves)
    for i, up in enumerate(ups):
        if i and not retain:
            y = m(*leaves)
        y.backward(up, retain_graph=retain)
    return {"out": y.detach(), **_grads(m, leaves)}


def _assert_equal(got, ref):
    assert got.keys() == ref.keys()
    for k in ref:
        assert (got[k] is None) == (ref[k] is None), k
        if ref[k] is not None:
            assert got[k].stride() == ref[k].stride() and torch.equal(got[k], ref[k]), k


# ---- 1. bit-identical outputs and gradients --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [CL, torch.contiguous_format], ids=["channels_last", "contiguous"])
@pytest.mark.parametrize("Cin,Cout,side,with_time", [(320, 320, 64, True), (320, 640, 32, True), (2560, 1280, 8, True),
                                                      (320, 640, 32, False)])
def test_res_block_checkpoint_is_bit_identical(Cin, Cout, side, with_time, fmt):
    m, inputs, up = _res_block(Cin, Cout, side, with_time, fmt)
    ref = _run(m, inputs, [up], False)
    got = _run(m, inputs, [up], True)
    _assert_equal(got, ref)
    assert ("input1" in got) == with_time and (m.time_embedding.weight.grad is None) == (not with_time)


@pytest.mark.gpu
@pytest.mark.parametrize("C,side", [(320, 64), (1280, 16)])
def test_block_checkpoint_is_bit_identical(C, side):
    m, inputs, up = _block(C, side)
    ref = _run(m, inputs, [up], False)
    _assert_equal(_run(m, inputs, [up], True), ref)
    assert ref["input1"].dtype == torch.float32  # the fp32 context's gradient


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [CL, torch.contiguous_format], ids=["channels_last", "contiguous"])
@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("C,side", [(320, 64), (1280, 16)])
def test_transformer_checkpoint_is_bit_identical(C, side, layers, fmt):
    m, inputs, up = _transformer(C, side, layers, fmt)
    ref = _run(m, inputs, [up], False)
    _assert_equal(_run(m, inputs, [up], True), ref)


@pytest.mark.gpu
def test_transformer_checkpoints_each_block_by_its_own_flag():
    """Each block follows its own use_checkpoint, as each of the reference's blocks does: a mixed stack gives the same bits."""
    m, inputs, up = _transformer(320, 16, 2)
    ref = _run(m, inputs, [up], False)
    m.blocks[1].use_checkpoint = True
    m.zero_grad(set_to_none=True)
    leaves = _leaves(inputs)
    y = m(*leaves)
    y.backward(up)
    _assert_equal({"out": y.detach(), **_grads(m, leaves)}, ref)


# ---- 2. autograd semantics -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which", list(SMALL))
def test_two_accumulating_backwards(which):
    m, inputs, up = SMALL[which]()
    up2 = torch.randn(up.shape, generator=torch.Generator().manual_seed(9)).to(DEV).to(up.dtype).contiguous(
        memory_format=CL if up.dim() == 4 else torch.contiguous_format)
    ref = _run(m, inputs, [up, up2], False)
    got = _run(m, inputs, [up, up2], True)
    _assert_equal(got, ref)
    single = _run(m, inputs, [up], True)
    assert not torch.equal(got["input0"], single["input0"])  # the second backward did add into .grad


@pytest.mark.gpu
@pytest.mark.parametrize("which", list(SMALL))
def test_retain_graph_recomputes_again(which):
    m, inputs, up = SMALL[which]()
    once = _run(m, inputs, [up], True)
    twice = _run(m, inputs, [up, up], True, retain=True)
    _assert_equal(twice, {k: v if k == "out" else 2 * v for k, v in once.items()})  # doubling is exact
    _assert_equal(twice, _run(m, inputs, [up, up], False, retain=True))


@pytest.mark.gpu
@pytest.mark.parametrize("which", list(SMALL))
def test_no_grad_saves_nothing_and_recomputes_nothing(which):
    m, inputs, _ = SMALL[which]()
    _set_checkpoint(m, False)
    with torch.no_grad():
        ref = m(*inputs)
    _set_checkpoint(m, True)
    packed = []
    n0 = _cabi.launch_count()
    with torch.no_grad(), torch.autograd.graph.saved_tensors_hooks(lambda t: packed.append(t) or t, lambda t: t):
        out = m(*inputs)
    launches = _cabi.launch_count() - n0
    n0 = _cabi.launch_count()
    with torch.no_grad():
        m(*inputs)
    assert out.grad_fn is None and not packed and torch.equal(out, ref)
    assert launches == _cabi.launch_count() - n0


@pytest.mark.gpu
@pytest.mark.parametrize("which", list(SMALL))
def test_graphed_forward_and_backward(which):
    """Forward and backward with use_checkpoint=True captured in one CUDA graph; a replay on new inputs gives the stored path's
    eager output and gradients."""
    m, inputs, up = SMALL[which]()
    static = _leaves(inputs)
    _set_checkpoint(m, True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # warm-up: workspaces and lazily set kernel attributes, before the capture
        for _ in range(2):
            m.zero_grad(set_to_none=True)
            m(*static).backward(up)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    m.zero_grad(set_to_none=True)
    for x in static:
        if x is not None:
            x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = m(*static)
        y.backward(up)
    _, new, _ = SMALL[which](seed=1)
    with torch.no_grad():
        for x, n in zip(static, new):
            if x is not None:
                x.copy_(n)
    graph.replay()
    torch.cuda.synchronize()
    got = {k: None if v is None else v.clone() for k, v in {"out": y.detach(), **_grads(m, static)}.items()}
    del y  # the captured autograd graph: the eager run below must not reuse its gradient accumulators (capture stream)
    graph.reset()
    _assert_equal(got, _run(m, new, [up], False))


# ---- 3. what autograd holds, and what backward launches ------------------------------------------------------------------------
def _forward_packing(m, inputs, flag):
    """Forward with use_checkpoint=flag under a packing hook: (output, the tensors autograd saved, bytes still allocated)."""
    _set_checkpoint(m, flag)
    leaves = _leaves(inputs)
    packed = []
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    with torch.autograd.graph.saved_tensors_hooks(lambda t: packed.append(t) or t, lambda t: t):
        y = m(*leaves)
    torch.cuda.synchronize()
    return y, leaves, packed, torch.cuda.memory_allocated() - m0


def _same_storage(t, others):
    return any(o is not None and t.data_ptr() == o.data_ptr() and t.shape == o.shape for o in others)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["res_block", "block"])
def test_checkpointed_block_holds_its_inputs_alone(which):
    m, inputs, up = SMALL[which]()
    _run(m, inputs, [up], True)  # warm-up: the shared workspaces reach their size
    y, leaves, packed, held = _forward_packing(m, inputs, True)
    params = m._params() if which == "res_block" else m._block_params()
    expect = [t for t in (*leaves, *params) if t is not None]
    assert len(packed) == len(expect) and all(_same_storage(t, expect) for t in packed)
    out_bytes = y.untyped_storage().nbytes()
    assert held <= out_bytes + (2 << 20), (held, out_bytes)  # the output, and nothing of the activations
    _, _, packed_stored, held_stored = _forward_packing(m, inputs, False)
    assert len(packed_stored) > len(packed) and held_stored > held + out_bytes


@pytest.mark.gpu
def test_checkpointed_transformer_holds_block_inputs_alone():
    """The outer GroupNorm and 1x1 convolutions keep their 9 tensors; each checkpointed block keeps its tokens, the context and
    its 20 parameters, nothing it computes."""
    layers = 2
    m, inputs, up = _transformer(320, 16, layers)
    _run(m, inputs, [up], True)
    _, _, packed, _ = _forward_packing(m, inputs, True)
    assert len(packed) == 9 + layers * (2 + BLOCK_PARAMS)
    block_params = [p for b in m.blocks for p in b._block_params()]
    assert sum(any(t.data_ptr() == p.data_ptr() and t.shape == p.shape for p in block_params) for t in packed) == layers * BLOCK_PARAMS


def _launches(fn):
    n0 = _cabi.launch_count()
    fn()
    return _cabi.launch_count() - n0


@pytest.mark.gpu
@pytest.mark.parametrize("which", list(SMALL))
def test_backward_adds_one_forward_of_launches(which):
    m, inputs, up = SMALL[which]()
    _run(m, inputs, [up], True)  # warm-up

    def fwd():
        with torch.no_grad():
            m(*inputs)

    stored = _launches(lambda: _run(m, inputs, [up], False))
    checkpointed = _launches(lambda: _run(m, inputs, [up], True))
    if which == "transformer":  # the blocks are rerun, not the outer GroupNorm and 1x1 convolutions
        B_, C, H, W = inputs[0].shape
        tokens = inputs[0].permute(0, 2, 3, 1).reshape(B_, H * W, C).contiguous()
        forward = 0
        for blk in m.blocks:
            with torch.no_grad():
                forward += _launches(lambda: blk(tokens, inputs[1]))
        assert forward > 0
    else:
        forward = _launches(fwd)
    assert checkpointed - stored == forward, (stored, checkpointed, forward)
