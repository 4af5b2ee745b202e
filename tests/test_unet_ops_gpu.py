"""Every op of the SD-UNet's native blocks, one at a time, and the modules' wiring of those ops (tests/_unet_taps.py).

For each block -- ResidualBlockWithTimeEmbeddingB200, CrossAttentionB200 (self and cross), SpatialTransformerB200 (GroupNorm and
to_latent, its SpatialTransformerBlocks, from_latent), ResDownsampleB200 and ResUpsampleB200 -- the eager bf16-autocast oracle
(oracle/unet_oracle.py::*_ops) runs forward and backward with every op boundary retained.  Then:

1. teacher forcing: each op of the block's table runs on eager's own inputs of that op, with the arguments the module passes.
   Its outputs must be within the float64 bound of the same op (``_unet_taps`` docstring), and within 1e-3 relative L2 of eager's
   output of the op (2e-3 for attention).  The ops whose rounding point the modules document as different from eager's are held
   to 2 x relerr(eager, float64) instead, and named in the rows (``rule=TWICE``):
     - the biased 3x3 / 1x1 convolutions that add their bias in fp32 (ResBlock conv1, conv2 and shortcut; to_latent, from_latent);
     - the packed input gradients summed in fp32 (self-attention's dx, cross-attention's dcontext);
     - GEGLU's backward (the dGEGLU epilogue) and the LayerNorm gradients rounded before the bf16 residual add.
2. wiring: the module's own forward and backward run on eager's stage input and upstream gradient while ``ops`` is replaced, in
   the three module files, by a recorder.  The recorded calls must be the table, every tensor argument bit-equal to its source in
   the table, every output within the float64 bound of the op on what it received, and the module's output, input gradients and
   parameter gradients bit-equal to the table's.

Shapes are SD-v1.5's at 512 px, at batch 1 and 3, and batch 8 at 8 x 8 (one 128-pixel tile holds two images)."""
import os
import sys
import time

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import attention, spatial_transformer, unet_blocks  # noqa: E402
from cflearn_b200.attention import CrossAttentionB200  # noqa: E402
from cflearn_b200.spatial_transformer import SpatialTransformerB200  # noqa: E402
from cflearn_b200.unet_blocks import ResDownsampleB200, ResUpsampleB200, ResidualBlockWithTimeEmbeddingB200  # noqa: E402
import _unet_taps as ut  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
CL = torch.channels_last
HEADS, CTX_T, CTX_D, TDIM = 8, 77, 768, 1280


def _load(m, seed):
    import unet_oracle as uo

    sd = uo.synthetic_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=seed)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def _randn(shape, g):
    """bf16 N(0, 1) on the GPU; as fp32 it is the same tensor (the upstream gradients: eager's bf16 output gradient is exact)."""
    return torch.randn(*shape, generator=g).to(BF).to(DEV)


def _eager(fn, sd, leaves, up, *args):
    """``fn`` (an oracle *_ops) under bf16 autocast with every boundary's value (E) and gradient (G) kept; G also holds the leaves'
    gradients and, under "p:<key>", the parameters'."""
    params = {k: v.to(DEV).detach().clone().requires_grad_(True) for k, v in sd.items()}
    lv = {k: v.detach().clone().requires_grad_(True) for k, v in leaves.items()}
    with torch.autocast("cuda", dtype=BF):
        o = fn(params, "", *lv.values(), *args)
    for t in o.values():
        if t.requires_grad and not t.is_leaf:
            t.retain_grad()
    (o["out"].float() * up.float()).sum().backward()
    E = {k: v.detach() for k, v in o.items()}
    G = {k: v.grad for k, v in o.items() if v.grad is not None}
    G.update({k: v.grad for k, v in lv.items()})
    G.update({"p:" + k: v.grad for k, v in params.items()})
    return E, G


def _module(m, inputs, up, call):
    """The module's forward and backward through autograd: its output, its inputs' and parameters' ("p:<name>") gradients."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in inputs.items()}
    out = call(m, leaves)
    out.backward(up)
    res = {"out": out.detach()}
    res.update({k: v.grad for k, v in leaves.items()})
    res.update({"p:" + k: p.grad for k, p in m.named_parameters()})
    return res


def _run(tag, rows, env, E, G, m, inputs, up, call, finals, monkeypatch):
    t0 = time.time()
    ut.REPORT.__init__()
    twice = ut.teacher_forced(rows, dict(env), E, G, tag + " [eager inputs]")
    rec = ut.Recorder()
    with monkeypatch.context() as mp:
        for mod in (unet_blocks, spatial_transformer, attention):
            mp.setattr(mod, "ops", rec)
        res = _module(m, inputs, up, call)
    torch.cuda.synchronize()
    env3 = dict(env)
    ut.wiring(rows, env3, rec.calls, tag + " [module]")
    ut.check_finals(finals, res, env3, tag)
    worst_eager = max((e / b, w) for w, e, b, _ in ut.REPORT.eager)
    print(f"\n{tag}: {len(rows)} ops; worst element-wise error / bound {ut.REPORT.worst[0]:.3f} ({ut.REPORT.worst[1]}); "
          f"worst relerr vs eager / bound {worst_eager[0]:.3f} ({worst_eager[1]}); 2x-eager ops: {sorted(set(twice))}; "
          f"{time.time() - t0:.1f} s")


# ---- ResBlock ----------------------------------------------------------------------------------------------------------------
RES = [(b, s, ci, co) for s, ci, co in ((64, 320, 320), (32, 320, 640), (16, 640, 1280), (8, 2560, 1280), (8, 1920, 1280))
       for b in (1, 3)] + [(8, 8, 2560, 1280)]


@pytest.mark.parametrize("B,side,Cin,Cout", RES)
def test_res_block_ops(B, side, Cin, Cout, monkeypatch):
    import unet_oracle as uo

    m, sd = _load(ResidualBlockWithTimeEmbeddingB200(Cin, Cout, norm_eps=1e-5, time_embedding_channels=TDIM), seed=Cin + side)
    g = torch.Generator().manual_seed(B + side)
    x, tn, up = _randn((B, Cin, side, side), g), _randn((B, TDIM), g), _randn((B, Cout, side, side), g)
    E, G = _eager(uo.res_block_ops, sd, {"x": x, "time": tn}, up)
    env = ut.res_block_env(sd, ut.nhwc(x), tn, ut.nhwc(up))
    _run(f"ResBlock B{B} {side}x{side} {Cin}->{Cout}", ut.res_block_table(B, side, side, Cin, Cout, TDIM), env, E, G, m,
         {"x": x.contiguous(memory_format=CL), "time": tn}, up.contiguous(memory_format=CL), lambda m, v: m(v["x"], v["time"]),
         ut.res_block_finals(Cin, Cout), monkeypatch)


# ---- CrossAttention ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cross", [False, True])
def test_cross_attention_ops(cross, monkeypatch):
    import unet_oracle as uo

    B, T, C = 3, 32 * 32, 640
    m, sd = _load(CrossAttentionB200(query_dim=C, context_dim=CTX_D if cross else None, num_heads=HEADS, head_dim=C // HEADS), seed=5)
    g = torch.Generator().manual_seed(6)
    x, up = _randn((B, T, C), g), _randn((B, T, C), g)
    ctx = _randn((B, CTX_T, CTX_D), g) if cross else None
    leaves = {"x": x, "context": ctx} if cross else {"x": x}
    E, G = _eager(lambda sd_, p, x_, c_=None: uo.cross_attention_ops(sd_, p, x_, c_, HEADS), sd, leaves, up)
    c = "ctx" if cross else None
    Er = lambda k: lambda E, G: ut.rows_(E[k])  # noqa: E731
    Gr = lambda k: lambda E, G: ut.rows_(G[k])  # noqa: E731
    rows = ut.attention_fwd_table("a.", "", B, HEADS, C, "x", c, None, "out", Er("out"))
    rows += ut.attention_bwd_table("a.", "", B, HEADS, C, T, CTX_T if cross else T, C, CTX_D if cross else C, "x", c, "dout", "dx", "dc",
                                   Gr("x"), Gr("context") if cross else None)
    env = {"x": ut.rows_(x), "dout": ut.rows_(up), **ut.attention_env(sd, "a.", "", not cross)}
    finals = [("out", lambda r: ut.rows_(r["out"]), "out"), ("dx", lambda r: ut.rows_(r["x"]), "dx")]
    if cross:
        env["ctx"] = ut.rows_(ctx)
        finals.append(("dcontext", lambda r: ut.rows_(r["context"]), "dc"))
    finals += ut.attention_finals("a.", C, not cross)
    _run(f"CrossAttention {'cross' if cross else 'self'} B{B} T{T} C{C}", rows, env, E, G, m, leaves, up,
         lambda m, v: m(v["x"], context=v.get("context")), finals, monkeypatch)


# ---- SpatialTransformer ------------------------------------------------------------------------------------------------------
ST = [(b, s, c, 1) for s, c in ((64, 320), (32, 640), (16, 1280), (8, 1280)) for b in (1, 3)] + [(8, 8, 1280, 1), (3, 16, 640, 2)]


@pytest.mark.parametrize("B,side,C,layers", ST)
def test_spatial_transformer_ops(B, side, C, layers, monkeypatch):
    import unet_oracle as uo

    m, sd = _load(SpatialTransformerB200(C, HEADS, C // HEADS, num_layers=layers, context_dim=CTX_D), seed=C + side)
    g = torch.Generator().manual_seed(B + side + layers)
    x, ctx, up = _randn((B, C, side, side), g), _randn((B, CTX_T, CTX_D), g), _randn((B, C, side, side), g)
    E, G = _eager(lambda sd_, p, x_, c_: uo.spatial_transformer_ops(sd_, p, x_, c_, HEADS), sd, {"x": x, "context": ctx}, up)
    rows, dc = ut.spatial_transformer_table(B, side, side, C, HEADS, layers, CTX_T, CTX_D)
    env = ut.spatial_transformer_env(sd, layers, ut.nhwc(x), ut.rows_(ctx), ut.nhwc(up))
    _run(f"SpatialTransformer B{B} {side}x{side} C{C} layers {layers}", rows, env, E, G, m,
         {"x": x.contiguous(memory_format=CL), "context": ctx}, up.contiguous(memory_format=CL),
         lambda m, v: m(v["x"], v["context"]), ut.spatial_transformer_finals(C, layers, dc), monkeypatch)


# ---- ResDownsample / ResUpsample ---------------------------------------------------------------------------------------------
RESAMPLE = [(up, b, s, c) for up, s, c in ((False, 64, 320), (False, 32, 640), (False, 16, 1280), (True, 8, 1280), (True, 16, 1280),
                                           (True, 32, 640)) for b in (1, 3)] + [(False, 8, 16, 1280), (True, 8, 8, 1280)]


@pytest.mark.parametrize("up,B,side,C", RESAMPLE)
def test_resample_ops(up, B, side, C, monkeypatch):
    import unet_oracle as uo

    m, sd = _load((ResUpsampleB200 if up else ResDownsampleB200)(C, True), seed=C + side)
    g = torch.Generator().manual_seed(B + side)
    so = 2 * side if up else side // 2
    x, dout = _randn((B, C, side, side), g), _randn((B, C, so, so), g)
    E, G = _eager(uo.resample_ops, sd, {"x": x}, dout)
    env = ut.resample_env(sd, up, B, ut.nhwc(x), ut.nhwc(dout))
    _run(f"{'ResUpsample' if up else 'ResDownsample'} B{B} {side}x{side} C{C}", ut.resample_table(up, B, side, side, C, C), env, E, G, m,
         {"x": x.contiguous(memory_format=CL)}, dout.contiguous(memory_format=CL), lambda m, v: m(v["x"]), ut.resample_finals(up, C),
         monkeypatch)
