"""UNetDiffuserB200's surface and the argument contracts of its two entry points (include/b200_cflearn_ext.h), checked without a GPU:
the reference's state_dict keys, shapes and order (fixtures dumped from the reference ``UNetDiffuser``), strict loading, every
refused option, the geometry rule, and every refusal of b200_pad_channels_bf16 / b200_noise_prediction_loss_bf16 (fake pointers,
never dereferenced: refused calls stop at the argument checks)."""
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cflearn_b200  # noqa: E402
from cflearn_b200 import _cabi  # noqa: E402
from cflearn_b200.unet import UNetDiffuserB200, noise_prediction_loss  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
ARG, ALIGN = -1, -2
FAKE = 1 << 20
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="accepted calls would launch kernels on fake pointers")


def _fixture(name):
    d = json.load(open(os.path.join(GOLDEN, name)))
    cfg = {k: tuple(v) if isinstance(v, list) else v for k, v in d["config"].items()}
    return cfg, d


def _build(cfg, **kw):
    cfg = dict(cfg)
    return UNetDiffuserB200(cfg.pop("in_channels"), cfg.pop("out_channels"), use_spatial_transformer=True, **cfg, **kw)


# ---- state dict ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["unet_sd_v1_5_state_dict_keys.json", "unet_small64_state_dict_keys.json"])
def test_state_dict_is_the_references(name):
    cfg, d = _fixture(name)
    with torch.device("meta"):  # SD-v1.5 holds 860 M parameters: the keys need no storage
        m = _build(cfg)
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == d["keys"]
    assert sum(p.numel() for p in m.parameters()) == d["num_params"]


def test_strict_loading_both_ways_and_zero_initialisation():
    cfg, d = _fixture("unet_small64_state_dict_keys.json")
    g = torch.Generator().manual_seed(0)
    ref_sd = {k: torch.randn(shape, generator=g) for k, shape in d["keys"]}  # a reference state dict: its keys, order and shapes
    m = _build(cfg)
    zero = [k for k, v in m.state_dict().items() if v.abs().sum() == 0 and not k.endswith(("norm.bias", "norm1.bias", "norm2.bias",
                                                                                            "norm3.bias", "head.0.bias"))]
    assert "head.2.weight" in zero and "head.2.bias" in zero
    assert any(k.endswith("conv2.weight") for k in zero) and any(k.endswith("from_latent.weight") for k in zero)
    m.load_state_dict(ref_sd, strict=True)
    back = _build(cfg)
    back.load_state_dict(m.state_dict(), strict=True)
    assert list(back.state_dict()) == [k for k, _ in d["keys"]]
    assert all(torch.equal(back.state_dict()[k], v) for k, v in ref_sd.items())


def test_num_head_channels():
    cfg, _ = _fixture("unet_small64_state_dict_keys.json")
    cfg.pop("num_heads")
    m = _build(cfg, num_head_channels=32)
    assert [t.num_heads for t in m.modules() if type(t).__name__ == "SpatialTransformerB200"] == [2, 4, 4, 4, 4, 2, 2]
    with pytest.raises(ValueError, match="num_heads"):
        _build(cfg)


# ---- refusals -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,option", [
    (dict(use_spatial_transformer=False), "use_spatial_transformer"), (dict(resample_with_conv=False), "resample_with_conv"),
    (dict(resample_with_resblock=True), "resample_with_resblock"), (dict(use_scale_shift_norm=True), "use_scale_shift_norm"),
    (dict(num_classes=10), "num_classes"), (dict(dropout=0.1), "dropout"), (dict(signal_dim=3), "signal_dim"),
    (dict(use_linear_in_transformer=True), "use_linear_in_transformer"), (dict(hooks_kwargs={}), "hooks_kwargs"),
])
def test_unsupported_options_raise(kw, option):
    cfg, _ = _fixture("unet_small64_state_dict_keys.json")
    cfg.update(use_spatial_transformer=True)
    cfg.update(kw)
    with pytest.raises(NotImplementedError, match=option):
        UNetDiffuserB200(cfg.pop("in_channels"), cfg.pop("out_channels"), **cfg)


def test_labels_and_control_raise():
    cfg, _ = _fixture("unet_small64_state_dict_keys.json")
    m = _build(cfg)
    x, ts = torch.zeros(1, 4, 16, 16), torch.zeros(1, dtype=torch.long)
    with pytest.raises(NotImplementedError, match="labels"):
        m(x, timesteps=ts, labels=torch.zeros(1, dtype=torch.long))
    with pytest.raises(NotImplementedError, match="control"):
        m(x, timesteps=ts, control=[x])
    with pytest.raises(cflearn_b200.B200Error, match="CUDA"):
        m(x, timesteps=ts)


# ---- geometry -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("side,level", [(64, None), (32, 2), (96, 0), (48, 0), (128, 0)])
def test_sd_geometry(side, level):
    """At SD-v1.5's four levels the tile rules admit 64 x 64 latents (512 px) only among these."""
    cfg, _ = _fixture("unet_sd_v1_5_state_dict_keys.json")
    with torch.device("meta"):
        m = _build(cfg)
    for B in (1, 2, 8):
        if level is None:
            m.check_geometry(B, side, side)
        else:
            with pytest.raises(cflearn_b200.B200Error, match=f"level {level} "):
                m.check_geometry(B, side, side)


@pytest.mark.parametrize("H,W", [(16, 16), (48, 64), (96, 32), (64, 16)])
def test_small_config_admits_non_square_latents(H, W):
    """Every block checks its own grid: the resampling layers at their input's size, the up-sampling one at the lower level."""
    cfg, _ = _fixture("unet_small64_state_dict_keys.json")
    m = _build(cfg)
    for B in (1, 3):
        m.check_geometry(B, H, W)


def test_forward_refuses_the_geometry_before_any_launch():
    cfg, _ = _fixture("unet_small64_state_dict_keys.json")
    m = _build(cfg)
    with pytest.raises(cflearn_b200.B200Error, match="level 0 .*ResDownsampleB200.*weight gradient"):
        m(torch.zeros(1, 4, 8, 8), timesteps=torch.zeros(1))


# ---- the two entries' argument contracts ----------------------------------------------------------------------------------------------
def _status(name, *args):
    rc = getattr(_cabi.lib(), name)(*args)
    return rc, _cabi.last_error()


@pytest.mark.parametrize("kw,code,text", [
    (dict(B=0), ARG, "non-positive size"), (dict(C=0), ARG, "non-positive size"), (dict(W=-1), ARG, "non-positive size"),
    (dict(Cp=0), ARG, "non-positive size"), (dict(Cp=60), ARG, "multiple of 8"), (dict(C=65), ARG, "at most Cp"),
    (dict(f32=2), ARG, "flags"), (dict(cl=-1), ARG, "flags"), (dict(B=1 << 22, H=1 << 10, W=1 << 10), ARG, "too many"),
    (dict(B=1, C=1, H=46341, W=46341, Cp=8), ARG, "H * W"), (dict(B=(1 << 31) - 1, H=1 << 10, W=1 << 10, Cp=1 << 30), ARG, "too many"),
    (dict(x=None), ARG, "null pointer"), (dict(out=None), ARG, "null pointer"), (dict(x=FAKE + 2), ALIGN, "element size"),
    (dict(x=FAKE + 1, f32=0), ALIGN, "element size"), (dict(out=FAKE + 8), ALIGN, "16-byte aligned"),
])
def test_pad_refusals(kw, code, text):
    a = dict(x=FAKE, f32=1, cl=0, out=FAKE, B=2, C=4, H=8, W=8, Cp=64)
    a.update(kw)
    rc, msg = _status("b200_pad_channels_bf16", a["x"], a["f32"], a["cl"], a["out"], a["B"], a["C"], a["H"], a["W"], a["Cp"], None)
    assert rc == code and text in msg, (rc, msg)


@pytest.mark.parametrize("kw,code,text", [
    (dict(B=0), ARG, "non-positive size"), (dict(N=0), ARG, "non-positive size"), (dict(B=1 << 30, N=1 << 20), ARG, "too many"),
    (dict(B=4, N=1 << 62), ARG, "too many"), (dict(B=(1 << 31) - 1, N=(1 << 62) + 1), ARG, "too many"),
    (dict(f32=3), ARG, "noise_f32"), (dict(pred=None), ARG, "null pointer"), (dict(noise=None), ARG, "null pointer"),
    (dict(loss=None), ARG, "exactly one"), (dict(dpred=FAKE, go=FAKE), ARG, "exactly one"), (dict(loss=None, dpred=FAKE), ARG, "grad_out"),
    (dict(pred=FAKE + 1), ALIGN, "element size"), (dict(noise=FAKE + 2), ALIGN, "element size"), (dict(loss=FAKE + 2), ALIGN, "element size"),
    (dict(loss=None, dpred=FAKE + 1, go=FAKE), ALIGN, "element size"), (dict(loss=None, dpred=FAKE, go=FAKE + 2), ALIGN, "element size"),
])
def test_loss_refusals(kw, code, text):
    a = dict(pred=FAKE, noise=FAKE, f32=1, loss=FAKE, dpred=None, go=None, B=2, N=1024)
    a.update(kw)
    rc, msg = _status("b200_noise_prediction_loss_bf16", a["pred"], a["noise"], a["f32"], a["loss"], a["dpred"], a["go"], a["B"], a["N"],
                      None)
    assert rc == code and text in msg, (rc, msg)


@no_device
def test_accepted_calls_pass_the_argument_checks():
    """The SD-v1.5 calls (latents 4 x 64 x 64 at batch 8) are refused only by the launch on a machine without a GPU."""
    for rc, msg in (_status("b200_pad_channels_bf16", FAKE, 1, 1, FAKE, 8, 4, 64, 64, 64, None),
                    _status("b200_noise_prediction_loss_bf16", FAKE, FAKE, 1, FAKE, None, None, 8, 16384, None),
                    _status("b200_noise_prediction_loss_bf16", FAKE, FAKE, 0, None, FAKE, FAKE, 8, 16384, None)):
        assert rc not in (ARG, ALIGN), msg


def test_the_loss_refuses_cpu_tensors():
    with pytest.raises(cflearn_b200.B200Error, match="CUDA"):
        noise_prediction_loss(torch.zeros(1, 4, 8, 8, dtype=torch.bfloat16), torch.zeros(1, 4, 8, 8))
