"""The KL autoencoder's decoder on native kernels (carefree-learn_b200/autoencoder.py), the wide-row convolutions and the row
softmax entry, checked without a GPU: the oracle against the reference's own decode, the state_dict against the zoo's f8 layout,
every refusal, the geometry rule, and the argument contracts of the C entries with fake pointers (never dereferenced: a refused
call stops before any tensor map is encoded or kernel launched; an admitted convolution reaches B200_ERR_DRIVER on a machine
without a GPU, so those calls run only there)."""
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import cflearn_b200  # noqa: F401,E402
from cflearn_b200 import B200Error, _cabi  # noqa: E402
from cflearn_b200.autoencoder import AttentionAutoEncoderKLB200  # noqa: E402
import ae_oracle as ao  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
ARG, ALIGN, DRIVER = -1, -2, -3
FAKE = 1 << 20
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="accepted calls would launch kernels on fake pointers")


def _model(name="kl_f8", **kw):
    cfg = ao.ae_config(name)
    cfg.update(kw)
    return AttentionAutoEncoderKLB200(cfg.pop("img_size"), cfg.pop("in_channels"), cfg.pop("out_channels"), cfg.pop("inner_channels"),
                                      cfg.pop("latent_channels"), cfg.pop("channel_multipliers"), **cfg)


# ---- the oracle and the state_dict -----------------------------------------------------------------------------------------------
def test_oracle_is_the_reference_decode():
    g = torch.load(os.path.join(GOLDEN, "ae_kl_tiny_reference.pt"))
    sd = ao.synthetic_state_dict(g["shapes"], seed=g["weights_seed"])
    with torch.no_grad():
        for key, no_head in (("head", False), ("no_head", True)):
            assert torch.equal(ao.decode(sd, g["z"], no_head=no_head), g["reference"][key]), key


def test_f8_state_dict_is_the_references():
    g = json.load(open(os.path.join(GOLDEN, "ae_kl_f8_state_dict_keys.json")))
    m = _model("kl_f8")
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == g["keys"]
    assert sum(p.numel() for p in m.parameters()) == g["parameters"]


def test_strict_loading_both_ways():
    """A reference-shaped state_dict loads into the module and comes back bit for bit, in the reference's key order."""
    g = torch.load(os.path.join(GOLDEN, "ae_kl_tiny_reference.pt"))
    sd = ao.synthetic_state_dict(g["shapes"], seed=3)
    m = _model("kl_tiny")
    m.load_state_dict(sd, strict=True)
    back = m.state_dict()
    assert list(back) == [k for k, _ in g["shapes"]]
    assert all(torch.equal(back[k], v) for k, v in sd.items())
    other = _model("kl_tiny")
    other.load_state_dict(back, strict=True)
    assert all(torch.equal(other.state_dict()[k], v) for k, v in sd.items())


# ---- refusals ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,option", [
    (dict(attention_resolutions=(32,)), "attention_resolutions"), (dict(dropout=0.1), "dropout"),
    (dict(resample_with_conv=False), "resample_with_conv"), (dict(attention_type="multi_head"), "attention_type"),
    (dict(apply_tanh=True), "apply_tanh"),
])
def test_constructor_refusals(kw, option):
    with pytest.raises(NotImplementedError, match=option):
        _model("kl_tiny", **kw)


@pytest.mark.parametrize("method", ["encode", "forward", "get_results", "reconstruct"])
def test_the_encoder_is_refused(method):
    m = _model("kl_tiny")
    with pytest.raises(NotImplementedError, match=method):
        getattr(m, method)(torch.zeros(1, 3, 16, 16))


class _Inputs:  # the reference's DecoderInputs, duck-typed
    def __init__(self, z, no_head=False, apply_tanh=None):
        self.z, self.no_head, self.apply_tanh = z, no_head, apply_tanh


def test_decode_refusals():
    m = _model("kl_tiny")
    z = torch.zeros(1, 4, 8, 8)
    with pytest.raises(NotImplementedError, match="apply_tanh"):
        m.decode(_Inputs(z, apply_tanh=True))
    with pytest.raises(B200Error, match="CPU|cuda|CUDA"):
        m.decode(_Inputs(z, apply_tanh=False))
    with pytest.raises(B200Error, match=r"\[B, 4, h, w\]"):
        m.decode(torch.zeros(1, 3, 8, 8))
    with pytest.raises(B200Error, match="fp32 or bf16"):
        m.decode(torch.zeros(1, 4, 8, 8, dtype=torch.float16))


# ---- geometry ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,side", [(1, 32), (8, 32), (1, 64), (8, 64)])
def test_f8_admits_256_and_512_px(B, side):
    _model("kl_f8").check_geometry(B, side, side)


def test_f8_refuses_768_px_naming_the_level():
    with pytest.raises(B200Error, match=r"level 3 \(96 x 96 of a 96 x 96 latent\).*width 96"):
        _model("kl_f8").check_geometry(1, 96, 96)


def test_non_square_and_later_levels():
    m = _model("kl_f8")
    m.check_geometry(2, 32, 64)
    with pytest.raises(B200Error, match=r"level 3 \(25 x 64.*height 25"):  # rows of 64 pixels go to 128-pixel tiles in pairs
        m.check_geometry(1, 25, 64)
    with pytest.raises(B200Error, match=r"level 3 \(64 x 48"):
        m.check_geometry(1, 64, 48)


# ---- the wide-row convolutions at their argument checks ------------------------------------------------------------------------------
def _conv(name, W, H=4, Cin=64, B=1):
    rc = getattr(_cabi.lib(), name)(FAKE, FAKE, None, FAKE, None, 64, B, H, W, Cin, 64, 0, None)
    return rc, _cabi.last_error()


CONVS = ["b200_conv3x3_nhwc_bf16", "b200_conv3x3_up2_nhwc_bf16"]


@no_device
@pytest.mark.parametrize("name", CONVS)
@pytest.mark.parametrize("W", [256, 512])
def test_wide_rows_reach_the_driver(name, W):
    rc, msg = _conv(name, W)
    assert rc == DRIVER, (rc, msg)


@pytest.mark.parametrize("name", CONVS)
@pytest.mark.parametrize("W", [48, 192, 384])
def test_other_widths_keep_the_old_refusal(name, W):
    rc, msg = _conv(name, W)
    assert rc == ARG and "width must divide 128" in msg, (rc, msg)


def test_stride2_and_gradients_keep_their_limits():
    lib = _cabi.lib()
    assert lib.b200_conv3x3_s2_nhwc_bf16(FAKE, FAKE, None, FAKE, None, 64, 1, 8, 512, 64, 64, 0, None) == ARG  # a 256-wide grid
    assert "width must divide 128" in _cabi.last_error()
    assert lib.b200_conv3x3_s2_dgrad_nhwc_bf16(FAKE, FAKE, FAKE, 1, 8, 512, 64, 64, None) == ARG
    assert "width must divide 128" in _cabi.last_error()
    assert lib.b200_conv3x3_wgrad_nhwc_bf16(FAKE, 64, FAKE, FAKE, 1, 4, 256, 64, 64, 1, None) == ARG
    assert "width must divide 64" in _cabi.last_error()


# ---- the row softmax ---------------------------------------------------------------------------------------------------------------
def _softmax(s=FAKE, lds=64, p=FAKE, ldp=64, rows=4, cols=64, scale=0.125):
    rc = _cabi.lib().b200_softmax_rows_bf16(s, lds, p, ldp, rows, cols, scale, None)
    return rc, _cabi.last_error()


@pytest.mark.parametrize("kw,code,text", [
    (dict(rows=0), ARG, "non-positive size"), (dict(cols=-1), ARG, "non-positive size"), (dict(scale=0.0), ARG, "scale"),
    (dict(scale=-1.0), ARG, "scale"), (dict(scale=float("inf")), ARG, "scale"), (dict(scale=float("nan")), ARG, "scale"),
    (dict(lds=63), ARG, "lds / ldp < cols"), (dict(ldp=32), ARG, "lds / ldp < cols"), (dict(s=None), ARG, "null pointer"),
    (dict(p=None), ARG, "null pointer"), (dict(s=FAKE + 2), ALIGN, "aligned"), (dict(p=FAKE + 1), ALIGN, "aligned"),
])
def test_softmax_refusals(kw, code, text):
    rc, msg = _softmax(**kw)
    assert rc == code and text in msg and msg.startswith("softmax_rows"), (rc, msg)
