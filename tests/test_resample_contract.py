"""The companion C-ABI (include/b200_cflearn_ext.h) held to the rules of the main header, and the resampling modules' surface,
checked without a GPU.

The pointers are fake and never dereferenced: refused calls stop at the argument checks, before any tensor map is encoded.  A call
that passes them reaches B200_ERR_DRIVER on a machine without a GPU; those run only there."""
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cflearn_b200  # noqa: E402
from cflearn_b200 import _cabi  # noqa: E402
from cflearn_b200.unet_blocks import ResDownsampleB200, ResUpsampleB200, check_resample_geometry  # noqa: E402

ARG, ALIGN, DRIVER = -1, -2, -3
FAKE = 1 << 20
ODD = FAKE + 8  # not 16-byte aligned
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="accepted calls would launch kernels on fake pointers")
EXT_HEADER = os.path.join(ROOT, "include", "b200_cflearn_ext.h")


def _declared(path):
    text = re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", text)))


# ---- the table ---------------------------------------------------------------------------------------------------------------------
def test_header_equals_table_and_every_entry_is_exported():
    declared = _declared(EXT_HEADER)
    assert declared and set(declared) == set(_cabi.EXT_SIGNATURES), set(declared) ^ set(_cabi.EXT_SIGNATURES)
    assert not set(_cabi.EXT_SIGNATURES) & set(_cabi.SIGNATURES)
    assert _cabi.available(), _cabi.load_error()
    assert _cabi.exported_ext_symbols() == list(_cabi.EXT_SIGNATURES)


def test_argument_counts_match_the_header():
    text = re.sub(r"/\*.*?\*/", "", open(EXT_HEADER).read(), flags=re.S)
    for name, (_, args) in _cabi.EXT_SIGNATURES.items():
        params = re.search(rf"\b{name}\s*\(([^)]*)\)", text).group(1)
        assert len(params.split(",")) == len(args), name


@pytest.mark.skipif(shutil.which("cc") is None and shutil.which("gcc") is None, reason="no C compiler")
def test_header_parses_as_c99(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    src = tmp_path / "t.c"
    src.write_text("#include \"b200_cflearn_ext.h\"\nint main(void) { return 0; }\n")
    res = subprocess.run([cc, "-std=c99", "-pedantic", "-Werror", "-Wall", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


def test_only_ops_calls_the_companion_entries():
    """The Python sources of the project (the package, the tools, the oracle and the scripts at the root) name a companion entry
    only in ops.py and _cabi.py."""
    pkg = os.path.join(ROOT, "carefree-learn_b200")
    sources = [os.path.join(ROOT, f) for f in os.listdir(ROOT) if f.endswith(".py")]
    for d in (pkg, os.path.join(ROOT, "tools"), os.path.join(ROOT, "oracle")):
        for dirpath, _, files in os.walk(d):
            sources += [os.path.join(dirpath, f) for f in files if f.endswith(".py")]
    callers = {os.path.relpath(path, ROOT) for path in sources if any(name in open(path).read() for name in _cabi.EXT_SIGNATURES)}
    assert callers <= {os.path.relpath(os.path.join(pkg, "ops.py"), ROOT), os.path.relpath(os.path.join(pkg, "_cabi.py"), ROOT)}, callers


# ---- the argument contracts ------------------------------------------------------------------------------------------------------------
def _status(name, *args):
    rc = getattr(_cabi.lib(), name)(*args)
    return rc, _cabi.last_error()


CONV = ["b200_conv3x3_s2_nhwc_bf16", "b200_conv3x3_up2_nhwc_bf16"]


def _conv(name, x=FAKE, w=FAKE, bias=None, out=FAKE, aux=None, ldo=64, B=2, H=16, W=16, Cin=64, Cout=64, epi=0):
    return _status(name, x, w, bias, out, aux, ldo, B, H, W, Cin, Cout, epi, None)


@pytest.mark.parametrize("name", CONV)
@pytest.mark.parametrize("kw,code,text", [
    (dict(B=0), ARG, "non-positive size"), (dict(H=-2), ARG, "non-positive size"), (dict(Cout=0), ARG, "non-positive size"),
    (dict(Cin=96), ARG, "multiple of 64"), (dict(Cout=60, ldo=64), ARG, "multiple of 8"),
    (dict(W=24), ARG, "width must divide 128"), (dict(H=12, W=32), ARG, "grid height"),
    (dict(x=None), ARG, "null pointer"), (dict(w=None), ARG, "null pointer"), (dict(out=None), ARG, "null pointer"),
    (dict(epi=1), ARG, "epilogue not offered"), (dict(epi=12), ARG, "unknown epilogue"), (dict(epi=10), ARG, "needs aux"),
    (dict(ldo=32), ARG, "ldo < N"), (dict(ldo=68), ALIGN, "16-byte aligned"), (dict(out=ODD), ALIGN, "16-byte aligned"),
    (dict(epi=10, aux=ODD), ALIGN, "16-byte aligned"),
])
def test_conv_refusals(name, kw, code, text):
    if name == CONV[1] and kw.get("H") == 12:  # the upsampling grid is H x W itself
        kw = dict(H=6, W=32)
    rc, msg = _conv(name, **kw)
    assert rc == code and text in msg, (rc, msg)


def test_stride2_needs_even_sides():
    for kw in (dict(H=15), dict(W=17)):
        rc, msg = _conv(CONV[0], **kw)
        assert rc == ARG and "must be even" in msg, msg


@pytest.mark.parametrize("kw,code,text", [
    (dict(B=0), ARG, "non-positive size"), (dict(H=15), ARG, "must be even"), (dict(Cout=96), ARG, "multiple of 64"),
    (dict(Cin=12), ARG, "multiple of 8"), (dict(W=48), ARG, "width must divide 128"), (dict(dy=None), ARG, "null pointer"),
    (dict(w=None), ARG, "null pointer"), (dict(dx=None), ARG, "null pointer"), (dict(dx=ODD), ALIGN, "16-byte aligned"),
])
def test_dgrad_refusals(kw, code, text):
    a = dict(dy=FAKE, w=FAKE, dx=FAKE, B=2, H=16, W=16, Cin=64, Cout=64)
    a.update(kw)
    rc, msg = _status("b200_conv3x3_s2_dgrad_nhwc_bf16", a["dy"], a["w"], a["dx"], a["B"], a["H"], a["W"], a["Cin"], a["Cout"], None)
    assert rc == code and text in msg, (rc, msg)


@pytest.mark.parametrize("kw,code,text", [
    (dict(B=0), ARG, "non-positive size"), (dict(W=13), ARG, "must be even"), (dict(Cin=32), ARG, "multiple of 64"),
    (dict(Cout=4), ARG, "multiple of 8"), (dict(H=2, W=256), ARG, "width must divide 64"), (dict(H=8, W=8), ARG, "multiple of 64"),
    (dict(dy=None), ARG, "null pointer"), (dict(x=None), ARG, "null pointer"), (dict(part=None), ARG, "null pointer"),
    (dict(part=ODD), ALIGN, "16-byte aligned"),
])
def test_wgrad_refusals(kw, code, text):
    a = dict(dy=FAKE, ld=64, x=FAKE, part=FAKE, B=2, H=16, W=16, Cin=64, Cout=64, splits=2)
    a.update(kw)
    rc, msg = _status("b200_conv3x3_s2_wgrad_nhwc_bf16", a["dy"], a["ld"], a["x"], a["part"], a["B"], a["H"], a["W"], a["Cin"], a["Cout"],
                      a["splits"], None)
    assert rc == code and text in msg, (rc, msg)


@pytest.mark.parametrize("name", ["b200_upsample_nearest2x_bf16", "b200_sum2x2_bf16"])
@pytest.mark.parametrize("kw,code,text", [
    (dict(B=0), ARG, "non-positive size"), (dict(W=-1), ARG, "non-positive size"), (dict(C=12), ARG, "multiple of 8"),
    (dict(x=None), ARG, "null pointer"), (dict(out=None), ARG, "null pointer"), (dict(x=ODD), ALIGN, "16-byte aligned"),
    (dict(out=ODD), ALIGN, "16-byte aligned"),
])
def test_copy_refusals(name, kw, code, text):
    a = dict(x=FAKE, out=FAKE, B=2, H=8, W=8, C=64)
    a.update(kw)
    rc, msg = _status(name, a["x"], a["out"], a["B"], a["H"], a["W"], a["C"], None)
    assert rc == code and text in msg, (rc, msg)


# the six resampling layers of SD-v1.5 at 512 px: (up, H, W, C)
SD_LAYERS = [(False, 64, 64, 320), (False, 32, 32, 640), (False, 16, 16, 1280), (True, 8, 8, 1280), (True, 16, 16, 1280),
             (True, 32, 32, 640)]


@no_device
@pytest.mark.parametrize("B", range(1, 9))
@pytest.mark.parametrize("up,H,W,C", SD_LAYERS)
def test_sd_shapes_are_admitted(up, H, W, C, B):
    """Every call the modules make at the SD shapes passes its argument checks (and reaches the tensor-map encode)."""
    check_resample_geometry("layer", up, H, W, C, C)
    if up:
        assert _conv(CONV[1], ldo=C, B=B, H=H, W=W, Cin=C, Cout=C, epi=10, aux=FAKE)[0] == DRIVER
        # backward: the stride-1 input and weight gradients at 2H x 2W (the copy kernels take any size with C % 8 == 0)
        assert _status("b200_conv3x3_nhwc_bf16", FAKE, FAKE, None, FAKE, None, C, B, 2 * H, 2 * W, C, C, 0, None)[0] == DRIVER
        assert _status("b200_conv3x3_wgrad_nhwc_bf16", FAKE, C, FAKE, FAKE, B, 2 * H, 2 * W, C, C, 2, None)[0] == DRIVER
    else:
        assert _conv(CONV[0], ldo=C, B=B, H=H, W=W, Cin=C, Cout=C, epi=10, aux=FAKE)[0] == DRIVER
        assert _status("b200_conv3x3_s2_dgrad_nhwc_bf16", FAKE, FAKE, FAKE, B, H, W, C, C, None)[0] == DRIVER
        assert _status("b200_conv3x3_s2_wgrad_nhwc_bf16", FAKE, C, FAKE, FAKE, B, H, W, C, C, 2, None)[0] == DRIVER


# ---- the modules ---------------------------------------------------------------------------------------------------------------------------
def test_state_dicts_match_the_reference():
    """ResDownsample(use_conv=True) owns `net` = Conv2d(3, stride 2, padding 1); ResUpsample owns `conv` = Conv2d(3, padding 1)."""
    down = ResDownsampleB200(320, True)
    assert [(k, tuple(v.shape)) for k, v in down.state_dict().items()] == [("net.weight", (320, 320, 3, 3)), ("net.bias", (320,))]
    assert down.net.stride == (2, 2) and down.net.padding == (1, 1)
    up = ResUpsampleB200(1280, True, out_channels=640)
    assert [(k, tuple(v.shape)) for k, v in up.state_dict().items()] == [("conv.weight", (640, 1280, 3, 3)), ("conv.bias", (640,))]
    assert all(v.dtype == torch.float32 for v in list(down.state_dict().values()) + list(up.state_dict().values()))
    # strict loading both ways
    ref = torch.nn.Conv2d(320, 640, 3, stride=2, padding=1)
    down2 = ResDownsampleB200(320, True, out_channels=640)
    down2.load_state_dict({"net." + k: v for k, v in ref.state_dict().items()}, strict=True)
    back = torch.nn.Module()
    back.net = torch.nn.Conv2d(320, 640, 3, stride=2, padding=1)
    back.load_state_dict(down2.state_dict(), strict=True)
    assert torch.equal(back.net.weight, ref.weight)


@pytest.mark.parametrize("cls", [ResDownsampleB200, ResUpsampleB200])
@pytest.mark.parametrize("kw,option", [(dict(use_conv=False), "use_conv"), (dict(signal_dim=3), "signal_dim"), (dict(padding=0), "padding"),
                                       (dict(padding=2), "padding")])
def test_unsupported_options_raise(cls, kw, option):
    args = dict(use_conv=True)
    args.update(kw)
    use_conv = args.pop("use_conv")
    with pytest.raises(NotImplementedError, match=option):
        cls(64, use_conv, **args)


def test_modules_refuse_cpu_tensors_and_bad_shapes():
    for m, shape in ((ResDownsampleB200(64, True), (1, 64, 16, 16)), (ResUpsampleB200(64, True), (1, 64, 8, 8))):
        with pytest.raises(cflearn_b200.B200Error, match="CUDA"):
            m(torch.zeros(shape, dtype=torch.bfloat16))
        with pytest.raises(cflearn_b200.B200Error):
            m(torch.zeros((1, 32) + shape[2:], dtype=torch.bfloat16))
    with pytest.raises(cflearn_b200.B200Error, match="even"):
        ResDownsampleB200(64, True)(torch.zeros((1, 64, 15, 16), dtype=torch.bfloat16))
    with pytest.raises(cflearn_b200.B200Error, match="multiple of 64"):
        check_resample_geometry("x", True, 8, 8, 96, 64)
