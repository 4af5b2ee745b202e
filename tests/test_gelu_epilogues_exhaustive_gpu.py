"""The exact-erf GELU epilogues over every bf16 bit pattern, against torch's fp32 GELU and its autograd on the rounded h.

The other GELU tests draw normal random h; these inputs also cover zeros, denormals, the tails where GELU is nearly zero,
the largest finite values, +-inf and NaN (tools/epilogue_ab.py builds them; it also compares two builds bit for bit).
Run on an H100: pytest -m gpu."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import cflearn_b200  # noqa: F401,E402
from epilogue_ab import all_patterns, exhaustive_outputs  # noqa: E402

pytestmark = pytest.mark.gpu
# Absolute error allowed on top of the relative one, per unit of the factor that scales the result: the GEMM's fast erf is
# accurate to ~1e-7 absolute (gelu and gelu'), not relatively, where GELU is nearly zero (h < -4), and its exp2 flushes what
# torch keeps as denormals.
ATOL = 2e-6


def _check(got, ref, ulps, what, scale=1.0):
    """bf16 `got` within `ulps` bf16 ulps (relative 2^-7 each) + ATOL * scale of bf16(ref); a non-finite one (fp32 values
    past bf16's largest round to inf) wants a non-finite result."""
    got, ref = got.float(), ref.to(torch.bfloat16).float()
    floor = ATOL * scale
    finite = torch.isfinite(ref)
    close = (got == ref) | ((got - ref).abs() <= ulps * 2.0 ** -7 * ref.abs() + floor)
    bad = finite & ~close
    assert not bad.any(), f"{what}: {int(bad.sum())} elements off, first at {bad.nonzero()[:4].tolist()}: got {got[bad][:4].tolist()} ref {ref[bad][:4].tolist()}"
    bad_nf = ~finite & torch.isfinite(got)
    assert not bad_nf.any(), f"{what}: finite results where the reference is not, at {bad_nf.nonzero()[:4].tolist()}"


@pytest.fixture(scope="module")
def outs():
    return exhaustive_outputs()


def test_patterns_cover_every_bf16_value():
    p = all_patterns().view(torch.int16).int() & 0xFFFF
    assert torch.equal(p, torch.arange(65536, dtype=torch.int32, device=p.device))


def test_gelu_forward_every_pattern(outs):
    h = outs["gelu_h"][0]
    pat = all_patterns()
    # t = bf16(0 + bias): every pattern but -0 (-> +0) and NaN payloads comes through unchanged
    num = ~torch.isnan(pat.float())
    assert torch.equal(h[num].float(), pat[num].float()) and torch.isnan(h[~num].float()).all()
    _check(outs["gelu_out"][0], F.gelu(h.float()), 1, "gelu(h)")
    nan_in = torch.isnan(h.float())
    assert torch.isnan(outs["gelu_out"][0][nan_in].float()).all()


def test_dgelu_every_pattern(outs):
    h, t, out = outs["dgelu_h"], outs["dgelu_t"], outs["dgelu_out"]
    hf = h.float().requires_grad_(True)
    F.gelu(hf).backward(t.float().expand_as(hf))
    for r in range(h.shape[0]):
        tr = t[r, 0].float().item()
        _check(out[r], hf.grad[r], 2, f"dgelu, t = {tr}", scale=abs(tr))
        nan_in = torch.isnan(h[r].float())
        assert torch.isnan(out[r][nan_in].float()).all()


def test_geglu_forward_every_gate_pattern(outs):
    hg, a = outs["geglu_hg"], outs["geglu_a"]
    Fd = a.shape[1]
    h, gate = hg[:, :Fd].float(), hg[:, Fd:].float()
    pat = all_patterns()
    num = ~torch.isnan(pat.float())
    assert torch.equal(gate[:, num], pat[num].float().expand(gate.shape[0], -1))
    # eager: a = bf16(h * bf16(gelu(gate)))
    ref = h * F.gelu(gate).to(torch.bfloat16).float()
    for r in range(a.shape[0]):
        _check(a[r], ref[r], 2, f"geglu, h = {h[r, 0].item()}", scale=abs(h[r, 0].item()))
