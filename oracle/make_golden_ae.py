"""TEST INFRASTRUCTURE ONLY -- pins ``oracle/ae_oracle.py`` against the real reference ``AttentionAutoEncoderKL``
(cflearn/modules/cv/ae/kl.py, imported unmodified through oracle/load_reference.py) and writes
  tests/golden/ae_kl_f8_state_dict_keys.json   keys, shapes and parameter count of the zoo's ae/kl.f8 config;
  tests/golden/ae_kl_tiny_reference.pt         the reference's own decode (CPU fp32) of a tiny config, with and without head.
Needs a carefree-learn checkout (oracle/load_reference.py):  python oracle/make_golden_ae.py"""
from __future__ import annotations

import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ae_oracle as ao  # noqa: E402
from load_reference import load_reference_modules  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")


def reference_ae(cfg):
    load_reference_modules()
    from cflearn.modules.cv.ae.kl import AttentionAutoEncoderKL

    return AttentionAutoEncoderKL(cfg["img_size"], cfg["in_channels"], cfg["out_channels"], cfg["inner_channels"], cfg["latent_channels"],
                                  cfg["channel_multipliers"], embedding_channels=cfg["embedding_channels"],
                                  num_res_blocks=cfg["num_res_blocks"])


def main():
    load_reference_modules()
    from cflearn.modules.cv.common import DecoderInputs

    f8 = reference_ae(ao.ae_config("kl_f8"))
    keys = {"config": ao.ae_config("kl_f8"), "parameters": sum(p.numel() for p in f8.parameters()),
            "keys": [[k, list(v.shape)] for k, v in f8.state_dict().items()]}
    os.makedirs(GOLDEN, exist_ok=True)
    with open(os.path.join(GOLDEN, "ae_kl_f8_state_dict_keys.json"), "w") as f:
        json.dump(keys, f, indent=0)
    print(f"wrote tests/golden/ae_kl_f8_state_dict_keys.json ({len(keys['keys'])} keys, {keys['parameters']} parameters)")

    cfg = ao.ae_config("kl_tiny")
    m = reference_ae(cfg).eval()
    shapes = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    sd = ao.synthetic_state_dict(shapes, seed=0)
    m.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(5)
    z = torch.randn(2, cfg["embedding_channels"], cfg["img_size"] // 2, cfg["img_size"] // 2, generator=g)
    ref = {}
    with torch.no_grad():
        for no_head in (False, True):
            out = m.decode(DecoderInputs(z=z.clone(), no_head=no_head))
            assert torch.equal(ao.decode(sd, z, no_head=no_head), out), f"oracle differs from the reference (no_head={no_head})"
            ref["no_head" if no_head else "head"] = out
    torch.save({"config_name": "kl_tiny", "shapes": shapes, "weights_seed": 0, "z": z, "reference": ref},
               os.path.join(GOLDEN, "ae_kl_tiny_reference.pt"))
    print("wrote tests/golden/ae_kl_tiny_reference.pt: the oracle's decode is bit-identical to the reference's, with and without head")


if __name__ == "__main__":
    main()
