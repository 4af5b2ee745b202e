"""Put all 65,536 bf16 bit patterns through the exact-erf GELU epilogues of two builds of the library and compare the outputs
byte for byte (NaN payloads included).

    python tools/epilogue_ab.py --base carefree-learn_b200/libb200_cflearn_main.so [--new carefree-learn_b200/libb200_cflearn.so]

Each build runs in its own process (B200_LIB_PATH selects it) and saves its outputs; the script then reports, per output,
whether the two builds agree bit for bit.  The inputs (`exhaustive_outputs`):
  * EPI_BIAS_GELU_BF16: A = 0, so t = the bias; N = 65,536 columns, one pattern per column.
  * EPI_DGELU_BF16: aux h = every pattern in every row, the upstream value t = bf16(acc) one of DGELU_T per row
    (A's first column is t, B's first row is 1, everything else 0).
  * GEGLU forward: the gate bias runs over every pattern, h = one of GEGLU_H per row (x's first column, W1's h rows 1).
"""
from __future__ import annotations

import argparse
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DGELU_T = [1.0, -1.0, 0.3, -2.5, 2.0 ** 60, -(2.0 ** -60), 0.0, 448.0]
GEGLU_H = [1.0, -1.0, 3.5, -0.0078125]
K = 64


def all_patterns(dev: str = "cuda") -> torch.Tensor:
    """Every bf16 bit pattern, in order (0x0000 .. 0xffff)."""
    return torch.arange(65536, dtype=torch.int32, device=dev).to(torch.int16).view(torch.bfloat16)


def exhaustive_outputs(dev: str = "cuda") -> dict:
    """Run the three epilogues over every bf16 pattern; returns their inputs and outputs (bf16 tensors)."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import cflearn_b200  # noqa: F401
    from cflearn_b200 import ops

    pat = all_patterns(dev)
    N = pat.numel()
    bf = dict(dtype=torch.bfloat16, device=dev)
    # GELU forward with the dual output: t = bf16(0 + bias)
    a = torch.zeros(1, K, **bf)
    w = torch.zeros(N, K, **bf)
    gelu_out1 = torch.empty(1, N, **bf)
    gelu_out0 = ops.gemm(a, w, bias=pat, epilogue=ops.EPI_BIAS_GELU_BF16, out1=gelu_out1)
    # dGELU: out0 = bf16(t * gelu'(h)), t = DGELU_T[row], h = every pattern
    dy = torch.zeros(len(DGELU_T), K, **bf)
    dy[:, 0] = torch.tensor(DGELU_T, **bf)
    w2 = torch.zeros(K, N, **bf)
    w2[0] = 1.0
    h = pat.unsqueeze(0).repeat(len(DGELU_T), 1).contiguous()
    dgelu = ops.gemm(dy, w2, b_mn_major=True, epilogue=ops.EPI_DGELU_BF16, aux=h)
    # GEGLU forward: h = GEGLU_H[row], gate = bf16(0 + gate bias) = every pattern
    x = torch.zeros(len(GEGLU_H), K, **bf)
    x[:, 0] = torch.tensor(GEGLU_H, **bf)
    w1 = torch.zeros(2 * N, K, **bf)
    w1[:N, 0] = 1.0
    b1 = torch.cat([torch.zeros(N, **bf), pat])
    hg, act = ops.geglu(x, w1, b1)
    torch.cuda.synchronize()
    return {"gelu_h": gelu_out0, "gelu_out": gelu_out1, "dgelu_h": h, "dgelu_t": dy[:, :1], "dgelu_out": dgelu,
            "geglu_hg": hg, "geglu_a": act}


def dump(out_dir: str) -> None:
    os.makedirs(out_dir, exist_ok=True)
    for name, t in exhaustive_outputs().items():
        np.save(os.path.join(out_dir, name + ".npy"), t.contiguous().view(torch.int16).cpu().numpy())


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", help="library build to compare against (e.g. the parent commit's)")
    ap.add_argument("--new", default=os.path.join(ROOT, "carefree-learn_b200", "libb200_cflearn.so"))
    ap.add_argument("--dump", help=argparse.SUPPRESS)  # child mode: save this build's outputs to the directory
    args = ap.parse_args()
    if args.dump:
        dump(args.dump)
        return
    if not args.base:
        ap.error("--base is required")
    tmp = tempfile.mkdtemp(prefix="epilogue_ab_")
    dirs = {}
    for name, lib in (("base", args.base), ("new", args.new)):
        dirs[name] = os.path.join(tmp, name)
        env = dict(os.environ, B200_LIB_PATH=os.path.abspath(lib))
        subprocess.run([sys.executable, os.path.abspath(__file__), "--dump", dirs[name]], env=env, check=True)
    identical = True
    for f in sorted(os.listdir(dirs["base"])):
        a, b = np.load(os.path.join(dirs["base"], f)), np.load(os.path.join(dirs["new"], f))
        same = a.shape == b.shape and a.tobytes() == b.tobytes()
        identical &= same
        ndiff = int((a != b).sum()) if a.shape == b.shape else -1
        print(f"{f[:-4]:<12} {str(a.shape):<14} {'identical' if same else f'DIFFERS at {ndiff} elements'}")
    shutil.rmtree(tmp, ignore_errors=True)
    print(f"\nall outputs bit-identical between {args.base} and {args.new}: {identical}")
    sys.exit(0 if identical else 1)


if __name__ == "__main__":
    main()
