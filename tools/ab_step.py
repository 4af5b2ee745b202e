"""A/B the whole training step between two builds of the library on one GPU, alternating runs so both see the same clocks.

    python tools/ab_step.py --base carefree-learn_b200/libb200_cflearn_main.so [--new carefree-learn_b200/libb200_cflearn.so]

Each run is `bench.py --gpus 1 --steps 30 --warmup 5 --no-cpu-baseline --dump-outputs DIR` with B200_LIB_PATH pointing at one
build.  Prints the median and spread (min .. max) of `value`, `ms_per_step` and every kernel-alone time of `roofline`, and
whether every run of both builds dumped bit-identical loss / gradient / parameter samples.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import shutil
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH_ARGS = ["--gpus", "1", "--steps", "30", "--warmup", "5", "--no-cpu-baseline"]


def run_bench(lib: str, dump_dir: str) -> dict:
    env = dict(os.environ, B200_LIB_PATH=os.path.abspath(lib))
    res = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *BENCH_ARGS, "--dump-outputs", dump_dir], cwd=ROOT, env=env,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    if res.returncode != 0 or not lines:
        raise RuntimeError(f"bench.py failed with {lib} (exit {res.returncode}):\n{res.stdout[-3000:]}")
    return json.loads(lines[-1])


def metrics(line: dict) -> dict:
    out = {"value": line["value"], "ms_per_step": line["ms_per_step"]}
    roof = line["roofline"]
    for k in [roof, *roof["others"]]:
        out[k["kernel"] + " [ms]"] = k["kernel_ms"]
    return out


def load_dump(d: str) -> dict:
    return {f: np.load(os.path.join(d, f)) for f in sorted(os.listdir(d)) if f.endswith(".npy")}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="library build to compare against (e.g. the parent commit's)")
    ap.add_argument("--new", default=os.path.join(ROOT, "carefree-learn_b200", "libb200_cflearn.so"))
    ap.add_argument("--runs", type=int, default=3, help="runs per build (alternating)")
    ap.add_argument("--out", default=None, help="directory for the bench JSON lines (default: a temporary directory)")
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp(prefix="ab_step_")
    os.makedirs(out, exist_ok=True)
    dump_root = tempfile.mkdtemp(prefix="ab_step_dumps_")  # tens of MB per run: compared, then removed
    builds = {"base": args.base, "new": args.new}
    results = {k: [] for k in builds}
    dumps = {k: [] for k in builds}
    for i in range(args.runs):
        for name, lib in builds.items():
            d = os.path.join(dump_root, f"{name}_{i}")
            line = run_bench(lib, d)
            results[name].append(line)
            dumps[name].append(d)
            print(f"run {i} {name}: {line['value']} samples/s, {line['ms_per_step']} ms/step", flush=True)
    with open(os.path.join(out, "ab_step.jsonl"), "w") as f:
        for name in builds:
            for line in results[name]:
                f.write(json.dumps({"build": name, **line}) + "\n")

    first = results["new"][0]
    print(f"\nclocks (first run of the new build): {json.dumps(first.get('clocks'))}")
    med = {}
    print(f"\n{'metric':<90} {'base median (min .. max)':>32} {'new median (min .. max)':>32} {'new/base':>9}")
    keys = list(metrics(results["base"][0]))
    for key in keys:
        row = []
        for name in builds:
            vals = [metrics(r)[key] for r in results[name]]
            med[name] = statistics.median(vals)
            row.append(f"{med[name]:.4g} ({min(vals):.4g} .. {max(vals):.4g})")
        print(f"{key:<90} {row[0]:>32} {row[1]:>32} {med['new'] / med['base']:>9.3f}")

    ref = load_dump(dumps["base"][0])
    identical = True
    for name in builds:
        for d in dumps[name]:
            got = load_dump(d)
            if got.keys() != ref.keys() or any(got[k].tobytes() != ref[k].tobytes() for k in ref):
                identical = False
                diff = [k for k in ref if k not in got or got[k].tobytes() != ref[k].tobytes()]
                print(f"dump {d} differs from {dumps['base'][0]} in {diff}")
    shutil.rmtree(dump_root, ignore_errors=True)
    print(f"\ndumps bit-identical across all runs of both builds: {identical} ({len(ref)} arrays each)")
    print(f"bench JSON lines in {out}/ab_step.jsonl")


if __name__ == "__main__":
    main()
