"""The wgmma kernels must compile for sm_90a without ptxas serialising their wgmma pipelines (C7510: a function call such
as a printf between wgmma groups makes every MMA wait for the previous one) and without spills or a stack frame."""
import os
import re
import shutil
import subprocess

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "carefree-learn_b200", "csrc")
NVCC = os.path.join(os.environ.get("CUDA_HOME") or "/usr/local/cuda", "bin", "nvcc")
if not os.path.isfile(NVCC):
    NVCC = shutil.which("nvcc")


@pytest.mark.skipif(NVCC is None, reason="nvcc not available")
@pytest.mark.parametrize("src", ["gemm_sm90.cu", "attention_sm90.cu"])
def test_wgmma_not_serialised_and_no_spills(src, tmp_path):
    res = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v",
                          "-c", os.path.join(CSRC, src), "-o", str(tmp_path / "k.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    log = res.stdout
    assert res.returncode == 0, log[-4000:]
    assert "C7510" not in log, "\n".join(ln for ln in log.splitlines() if "C7510" in ln)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert frames, log[-2000:]
    assert all(f == ("0", "0", "0") for f in frames), log
