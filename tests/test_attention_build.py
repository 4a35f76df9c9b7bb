"""Compiler diagnostics of the fused attention kernel (csrc/attention5_tc.cu), both instantiations (NSPLIT 1 and 2).

ptxas must neither serialise the wgmma chains (diagnostic C7520: every MMA would wait for the one before it) nor spill
registers to local memory. Needs nvcc, not a GPU: the kernel is cross-compiled for sm_90a."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "multi-task-transformer_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC) and shutil.which(NVCC) is None, reason="nvcc not found")


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    out = tmp_path_factory.mktemp("attn_build") / "attention5_tc.o"
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", os.path.join(CSRC, "attention5_tc.cu"),
                        "-o", str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stdout + r.stderr


@pytest.mark.parametrize("nsplit", [1, 2])
def test_attention_kernel_no_serialised_wgmma_no_spills(ptxas_log, nsplit):
    fn = f"attention5_kernelILi{nsplit}E"
    assert fn in ptxas_log
    serialised = [ln for ln in ptxas_log.splitlines() if "C7520" in ln and fn in ln]
    assert not serialised, serialised
    m = re.search(r"Function properties for \S*" + fn + r"\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", ptxas_log)
    assert m, ptxas_log
    assert (int(m.group(2)), int(m.group(3))) == (0, 0), m.group(0)
