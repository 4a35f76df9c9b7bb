"""Compiler diagnostics of the wgmma GEMM / implicit-GEMM convolution kernels (csrc/gemm_tc.cu), all 90 instantiations.

The file is compiled once, with the Makefile's flags, and ptxas's report is checked: every instantiation is built, no
wgmma chain is serialised (diagnostic C7520: every MMA would wait for the one before it) except in the stream-K kernels,
where it already was, and no instantiation spills more than the table below. Needs nvcc, not a GPU: the kernels are
cross-compiled for sm_90a."""
import itertools
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "multi-task-transformer_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC) and shutil.which(NVCC) is None, reason="nvcc not found")

# An instantiation: (kind, nsplit, tile width, activation, outputs). kind: "single" (gemm_tc_kernel), "streamk"
# (gemm_tc_kernel with SK, 256-wide tiles only) or "grouped" (gemm_tc_grouped_kernel); activation: mtt_act (0 none,
# 1 GELU, 2 ReLU); outputs: 1 fp32, 2 split-bf16, 3 both.
EPILOGUES = list(itertools.product((0, 1, 2), (1, 2, 3)))
KERNELS = ([("single", n, bn) + e for n in (1, 2) for bn in (128, 256) for e in EPILOGUES]
           + [("streamk", n, 256) + e for n in (1, 2) for e in EPILOGUES]
           + [("grouped", n, bn) + e for n in (1, 2) for bn in (128, 256) for e in EPILOGUES])

# Spill bytes (stores, loads) of the 128 x 256 instantiations that spill, as nvcc 12.9 builds them; every other
# instantiation spills nothing. The 128 x 256 tile's accumulator leaves few registers for the epilogue.
SPILLS = {
    ("single", 1, 256, 0, 3): (8, 4), ("single", 1, 256, 1, 1): (4, 8), ("single", 1, 256, 1, 2): (4, 8),
    ("single", 1, 256, 1, 3): (36, 36), ("single", 1, 256, 2, 3): (8, 4),
    ("single", 2, 256, 0, 3): (12, 12), ("single", 2, 256, 1, 1): (4, 8), ("single", 2, 256, 1, 2): (4, 8),
    ("single", 2, 256, 1, 3): (52, 52), ("single", 2, 256, 2, 3): (12, 12),
    ("streamk", 1, 256, 0, 1): (16, 20), ("streamk", 1, 256, 0, 2): (12, 16), ("streamk", 1, 256, 0, 3): (20, 24),
    ("streamk", 1, 256, 1, 1): (20, 24), ("streamk", 1, 256, 1, 2): (20, 24), ("streamk", 1, 256, 1, 3): (64, 68),
    ("streamk", 1, 256, 2, 1): (20, 24), ("streamk", 1, 256, 2, 2): (20, 24), ("streamk", 1, 256, 2, 3): (20, 24),
    ("streamk", 2, 256, 0, 1): (16, 16), ("streamk", 2, 256, 0, 2): (12, 16), ("streamk", 2, 256, 0, 3): (32, 36),
    ("streamk", 2, 256, 1, 1): (20, 24), ("streamk", 2, 256, 1, 2): (20, 24), ("streamk", 2, 256, 1, 3): (64, 68),
    ("streamk", 2, 256, 2, 1): (16, 20), ("streamk", 2, 256, 2, 2): (20, 24), ("streamk", 2, 256, 2, 3): (32, 36),
    ("grouped", 1, 256, 1, 1): (4, 8), ("grouped", 1, 256, 1, 2): (4, 8), ("grouped", 1, 256, 1, 3): (40, 44),
    ("grouped", 2, 256, 0, 3): (4, 8), ("grouped", 2, 256, 1, 1): (4, 8), ("grouped", 2, 256, 1, 2): (4, 8),
    ("grouped", 2, 256, 1, 3): (56, 60), ("grouped", 2, 256, 2, 3): (4, 8),
}

# The stream-K kernels' wgmma chains are serialised (C7520); no other kernel's may be.
SERIALISED = {k for k in KERNELS if k[0] == "streamk"}


def mangled(kernel):
    kind, n, bn, act, out = kernel
    if kind == "grouped":
        return f"_ZN3mtt22gemm_tc_grouped_kernelILi{n}ELi{bn}ELi{act}ELi{out}EEEv"
    return f"_ZN3mtt14gemm_tc_kernelILi{n}ELi{bn}ELb{int(kind == 'streamk')}ELi{act}ELi{out}EEEv"


def makefile_flags():
    mk = open(os.path.join(CSRC, "Makefile")).read()
    var = dict(re.findall(r"^(\w+) := (.*)$", mk, re.M))
    return re.sub(r"\$\((\w+)\)", lambda m: var[m.group(1)], var["NVCCFLAGS"]).split()


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    out = tmp_path_factory.mktemp("gemm_build") / "gemm_tc.o"
    r = subprocess.run([NVCC, *makefile_flags(), "-c", os.path.join(CSRC, "gemm_tc.cu"), "-o", str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stdout + r.stderr


def test_gemm_all_instantiations_built(ptxas_log):
    built = set(re.findall(r"Compiling entry function '(\S+)'", ptxas_log))
    assert len(KERNELS) == 90
    missing = [k for k in KERNELS if not any(f.startswith(mangled(k)) for f in built)]
    assert not missing, missing
    assert len(built) == len(KERNELS), sorted(built)


def test_gemm_no_serialised_wgmma(ptxas_log):
    serialised = {f for f in re.findall(r"C7520\).*function '(\S+)'", ptxas_log)}
    unexpected = [k for k in KERNELS if k not in SERIALISED and any(f.startswith(mangled(k)) for f in serialised)]
    assert not unexpected, unexpected


def test_gemm_spills_within_table(ptxas_log):
    props = re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", ptxas_log)
    grown = []
    for k in KERNELS:
        got = [(int(s), int(ld)) for f, s, ld in props if f.startswith(mangled(k))]
        assert len(got) == 1, (k, got)
        limit = SPILLS.get(k, (0, 0))
        if got[0][0] > limit[0] or got[0][1] > limit[1]:
            grown.append((k, got[0], limit))
    assert not grown, grown
