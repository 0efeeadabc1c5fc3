"""Register budget of the headline step kernel, highway_step_kernel<64, true>: 128 registers per thread is what lets
two 256-thread blocks share an SM, and its few spilled words sit off the hot path.  Cross-compiles hwy_highway.cu for
sm_90a (no GPU needed) with the library's flags and reads ptxas' report."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# ptxas of CUDA 12.9 for sm_90a before dense env segments existed: 156 B spill stores, 268 B spill loads
MAX_REGISTERS, MAX_SPILL_STORES, MAX_SPILL_LOADS = 128, 156 + 16, 268 + 16


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_headline_step_kernel_registers_and_spills(tmp_path):
    from highwayenv_b200 import build

    flags = [f for f in build.NVCC_FLAGS if f not in ("-Xcompiler", "-fPIC", "-shared")]
    out = subprocess.run(["nvcc"] + flags + ["-Xptxas", "-v", "-cubin", "-o", str(tmp_path / "k.cubin"),
                                             os.path.join(ROOT, "highwayenv_b200", "csrc", "hwy_highway.cu")],
                         cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-800:]
    lines = out.stderr.splitlines()
    # both instantiations: TPE-thread segments (small batches) and dense segments (the headline's 5 envs per block)
    found = [k for k, l in enumerate(lines) if "Compiling entry function" in l and "highway_step_kernelILi64ELb1E" in l]
    assert len(found) == 2, found
    for k in found:
        report = " ".join(lines[k + 1:k + 4])
        stores = int(re.search(r"(\d+) bytes spill stores", report).group(1))
        loads = int(re.search(r"(\d+) bytes spill loads", report).group(1))
        regs = int(re.search(r"Used (\d+) registers", report).group(1))
        assert regs <= MAX_REGISTERS, (lines[k], report)
        assert stores <= MAX_SPILL_STORES and loads <= MAX_SPILL_LOADS, (lines[k], report)
