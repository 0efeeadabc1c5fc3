"""In-tree build of the sm_90a kernels:  python -m highwayenv_b200.build

nvcc cross-compiles without a GPU.  -fmad=false: the fp64 simulation follows the
reference's separately rounded operations (explicit fma() only where numpy fuses).
"""
from __future__ import annotations

import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = [os.path.join(_HERE, "csrc", f) for f in ("hwy_highway.cu", "hwy_network.cu", "hwy_observe.cu", "hwy_plan.cu", "hwy_copy.cu", "hwy_lane_keeping.cu", "hwy_lanes_debug.cu")]
DEPS = SRC + [os.path.join(_HERE, "csrc", h) for h in ("hwy_math.cuh", "hwy_device.cuh", "hwy_lanes.cuh", "hwy_bicycle.cuh", "hwy_abi.h", "hwy_highway_step.cuh", "hwy_highway_reset.cuh")] + [
    os.path.join(os.path.dirname(_HERE), "include", "hwyb200.h")]
OUT = os.path.join(_HERE, "csrc", "libhwyb200.so")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-fmad=false", "-Xcompiler", "-fPIC", "-shared", "--threads", "7",  # the seven sources compile concurrently
]


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= max(map(os.path.getmtime, DEPS)):
        return OUT
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT] + SRC
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
