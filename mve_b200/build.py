"""Builds mve_b200/libb200mvs.so (sm_90a) in-tree with nvcc."""
from __future__ import annotations

import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, "libb200mvs.so")
SOURCES = [os.path.join(HERE, "csrc", "b200mvs.cu"), os.path.join(HERE, "csrc", "depthmap.cu")]
DEPS = SOURCES + [os.path.join(HERE, "csrc", "patch_opt.cuh"), os.path.join(HERE, "csrc", "patch_thread.cuh"), os.path.join(HERE, "csrc", "patch_warp.cuh"),
               os.path.join(HERE, "csrc", "pset_device.cuh"), os.path.join(HERE, "csrc", "host_common.cuh"),
               os.path.join(HERE, "csrc", "plan_device.cuh"), os.path.join(HERE, "csrc", "undistort.cuh"),
               os.path.join(HERE, "csrc", "prior_seed.cuh"), os.path.join(HERE, "csrc", "prior_align.cuh"),
               os.path.join(ROOT, "include", "b200mvs.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v"]


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", LIB] + SOURCES
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        print(res.stdout)
        print(res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed for libb200mvs.so")
    with open(os.path.join(HERE, "csrc", "ptxas_info.txt"), "w") as f:
        f.write(res.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
