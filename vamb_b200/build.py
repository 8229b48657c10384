"""Build recipe for the in-tree CUDA extension ``vamb_b200/_vk.so`` (sm_90a only).

Plain ``nvcc -shared``: the library exposes the C ABI of include/vamb_b200.h and links
the CUDA runtime statically, so it has no torch / Python dependency.  The built ``.so`` is
git-ignored: ``__graft_entry__.build()`` makes it in the tree.
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_vk.so")
OUT_TIMELINE = os.path.join(HERE, "_vk_timeline.so")  # diagnostic build with in-kernel time stamps
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-ffp-contract=off",
    "--expt-relaxed-constexpr",
    "-shared",
]


def sources() -> list:
    return sorted(glob.glob(os.path.join(HERE, "csrc", "*.cu")))


def needs_build() -> bool:
    if not os.path.isfile(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = sources() + glob.glob(os.path.join(HERE, "csrc", "*.cuh")) + [
        os.path.join(HERE, "..", "include", "vamb_b200.h")
    ]
    return any(os.path.getmtime(p) > t for p in deps)


def build(force: bool = False, verbose: bool = False, timeline: bool = False) -> str:
    if timeline:
        force = True
    if not force and not needs_build():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    out = OUT_TIMELINE if timeline else OUT
    cmd = ([nvcc] + NVCC_FLAGS + (["-DVK_TIMELINE"] if timeline else []) + (["-Xptxas", "-v"] if verbose else [])
           + ["-o", out] + sources() + ["-lcuda"])
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building vamb_b200/_vk.so")
    return out


if __name__ == "__main__":
    print(build(force=True, verbose="-v" in sys.argv, timeline="--timeline" in sys.argv))
