"""TEST INFRASTRUCTURE -- build recipe for the oracle's C inner loops.

gcc only; output goes to oracle/_build/ (git-ignored, built by build()).
``-ffp-contract=off`` keeps every a*b+c unfused unless written as fmaf();
``-mfma`` makes fmaf() a single hardware instruction (IEEE-exact either way).
"""
import os
import subprocess


def build(force: bool = False) -> str:
    here = os.path.dirname(os.path.abspath(__file__))
    src = os.path.join(here, "csrc", "oracle_kernels.c")
    out_dir = os.path.join(here, "_build")
    out = os.path.join(out_dir, "liboracle.so")
    os.makedirs(out_dir, exist_ok=True)
    if not force and os.path.isfile(out) and os.path.getmtime(out) >= os.path.getmtime(src):
        return out
    cmd = ["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-mfma", "-fvisibility=hidden",
           "-o", out, src, "-lm"]
    subprocess.run(cmd, check=True)
    return out


if __name__ == "__main__":
    print(build(force=True))
