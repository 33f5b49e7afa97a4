"""Build rodio_b200/librodio_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache, the .so travels with the repo)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "librodio_b200.so")
SOURCES = ["rb_api.cu", "rb_kernels.cu", "rb_fused.cu", "rb_fx.cu", "rb_lanes.cu", "rb_lanes_batch.cu", "rb_p2p.cu", "rb_master.cu"]
HEADERS = ["rb_internal.h", "rb_dsp.cuh", "rb_fused.h", "rb_fused_rows.h", "rb_lanes.h", "rb_lanes_core.h", "rb_duo_core.h", "rb_lanes_plan.h", "rb_session_plan.h", "rb_simt.h", "rb_p2p.h", os.path.join("..", "..", "include", "rodio_b200.h")]

NVCC_FLAGS = [
    "-O3", "-std=c++17",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "--fmad=false",            # rustc never contracts a*b+c; bit parity depends on it
    "-Xcompiler", "-fPIC,-ffp-contract=off,-fno-fast-math",
    "-cudart", "static",
    "--shared",
    "--threads", "0",          # the translation units compile side by side
    "-ldl",                    # libnccl is loaded at first use (rb_comm_*)
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, extra_flags=(), out: str = LIB) -> str:
    if not force and out == LIB and not needs_build():
        return LIB
    cmd = [_nvcc()] + NVCC_FLAGS + list(extra_flags) + (["-Xptxas", "-v"] if verbose else []) + \
        [os.path.join(CSRC, s) for s in SOURCES] + ["-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed building librodio_b200.so")
    if verbose:
        sys.stderr.write(r.stdout + r.stderr)
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
