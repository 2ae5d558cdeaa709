"""Build the CUDA library in-tree: nvcc, sm_90a (H100) only (no other arch, no CPU build)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "_build", "libdplonk.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def sources():
    deps = [os.path.join(SRC, f) for f in sorted(os.listdir(SRC))]
    deps.append(os.path.join(os.path.dirname(HERE), "include", "dplonk.h"))
    return deps


def is_stale() -> bool:
    return not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in sources())


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return OUT
    import fcntl
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT + ".lock", "w") as lock:          # several ranks of one job may get here together
        fcntl.flock(lock, fcntl.LOCK_EX)
        if not force and not is_stale():            # another process built it while we waited
            return OUT
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        tmp = f"{OUT}.tmp.{os.getpid()}"
        cmd = [nvcc, *NVCC_FLAGS, "-o", tmp, os.path.join(SRC, "dplonk.cu")]
        if verbose:
            cmd[1:1] = ["-Xptxas", "-v"]
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
        os.replace(tmp, OUT)                        # atomic: a loader never sees a half-written library
    return OUT


if __name__ == "__main__":
    print(build(force="-f" in sys.argv, verbose="-v" in sys.argv))
