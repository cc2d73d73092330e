"""Build liblightglue_b200.so in-tree with nvcc for sm_90a (``make -C lightglue_b200/csrc``).

The library is plain CUDA C++ behind a C ABI (include/lightglue_b200.h); it does not link against
torch.  nvcc cross-compiles without a GPU, so this runs in the CPU-only build container and the
resulting .so travels to the GPU box with the repo snapshot.
"""
from __future__ import annotations

import fcntl
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "liblightglue_b200.so")


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".h", ".cuh")) or f == "Makefile"]
    srcs.append(os.path.join(os.path.dirname(HERE), "include", "lightglue_b200.h"))
    srcs.append(os.path.join(os.path.dirname(HERE), "include", "superpoint_b200.h"))
    srcs.append(os.path.join(os.path.dirname(HERE), "include", "aliked_b200.h"))
    srcs.append(os.path.join(os.path.dirname(HERE), "include", "sift_b200.h"))
    return any(os.path.getmtime(s) > t for s in srcs)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile the CUDA library if it is missing or older than its sources; returns its path.  Serialised with a
    file lock: the ranks of a torchrun job import the package at the same time and must not run `make` concurrently
    (the first one builds, the others then find the library up to date)."""
    if not (force or _stale()):
        return LIB
    with open(os.path.join(CSRC, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if force or _stale():
                jobs = str(min(8, os.cpu_count() or 1))
                cmd = ["make", "-C", CSRC, "-j", jobs] + (["-B"] if force else [])
                res = subprocess.run(cmd, capture_output=True, text=True)
                if verbose or res.returncode != 0:
                    print(res.stdout[-4000:])
                    print(res.stderr[-8000:])
                if res.returncode != 0:
                    raise RuntimeError("building liblightglue_b200.so failed (see output above)")
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
