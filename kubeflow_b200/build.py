"""Build libkbo.so in-tree with nvcc for sm_90a (the only target).  Used by __graft_entry__.build()."""
from __future__ import annotations

import glob
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libkbo.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(HERE, "..", "include", "kbo.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu into kubeflow_b200/libkbo.so (sm_90a only).  Safe under torchrun: ranks serialise on a lock
    file and the library is written to a temporary name first, so no rank ever dlopens a half-written .so."""
    import fcntl
    if not force and not needs_build():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    with open(LIB + ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not needs_build():      # another rank built it while we waited
                return LIB
            tmp = LIB + f".tmp{os.getpid()}"
            cmd = [nvcc, "-shared", "-Xcompiler", "-fPIC", "-std=c++17", "-O3", "-lineinfo", *ARCH, "-o", tmp, *sources()]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            subprocess.run(cmd, check=True)
            os.replace(tmp, LIB)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
