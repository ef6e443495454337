"""Build libb2gram.so (sm_90a, H100) in-tree with nvcc.  No torch, no JIT cache: the .so ships with the tree."""
from __future__ import annotations

import glob
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libb2gram.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
    "-Xptxas", "-v",
]


def find_nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: libb2gram.so cannot be built (there is no CPU fallback)")
    return nvcc


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def is_stale() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [
        os.path.join(os.path.dirname(PKG_DIR), "include", "b2gram.h")]
    return any(os.path.getmtime(p) > t for p in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile into a temporary file and rename it into place (a concurrent dlopen never sees a half-written library);
    an exclusive file lock serialises the ranks of a torchrun launch, the late ones find the library fresh."""
    if not force and not is_stale():
        return LIB_PATH
    import fcntl
    log = ""
    with open(os.path.join(PKG_DIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not is_stale():       # another process built it while we waited
                return LIB_PATH
            tmp = f"{LIB_PATH}.{os.getpid()}.tmp"
            cmd = [find_nvcc()] + NVCC_FLAGS + ["-o", tmp] + sources() + ["-ldl"]
            proc = subprocess.run(cmd, capture_output=True, text=True)
            log = proc.stdout + proc.stderr
            log_tmp = os.path.join(PKG_DIR, f"build.log.{os.getpid()}.tmp")
            with open(log_tmp, "w") as fh:
                fh.write(" ".join(cmd) + "\n" + log)
            os.replace(log_tmp, os.path.join(PKG_DIR, "build.log"))
            if proc.returncode != 0:
                if os.path.exists(tmp):
                    os.remove(tmp)
                raise RuntimeError("nvcc failed:\n" + log[-6000:])
            os.replace(tmp, LIB_PATH)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    if verbose:
        print(log)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
