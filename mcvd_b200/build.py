"""Build the sm_90a (H100) C-ABI library ``mcvd_b200/_lib/libmcvd_b200.so`` in-tree with nvcc.

``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` cross-compiles without a GPU; the .so is
git-ignored but travels to the GPU box with the repo snapshot.  Rebuilds only when a source is
newer than the library.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "_lib")
LIB = os.path.join(LIBDIR, "libmcvd_b200.so")
SOURCES = ["api.cu", "elementwise.cu", "conv_simt.cu", "conv_smalln.cu", "attention_simt.cu", "conv_umma.cu",
           "attention_umma.cu"]
HEADERS = [os.path.join(CSRC, "mcvd_common.cuh"), os.path.join(CSRC, "umma_ptx.cuh"), os.path.join(CSRC, "wgmma_ops.cuh"), os.path.join(os.path.dirname(HERE), "include", "mcvd_b200.h")]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in sources() + HEADERS)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile and link under a cross-process file lock (torchrun starts one rank per GPU: with a missing or
    stale library they would otherwise all write the same .o / .so); objects and the library are written to
    temporary names and renamed into place, so a concurrent dlopen never sees a half-written file."""
    import fcntl
    os.makedirs(LIBDIR, exist_ok=True)
    with open(os.path.join(LIBDIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(force: bool, verbose: bool) -> str:
    if not force and not needs_build():          # another process may have built it while we waited for the lock
        return LIB
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(LIBDIR, os.path.basename(src).replace(".cu", ".o"))
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(
                os.path.getmtime(p) for p in [src] + HEADERS):
            continue
        tmp = obj + f".tmp{os.getpid()}"
        cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
               "-Xcompiler", "-fPIC", "-Xptxas", "-v" if verbose else "-warn-spills", "-c", src, "-o", tmp]
        procs.append((src, tmp, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = None
    for src, tmp, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = failed or f"nvcc failed for {src}:\n{out}"
            if os.path.exists(tmp):
                os.remove(tmp)
            continue
        os.replace(tmp, obj)
        if verbose or "warning" in out.lower():
            sys.stderr.write(out)
    if failed:
        raise RuntimeError(failed)
    tmp_lib = LIB + f".tmp{os.getpid()}"
    cmd = [_nvcc(), "-shared", "-o", tmp_lib] + objs + ["-cudart", "static"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    os.replace(tmp_lib, LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
