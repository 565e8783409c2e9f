"""Build libb200mppi.so (the C-ABI of include/b200mppi.h) in-tree with nvcc for sm_90a (H100).

    python mppi_numba_b200/build.py   (or: python __graft_entry__.py)   # rebuild if sources are newer than the .so

nvcc cross-compiles without a GPU; the built .so is git-ignored.
"""
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libb200mppi.so")
SOURCES = ["api.cu", "rollout.cu", "rollout_win.cu", "reduce.cu", "sample.cu", "p2p.cu"]
HEADERS = ["common.cuh", "kernels.h", os.path.join(ROOT, "include", "b200mppi.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-ftz=true", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _objects():
    return [os.path.join(CSRC, src.replace(".cu", ".o")) for src in SOURCES]


def _stale():
    hdrs = [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    return (any(_newer(o, [os.path.join(CSRC, s)] + hdrs) for s, o in zip(SOURCES, _objects()))
            or _newer(LIB, _objects()))


def build_library(force=False, verbose=False):
    """Compile every .cu under csrc/ and link the shared library.  Returns its path.
    Serialised with a file lock: the ranks of a torchrun launch all call this at start-up, the first one
    builds (if anything is stale), the others find everything up to date once they hold the lock.
    An up-to-date build writes nothing, so a built tree may be read-only."""
    if not force and not _stale():
        return LIB
    import fcntl
    with open(os.path.join(CSRC, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(force, verbose):
    extra = os.environ.get("B200MPPI_NVCC_FLAGS", "").split()      # A/B builds of compile-time switches (e.g. -DSG_POPC_VARIANT=0)
    hdrs = [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    objs = _objects()
    log = []
    for src, o in zip(SOURCES, objs):
        s = os.path.join(CSRC, src)
        if force or _newer(o, [s] + hdrs):
            cmd = [NVCC] + FLAGS + extra + ["-c", s, "-o", o]
            r = subprocess.run(cmd, capture_output=True, text=True)
            log.append(r.stderr)
            if r.returncode != 0:
                raise RuntimeError("nvcc failed for %s:\n%s" % (src, r.stderr))
    if force or _newer(LIB, objs):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ARCH
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s" % r.stderr)
    if verbose:
        sys.stderr.write("".join(log))
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose=True))
