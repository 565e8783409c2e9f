"""Compile the reference package (mit-acl/mppi_numba) to bytecode under oracle/_ref/ -- TEST INFRASTRUCTURE.

The GPU-side parity test (tests/test_gpu_vs_reference.py) and bench.py's `numba_cuda_baseline` leg run the
UNMODIFIED reference's Numba-CUDA kernels next to the engine.  The reference cannot be part of this repository and
is not installed where the GPU runs, so build() compiles it here, where it is readable (ref_loader.REFERENCE_ROOT),
into git-ignored sourceless bytecode: oracle/_ref/mppi_numba/*.pyc, importable with oracle/_ref on sys.path (Numba
compiles kernels from bytecode).  Without a readable reference nothing is built and the consumers report it missing.
"""
import glob
import os
import py_compile

HERE = os.path.dirname(os.path.abspath(__file__))
REF_OUT = os.path.join(HERE, "_ref")


def compiled_reference():
    """The directory to put on sys.path to import the compiled reference, or None if it was not built."""
    return REF_OUT if os.path.isfile(os.path.join(REF_OUT, "mppi_numba", "mppi.pyc")) else None


def build_reference():
    from oracle.ref_loader import REFERENCE_ROOT
    src = os.path.join(REFERENCE_ROOT, "mppi_numba")
    if not os.access(os.path.join(src, "mppi.py"), os.R_OK):
        return None
    dst = os.path.join(REF_OUT, "mppi_numba")
    os.makedirs(dst, exist_ok=True)
    for path in sorted(glob.glob(os.path.join(src, "*.py"))):
        name = os.path.basename(path)
        out = os.path.join(dst, name[:-3] + ".pyc")
        if not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(path):
            py_compile.compile(path, cfile=out, dfile=os.path.join("mppi_numba", name), doraise=True,
                               invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)
    return REF_OUT
