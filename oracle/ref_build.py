"""Compile the reference package (mit-acl/mppi_numba) to bytecode under oracle/_ref/ -- TEST INFRASTRUCTURE.

The GPU-side parity test (tests/test_gpu_vs_reference.py) and bench.py's `numba_cuda_baseline` leg run the
UNMODIFIED reference's Numba-CUDA kernels next to the engine.  The reference cannot be part of this repository and
is not installed where the GPU runs, so build() compiles it here, where it is readable (ref_loader.REFERENCE_ROOT),
into git-ignored sourceless bytecode: oracle/_ref/mppi_numba/*.pyc, importable with oracle/_ref on sys.path (Numba
compiles kernels from bytecode).  The map-free variant lives in a notebook (barebone_mppi_numba.ipynb): its code cells
2-3 (Config, then the cost functions and MPPI_Numba with its kernels), behind the imports of its cell 1 without the
plotting ones, become the module oracle/_ref/barebone_mppi_numba.pyc; the generated source is written to a temporary
directory outside the repository and removed.  Without a readable reference nothing is built and the consumers report
it missing.
"""
import glob
import json
import os
import py_compile
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF_OUT = os.path.join(HERE, "_ref")

# the notebook's cell 1 without matplotlib (what oracle/make_golden.load_barebone_notebook executes as well)
NOTEBOOK_HEADER = ("import numpy as np\nimport math\nimport copy\nimport numba\nimport time\nfrom numba import cuda\n"
                   "from numba.cuda.random import create_xoroshiro128p_states, xoroshiro128p_normal_float32\n")


def compiled_reference():
    """The directory to put on sys.path to import the compiled reference, or None if it was not built."""
    return REF_OUT if os.path.isfile(os.path.join(REF_OUT, "mppi_numba", "mppi.pyc")) else None


def compiled_notebook():
    """The directory to put on sys.path to import the compiled notebook as ``barebone_mppi_numba``, or None."""
    return REF_OUT if os.path.isfile(os.path.join(REF_OUT, "barebone_mppi_numba.pyc")) else None


def _compile(path, out, dfile):
    py_compile.compile(path, cfile=out, dfile=dfile, doraise=True,
                       invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)


def notebook_source(nb_path):
    """The module source of the notebook's code cells 2-3 behind NOTEBOOK_HEADER."""
    with open(nb_path) as f:
        nb = json.load(f)
    code = [c for c in nb["cells"] if c["cell_type"] == "code"]
    return NOTEBOOK_HEADER + "\n" + "".join(code[1]["source"]) + "\n\n" + "".join(code[2]["source"]) + "\n"


def build_reference(out_dir=REF_OUT):
    from oracle.ref_loader import REFERENCE_ROOT
    src = os.path.join(REFERENCE_ROOT, "mppi_numba")
    if not os.access(os.path.join(src, "mppi.py"), os.R_OK):
        return None
    dst = os.path.join(out_dir, "mppi_numba")
    os.makedirs(dst, exist_ok=True)
    for path in sorted(glob.glob(os.path.join(src, "*.py"))):
        name = os.path.basename(path)
        out = os.path.join(dst, name[:-3] + ".pyc")
        if not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(path):
            _compile(path, out, os.path.join("mppi_numba", name))
    nb = os.path.join(REFERENCE_ROOT, "barebone_mppi_numba.ipynb")
    out = os.path.join(out_dir, "barebone_mppi_numba.pyc")
    if os.access(nb, os.R_OK) and (not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(nb)):
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "barebone_mppi_numba.py")
            with open(path, "w") as f:
                f.write(notebook_source(nb))
            _compile(path, out, "barebone_mppi_numba.py")
    return out_dir
