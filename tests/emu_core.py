"""The kernel emulators' toolkit (TEST INFRASTRUCTURE): lift kernel text out of csrc/, rewrite what the host compiler
cannot take, compile it against tests/emu_cuda.h with g++ and bind its entry points.

Each emulator (tests/emu_*.py) is the text between ``// [emu:begin NAME]`` / ``// [emu:end NAME]`` markers of the CUDA
sources, pasted inside namespace b200 after the header, plus an ``extern "C"`` harness that sets up the arguments as
the host code does and runs the kernels with ``emu::launch`` / ``emu::launch_serial``.  The ctypes signature of every
entry point comes from its C declaration in the harness, so a pointer can never be passed as a 32-bit int."""
import ctypes as C
import os
import re
import subprocess

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
CSRC = os.path.join(ROOT, "mppi_numba_b200", "csrc")
ENGINE_DIR = os.path.join(ROOT, "mppi_numba_b200")

FLAGS = ["-O1", "-std=c++20", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", TESTS]


def region(file, name):
    """The text between the ``[emu:begin name]`` and ``[emu:end name]`` markers of csrc/<file>."""
    path = os.path.join(CSRC, file)
    m = re.search(r"// \[emu:begin %s\][^\n]*\n(.*?)// \[emu:end %s\]" % (name, name), open(path).read(), re.S)
    assert m, "marker %s not found in %s" % (name, path)
    return m.group(1)


def _subn(pattern, repl, src, count, what):
    out, n = re.subn(pattern, repl, src)
    assert n == count, "%s: %d replacements, expected %d" % (what, n, count)
    return out


def shared_static(src, count):
    """Function-scope ``__shared__`` declarations -> ``static``: one instance for the threads of the running block."""
    return _subn(r"(?m)^(\s*)__shared__ ", r"\1static ", src, count, "__shared__ -> static")


def extern_shared(src, count):
    """``extern __shared__ [__align__(n)] T x[];`` -> ``T* const x``, a view of the header's shared-memory buffer."""
    return _subn(r"extern __shared__ (?:__align__\(\d+\) )?(\w[\w ]*?) (\w+)\[\];",
                 r"\1* const \2 = reinterpret_cast<\1*>(emu::smem);", src, count, "extern __shared__")


def cell_index_rzi(src):
    """The ``cvt.rzi`` of cell_index_exact -> a C cast (truncation toward zero)."""
    return _subn(r'int k; asm\("cvt\.rzi\.ftz\.s32\.f32[^;]*;[^;]*;', "int k = (int)res;   /* cvt.rzi */", src, 1,
                 "cvt.rzi of cell_index_exact")


def drop_fences(src, count):
    """The mbarrier-init, async-proxy and tensor-map fences of the windowed kernel -> empty statements: the stand-ins
    finish every copy before they return."""
    return _subn(r'asm volatile ?\("fence\.[^;]*;[^;]*;', ";", src, count, "fences")


_CTYPES = {"void": None, "int": C.c_int, "long long": C.c_longlong, "float": C.c_float, "double": C.c_double,
           "uint32_t": C.c_uint32, "size_t": C.c_size_t}


def _ctype(decl, where):
    t = " ".join(decl.replace("const", " ").split())
    if "*" in t:
        return C.c_void_p
    assert t in _CTYPES, "%s: C type '%s' has no ctypes binding in tests/emu_core.py" % (where, t)
    return _CTYPES[t]


def bind(lib, harness):
    """restype / argtypes of every ``extern "C"`` function declared in the harness text, from its declaration."""
    for ret, name, params in re.findall(r'extern "C"\s+([^(]*?)\s*\b(\w+)\s*\(([^)]*)\)', harness):
        fn = getattr(lib, name)
        fn.restype = _ctype(ret, name)
        args = [p.strip() for p in params.split(",") if p.strip() not in ("", "void")]
        fn.argtypes = [_ctype(re.sub(r"\w+$", "", p), "%s(%s)" % (name, p)) for p in args]
    return lib


def build(out_dir, stem, parts, harness, link_engine=False):
    """Compile emu_cuda.h + the kernel text ``parts`` (inside namespace b200) + ``harness`` into
    out_dir/lib<stem>.so and bind its entry points.  ``link_engine``: link libb200mppi.so for the host-side table
    builders the harness calls."""
    src = '#include "emu_cuda.h"\nnamespace b200 {\n' + "".join(parts) + "}  // namespace b200\n" + harness
    cpp, so = os.path.join(out_dir, stem + ".cpp"), os.path.join(out_dir, "lib%s.so" % stem)
    with open(cpp, "w") as f:
        f.write(src)
    cmd = ["g++"] + FLAGS + [cpp, "-o", so]
    if link_engine:
        cmd += ["-L" + ENGINE_DIR, "-l:libb200mppi.so", "-Wl,-rpath," + ENGINE_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-6000:]
    return bind(C.CDLL(so), harness)
