"""Arithmetic objects of the oracle (TEST INFRASTRUCTURE, see oracle/__init__.py).

``oracle/mppi_ref.py`` and ``oracle/xoroshiro.py`` evaluate every floating-point operation of a rollout through one of
these objects, so that the same restatement serves two purposes:

* ``NUMPY`` (the default): numpy expressions -- float32 sin / cos / sqrt / log and IEEE division standing in for the
  GPU's approximate operations, ``fma32`` as a float64 multiply-add rounded twice, ``fma64`` as a float64 product and a
  float64 sum.  Fast, within a few ulp of the kernels, and what the golden vectors of the reference are checked against.
* ``Exact(provider, ftz)``: each operation rounded exactly as the kernels round it -- ``fma32`` / ``fma64`` rounded
  once (C ``fmaf`` / ``fma``), float32 add / sub / mul / conversions rounded to nearest, and with ``ftz`` the ``.ftz``
  semantics of csrc/common.cuh (float32 inputs and results that are subnormal become zeros of the same sign, also in
  ``cvt.ftz.f64.f32`` and ``cvt.rn.ftz.f32.f64``).  The approximate operations come from a provider:

  - ``LibmProvider()``: glibc ``sinf`` / ``cosf`` / ``sqrtf`` / ``logf`` and IEEE division -- exactly what the host
    emulation of the kernels (tests/emu_*.py) substitutes for them;
  - ``DeviceProvider(lib)``: the device's own ``sin.approx`` / ``cos.approx`` / ``sqrt.approx`` / ``div.approx`` /
    ``div.full`` and libdevice ``logf`` / ``cosf``, evaluated by ``b200mppi_debug_device_math`` with the library's
    compile flags.  These are deterministic functions of their inputs, so with ``ftz=True`` the oracle predicts what
    the kernels compute on that GPU, bit for bit.

The host helper (``fmaf`` / ``fma`` / glibc math over arrays) is compiled with g++ on first use into a per-user
temporary directory: no fast-math, no FMA contraction, no assumption about the host's FMA instructions.
"""
import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

F32 = np.float32
F64 = np.float64
_TINY32 = F32(2.0 ** -126)

_HELPER_SRC = r'''
#include <cmath>
extern "C" {
void h_fmaf(const float* a, const float* b, const float* c, float* o, long n) { for (long i = 0; i < n; ++i) o[i] = std::fma(a[i], b[i], c[i]); }
void h_fma(const double* a, const double* b, const double* c, double* o, long n) { for (long i = 0; i < n; ++i) o[i] = std::fma(a[i], b[i], c[i]); }
void h_sinf(const float* a, float* o, long n) { for (long i = 0; i < n; ++i) o[i] = sinf(a[i]); }
void h_cosf(const float* a, float* o, long n) { for (long i = 0; i < n; ++i) o[i] = cosf(a[i]); }
void h_sqrtf(const float* a, float* o, long n) { for (long i = 0; i < n; ++i) o[i] = sqrtf(a[i]); }
void h_logf(const float* a, float* o, long n) { for (long i = 0; i < n; ++i) o[i] = logf(a[i]); }
}
'''
_helper = None


def helper():
    """The compiled host helper (ctypes CDLL), built once per process into a per-user temporary directory."""
    global _helper
    if _helper is not None:
        return _helper
    tag = hashlib.sha256(_HELPER_SRC.encode()).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), "b200mppi_oracle_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, "libarith_%s.so" % tag)
    if not os.path.exists(so):
        work = tempfile.mkdtemp(dir=d)
        try:
            cpp = os.path.join(work, "arith.cpp")
            with open(cpp, "w") as fh:
                fh.write(_HELPER_SRC)
            tmp_so = os.path.join(work, "libarith.so")
            r = subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-fno-fast-math", "-ffp-contract=off", cpp, "-o",
                                tmp_so], capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError("g++ failed on the oracle's arithmetic helper:\n" + r.stderr[-3000:])
            os.replace(tmp_so, so)
        finally:
            shutil.rmtree(work, ignore_errors=True)
    lib = C.CDLL(so)
    P, L = C.c_void_p, C.c_long
    for name in ("h_fmaf", "h_fma"):
        getattr(lib, name).argtypes = [P, P, P, P, L]
        getattr(lib, name).restype = None
    for name in ("h_sinf", "h_cosf", "h_sqrtf", "h_logf"):
        getattr(lib, name).argtypes = [P, P, L]
        getattr(lib, name).restype = None
    _helper = lib
    return lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _call(fn, dtype, *args):
    """fn over same-shape contiguous copies of the broadcast arguments; returns an array of that shape."""
    arrs = np.broadcast_arrays(*[np.asarray(a, dtype=dtype) for a in args])
    shape = arrs[0].shape
    flat = [np.ascontiguousarray(a, dtype=dtype).reshape(-1) for a in arrs]
    out = np.empty(flat[0].size, dtype=dtype)
    fn(*[_ptr(a) for a in flat], _ptr(out), out.size)
    return out.reshape(shape)


def fma32_once(a, b, c):
    """float32 a*b + c rounded once (C fmaf)."""
    return _call(helper().h_fmaf, F32, a, b, c)


def fma64_once(a, b, c):
    """float64 a*b + c rounded once (C fma)."""
    return _call(helper().h_fma, F64, a, b, c)


def _as(x, dtype):
    """Array -> array of dtype, scalar -> numpy scalar of dtype."""
    return x.astype(dtype) if isinstance(x, np.ndarray) else dtype(x)


def flush32(x):
    """Subnormal float32 values -> zero of the same sign (the .ftz input / output rule)."""
    x = np.asarray(x, dtype=F32)
    return np.where((np.abs(x) < _TINY32) & (x != 0), np.copysign(F32(0), x), x).astype(F32)


# ----------------------------------------------------------------------------- approximate-operation providers
class LibmProvider:
    """glibc sinf / cosf / sqrtf / logf and IEEE float32 division: what tests/emu_*.py substitute for the MUFU
    operations, the approximate divisions and libdevice's logf / cosf."""
    name = "libm"

    def sin(self, x):
        return _call(helper().h_sinf, F32, x)

    def cos(self, x):
        return _call(helper().h_cosf, F32, x)

    def sqrt(self, x):
        return _call(helper().h_sqrtf, F32, x)

    def div_approx(self, a, b):
        return np.divide(np.asarray(a, F32), np.asarray(b, F32), dtype=F32)

    div_full = div_approx

    def logf(self, x):
        return _call(helper().h_logf, F32, x)

    cosf = cos


class DeviceProvider:
    """The GPU's approximate operations, evaluated on the device (b200mppi_debug_device_math).  ``lib`` is the
    package's ctypes module (mppi_numba_b200._lib)."""
    name = "device"
    OPS = dict(sin=0, cos=1, sqrt=2, div_approx=3, div_full=4, logf=5, cosf=6)

    def __init__(self, lib):
        self.L = lib

    def _run(self, op, a, b=None):
        args = [a] if b is None else [a, b]
        arrs = np.broadcast_arrays(*[np.asarray(v, dtype=F32) for v in args])
        shape = arrs[0].shape
        flat = [np.ascontiguousarray(v).reshape(-1) for v in arrs]
        out = np.empty(flat[0].size, dtype=F32)
        self.L.check(self.L.lib.b200mppi_debug_device_math(self.OPS[op], _ptr(flat[0]),
                                                           _ptr(flat[1]) if b is not None else None, _ptr(out),
                                                           out.size))
        return out.reshape(shape)

    def sin(self, x):
        return self._run("sin", x)

    def cos(self, x):
        return self._run("cos", x)

    def sqrt(self, x):
        return self._run("sqrt", x)

    def div_approx(self, a, b):
        return self._run("div_approx", a, b)

    def div_full(self, a, b):
        return self._run("div_full", a, b)

    def logf(self, x):
        return self._run("logf", x)

    def cosf(self, x):
        return self._run("cosf", x)


# ----------------------------------------------------------------------------- arithmetic objects
class NumpyArith:
    """The oracle's default arithmetic: numpy expressions (see the module docstring).  Its results are those of the
    oracle before arithmetic objects existed, byte for byte."""
    exact = False
    ftz = False

    def add32(self, a, b):
        return _as(a + b, F32)

    def sub32(self, a, b):
        return _as(a - b, F32)

    def mul32(self, a, b):
        return _as(a * b, F32)

    def fma32(self, a, b, c):
        return (np.asarray(a).astype(F64) * np.asarray(b).astype(F64) + np.asarray(c).astype(F64)).astype(F32)

    def fma64(self, a, b, c):
        return a * b + c

    def f2d(self, a):
        return _as(a, F64)

    def d2f(self, a):
        return _as(a, F32)

    def floor32(self, a):
        return np.floor(a)

    def sin32(self, x):
        return np.sin(x).astype(F32)

    def cos32(self, x):
        return np.cos(x).astype(F32)

    def sqrt32(self, x):
        return np.sqrt(x).astype(F32)

    def div_approx32(self, a, b):
        return _as(a / b, F32)

    div_full32 = div_approx32
    div_rn32 = div_approx32

    def logf32(self, x):
        return np.log(x)

    def cosf32(self, x):
        return np.cos(x)


class Exact:
    """Every operation rounded as the kernels round it; the approximate ones from ``provider``; ``ftz``: the .ftz
    behaviour of csrc/common.cuh's helpers (float32 subnormal inputs and results flushed to signed zero)."""
    exact = True

    def __init__(self, provider, ftz=False):
        self.p = provider
        self.ftz = bool(ftz)

    def _in(self, x):
        x = np.asarray(x, dtype=F32)
        return flush32(x) if self.ftz else x

    _out = _in

    def add32(self, a, b):
        return self._out(np.add(self._in(a), self._in(b), dtype=F32))

    def sub32(self, a, b):
        return self._out(np.subtract(self._in(a), self._in(b), dtype=F32))

    def mul32(self, a, b):
        return self._out(np.multiply(self._in(a), self._in(b), dtype=F32))

    def fma32(self, a, b, c):
        return self._out(fma32_once(self._in(a), self._in(b), self._in(c)))

    def fma64(self, a, b, c):
        return fma64_once(a, b, c)

    def f2d(self, a):                                   # cvt(.ftz).f64.f32
        return self._in(a).astype(F64)

    def d2f(self, a):                                   # cvt.rn(.ftz).f32.f64
        return self._out(np.asarray(a, dtype=F64).astype(F32))

    def floor32(self, a):                               # cvt.rmi(.ftz).f32.f32
        return self._out(np.floor(self._in(a)))

    def sin32(self, x):
        return self._out(self.p.sin(self._in(x)))

    def cos32(self, x):
        return self._out(self.p.cos(self._in(x)))

    def sqrt32(self, x):
        return self._out(self.p.sqrt(self._in(x)))

    def div_approx32(self, a, b):
        return self._out(self.p.div_approx(self._in(a), self._in(b)))

    def div_full32(self, a, b):
        return self._out(self.p.div_full(self._in(a), self._in(b)))

    def div_rn32(self, a, b):
        return self._out(np.divide(self._in(a), self._in(b), dtype=F32))

    # libdevice logf / cosf of the Box-Muller noise: the provider's own results (the library is built with -ftz=true,
    # which selects libdevice's flushing variants; the provider evaluates them under the same flag)
    def logf32(self, x):
        return self.p.logf(np.asarray(x, dtype=F32))

    def cosf32(self, x):
        return self.p.cosf(np.asarray(x, dtype=F32))


NUMPY = NumpyArith()
