"""ctypes binding of libb200mppi.so (include/b200mppi.h) and the thin device-array handle the
Python API hands out in place of Numba's DeviceNDArray.

There is no CPU fallback: if the shared library is missing, importing this module raises; if no
CUDA device is present, creating a planner/TDM raises B200MPPIError (the library itself still loads
on a GPU-less host so that the ABI can be checked there).
"""
import ctypes as C
import os

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libb200mppi.so")

MODE_TDM, MODE_DET_DYN, MODE_SPEED_MAP, MODE_BAREBONE = 0, 1, 2, 3

BUF_NOISE, BUF_U_CUR, BUF_COSTS, BUF_WEIGHTS, BUF_COSTS_NM, BUF_RNG, BUF_PARTIAL, BUF_U_PREV, \
    BUF_STATE_ROLLOUT = range(9)

T_NAMES = ("sample_grids", "noise", "rollout", "cvar", "update", "total")


class B200MPPIError(RuntimeError):
    pass


class ConfigPOD(C.Structure):
    _fields_ = [("num_steps", C.c_int32), ("num_control_rollouts", C.c_int32),
                ("num_grid_samples", C.c_int32), ("max_map_rows", C.c_int32),
                ("max_map_cols", C.c_int32), ("tdm_thread_x", C.c_int32), ("tdm_thread_y", C.c_int32),
                ("num_vis_state_rollouts", C.c_int32), ("mode", C.c_int32), ("device", C.c_int32),
                ("rank", C.c_int32), ("world_size", C.c_int32), ("seed", C.c_uint64)]


class ParamsPOD(C.Structure):
    _fields_ = [("dt", C.c_float), ("x0", C.c_float * 3), ("xgoal", C.c_float * 2),
                ("goal_tolerance", C.c_float), ("v_post_rollout", C.c_float), ("cvar_alpha", C.c_float),
                ("lambda_weight", C.c_float), ("u_std", C.c_float * 2), ("vrange", C.c_float * 2),
                ("wrange", C.c_float * 2), ("obs_penalty", C.c_float), ("unknown_penalty", C.c_float),
                ("dist_weight", C.c_float), ("num_opt", C.c_int32), ("alpha_dyn", C.c_double)]


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "mppi_numba_b200: %s is missing. Build it with `python mppi_numba_b200/build.py` "
            "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    P, I32, I64, F, D, SZ = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_double, C.c_size_t
    sigs = {
        "b200mppi_last_error": (C.c_char_p, []),
        "b200mppi_version": (C.c_int, []),
        "b200mppi_device_count": (C.c_int, []),
        "b200mppi_tdm_create": (C.c_int, [C.POINTER(ConfigPOD), C.POINTER(P)]),
        "b200mppi_tdm_destroy": (C.c_int, [P]),
        "b200mppi_tdm_set_stream": (C.c_int, [P, P]),
        "b200mppi_tdm_set_pmf": (C.c_int, [P, P, I32, I32, I32, P, P, F, P, P]),
        "b200mppi_tdm_set_pmf_collapsed": (C.c_int, [P, P, I32, I32, I32, I32, I32, I32, P, P, F, P, P, D, P, P, C.POINTER(I32)]),
        "b200mppi_tdm_set_bin_quantisation": (C.c_int, [P, P, I32]),
        "b200mppi_tdm_sample_grid_view": (C.c_int, [P, C.POINTER(P), C.POINTER(I32)]),
        "b200mppi_tdm_set_masks": (C.c_int, [P, P, P, I32, I32]),
        "b200mppi_tdm_set_risk_map": (C.c_int, [P, P, I32, I32]),
        "b200mppi_tdm_sample_grids": (C.c_int, [P, D]),
        "b200mppi_tdm_get_sample_grids": (C.c_int, [P, P, SZ]),
        "b200mppi_tdm_set_sample_grids": (C.c_int, [P, P, SZ]),
        "b200mppi_tdm_num_generators": (C.c_int, [P, C.POINTER(I64)]),
        "b200mppi_tdm_get_rng_states": (C.c_int, [P, P, SZ]),
        "b200mppi_tdm_set_rng_states": (C.c_int, [P, P, SZ]),
        "b200mppi_planner_create": (C.c_int, [C.POINTER(ConfigPOD), C.POINTER(P)]),
        "b200mppi_planner_destroy": (C.c_int, [P]),
        "b200mppi_planner_set_stream": (C.c_int, [P, P]),
        "b200mppi_planner_set_tdms": (C.c_int, [P, P, P]),
        "b200mppi_planner_set_obstacles": (C.c_int, [P, P, P, I32]),
        "b200mppi_planner_set_params": (C.c_int, [P, C.POINTER(ParamsPOD)]),
        "b200mppi_planner_set_u": (C.c_int, [P, P]),
        "b200mppi_planner_get_u": (C.c_int, [P, P]),
        "b200mppi_planner_shift_u": (C.c_int, [P, I32]),
        "b200mppi_planner_solve": (C.c_int, [P, P]),
        "b200mppi_planner_solve_local": (C.c_int, [P, I32]),
        "b200mppi_planner_solve_reduce": (C.c_int, [P, P]),
        "b200mppi_planner_solve_finish": (C.c_int, [P, P, P]),
        "b200mppi_debug_sample_threshold": (C.c_int, [C.c_double, C.c_int32, P, C.c_int64, P]),
        "b200mppi_planner_p2p_export": (C.c_int, [P, P, C.c_size_t]),
        "b200mppi_planner_p2p_import": (C.c_int, [P, P, C.c_size_t]),
        "b200mppi_planner_p2p_connect_local": (C.c_int, [P, P, C.c_int32]),
        "b200mppi_planner_p2p_push": (C.c_int, [P]),
        "b200mppi_planner_p2p_reduce": (C.c_int, [P]),
        "b200mppi_planner_p2p_finish": (C.c_int, [P, P]),
        "b200mppi_planner_solve_p2p": (C.c_int, [P, P]),
        "b200mppi_combine_partials_host": (C.c_int, [P, I32, I32, F, P, P, P, P]),
        "b200mppi_planner_sample_noise": (C.c_int, [P]),
        "b200mppi_planner_set_noise": (C.c_int, [P, P, SZ]),
        "b200mppi_planner_rollout": (C.c_int, [P]),
        "b200mppi_planner_cvar": (C.c_int, [P]),
        "b200mppi_planner_update": (C.c_int, [P, P]),
        "b200mppi_planner_get_state_rollout": (C.c_int, [P, P, SZ]),
        "b200mppi_planner_buffer": (C.c_int, [P, I32, C.POINTER(P), C.POINTER(SZ)]),
        "b200mppi_planner_copy_out": (C.c_int, [P, I32, P, SZ]),
        "b200mppi_planner_copy_in": (C.c_int, [P, I32, P, SZ]),
        "b200mppi_planner_synchronize": (C.c_int, [P]),
        "b200mppi_planner_set_profiling": (C.c_int, [P, I32]),
        "b200mppi_planner_last_timings": (C.c_int, [P, P]),
        "b200mppi_planner_launch_count": (C.c_int, [P, C.POINTER(I64)]),
        "b200mppi_planner_sample_box": (C.c_int, [P, C.POINTER(I32 * 5)]),
        "b200mppi_debug_rollout_cta_times": (C.c_int, [I32, P, I32]),
        "b200mppi_batch_create": (C.c_int, [C.POINTER(P), I32, C.POINTER(P)]),
        "b200mppi_batch_destroy": (C.c_int, [P]),
        "b200mppi_batch_set_stream": (C.c_int, [P, P]),
        "b200mppi_batch_solve": (C.c_int, [P, P]),
        "b200mppi_batch_launch_count": (C.c_int, [P, C.POINTER(I64)]),
    }
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name)          # AttributeError here == ABI drift, fail loudly
        fn.restype = res
        fn.argtypes = args
    return lib, tuple(sigs)


lib, EXPORTS = _load()


def check(rc):
    if rc != 0:
        raise B200MPPIError("b200mppi error %d: %s" % (rc, lib.b200mppi_last_error().decode()))


def device_count():
    return int(lib.b200mppi_device_count())


def ptr(a):
    """void* of a C-contiguous numpy array (kept alive by the caller)."""
    return a.ctypes.data_as(C.c_void_p)


def c_floats(values, n):
    arr = (C.c_float * n)()
    for i in range(n):
        arr[i] = float(values[i])
    return arr


class DeviceArray(object):
    """Stand-in for numba's DeviceNDArray: ``.shape``, ``.dtype``, ``.copy_to_host()``,
    ``.copy_to_device(host_array)`` and ``__cuda_array_interface__`` (zero-copy views for torch /
    numba / cupy).  The memory belongs to the planner / TDM handle that created it."""

    def __init__(self, owner, shape, dtype, reader, writer=None, dev_ptr=None, strides=None):
        self._owner = owner           # keeps the handle alive
        self.shape = tuple(int(s) for s in shape)
        self.dtype = np.dtype(dtype)
        self._reader, self._writer = reader, writer
        self._dev_ptr, self._strides = dev_ptr, strides

    @property
    def size(self):
        return int(np.prod(self.shape))

    @property
    def nbytes(self):
        return self.size * self.dtype.itemsize

    def __len__(self):
        return self.shape[0]

    def copy_to_host(self, ary=None):
        out = np.empty(self.shape, dtype=self.dtype) if ary is None else ary
        assert out.flags["C_CONTIGUOUS"] and out.nbytes == self.nbytes
        self._reader(out)
        return out

    def copy_to_device(self, ary):
        if self._writer is None:
            raise B200MPPIError("this device array is read-only from the host")
        src = np.ascontiguousarray(ary, dtype=self.dtype)
        assert src.size == self.size, "copy_to_device: size mismatch"
        self._writer(src)

    @property
    def __cuda_array_interface__(self):
        if self._dev_ptr is None:
            raise AttributeError("no raw device view for this array")
        return {"shape": self.shape, "typestr": self.dtype.str, "data": (int(self._dev_ptr()), False),
                "version": 3, "strides": self._strides}
