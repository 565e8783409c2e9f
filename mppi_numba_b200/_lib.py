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


class TrialDesc(C.Structure):
    """b200mppi_trial_desc: one planner's closed-loop trial (ground-truth grid, start, goal, padded limits)."""
    _fields_ = [("lin", C.c_void_p), ("ang", C.c_void_p), ("height", C.c_int32), ("width", C.c_int32),
                ("xlo", C.c_double), ("ylo", C.c_double), ("res", C.c_double), ("x0", C.c_double * 3),
                ("xgoal", C.c_double * 2), ("goal_tolerance", C.c_double), ("v_post_rollout", C.c_double),
                ("dt", C.c_double), ("pxlim", C.c_double * 2), ("pylim", C.c_double * 2)]


class TrialResult(C.Structure):
    """b200mppi_trial_result"""
    _fields_ = [("cum_obj", C.c_double), ("cum_dist_to_goal", C.c_double), ("dist_to_goal", C.c_double),
                ("steps", C.c_int32), ("status", C.c_int32)]


TRIAL_GOAL, TRIAL_MAX_STEPS, TRIAL_LEFT_MAP, TRIAL_NOT_RUN = 1, 2, 3, 4
TRIALS_MAP, TRIALS_STOCHASTIC, TRIALS_BAREBONE, TRIALS_MIXED = 0, 1, 2, 3


class LoopSummary(C.Structure):
    """b200mppi_loop_summary"""
    _fields_ = [("solves", C.c_int32), ("shifts", C.c_int32), ("status", C.c_int32), ("pad_", C.c_int32),
                ("x", C.c_double * 3)]


class LoopTask(C.Structure):
    """b200mppi_loop_task"""
    _fields_ = [("took_goal", C.c_int32), ("took_obstacles", C.c_int32), ("num_obstacles", C.c_int32),
                ("pad_", C.c_int32), ("goal", C.c_double * 2)]


POSE_F64, POSE_F32 = 0, 1
LOOP_RUNNING, LOOP_STOPPED, LOOP_BAD_OBSTACLES = 0, 5, 6
EINVAL = -1


def refuse_in_loop(obj, name):
    """ValueError when ``obj`` (a planner or TDM) belongs to the batch of an open device loop, naming the planner."""
    held = getattr(obj, "_device_loop", None)
    if held is not None:
        raise ValueError("%s: planner %d is in an open device loop (its batch's DeviceLoop owns its state until it "
                         "closes)" % (name, held))


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
        "b200mppi_tdm_draw_realisations": (C.c_int, [P, P, I32, C.POINTER(P)]),
        "b200mppi_realisations_destroy": (C.c_int, [P]),
        "b200mppi_realisations_info": (C.c_int, [P, C.POINTER(I32), C.POINTER(I32), C.POINTER(I32), C.POINTER(D),
                                                 C.POINTER(D), C.POINTER(D), C.POINTER(I32)]),
        "b200mppi_realisations_planes": (C.c_int, [P, I32, C.POINTER(P), C.POINTER(P)]),
        "b200mppi_realisations_copy_out": (C.c_int, [P, I32, P, P]),
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
        "b200mppi_debug_device_math": (C.c_int, [C.c_int32, P, P, P, C.c_int64]),
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
        "b200mppi_planner_sample_window": (C.c_int, [P, C.POINTER(I32 * 6)]),
        "b200mppi_debug_rollout_cta_times": (C.c_int, [I32, P, I32]),
        "b200mppi_batch_create": (C.c_int, [C.POINTER(P), I32, C.POINTER(P)]),
        "b200mppi_batch_create_stochastic": (C.c_int, [C.POINTER(P), I32, C.POINTER(P)]),
        "b200mppi_batch_create_mixed": (C.c_int, [C.POINTER(P), I32, C.POINTER(P)]),
        "b200mppi_batch_destroy": (C.c_int, [P]),
        "b200mppi_batch_set_stream": (C.c_int, [P, P]),
        "b200mppi_batch_solve": (C.c_int, [P, P]),
        "b200mppi_batch_launch_count": (C.c_int, [P, C.POINTER(I64)]),
        "b200mppi_batch_share_tdms": (C.c_int, [P, I32]),
        "b200mppi_batch_run_stochastic_trials": (C.c_int, [P, C.POINTER(TrialDesc), I32, P, P, C.POINTER(TrialResult),
                                                           C.POINTER(I32)]),
        "b200mppi_batch_run_trials": (C.c_int, [P, C.POINTER(TrialDesc), I32, P, P, C.POINTER(TrialResult),
                                                C.POINTER(I32)]),
        "b200mppi_batch_run_mixed_trials": (C.c_int, [P, C.POINTER(TrialDesc), I32, P, P, C.POINTER(TrialResult),
                                                      C.POINTER(I32)]),
        "b200mppi_batch_run_barebone_trials": (C.c_int, [P, C.POINTER(TrialDesc), I32, P, P, C.POINTER(TrialResult), P,
                                                         C.POINTER(I32)]),
        "b200mppi_batch_get_state_rollout": (C.c_int, [P, P, SZ]),
        "b200mppi_batch_run_trials_recorded": (C.c_int, [P, I32, C.POINTER(TrialDesc), I32, P, P,
                                                         C.POINTER(TrialResult), P, I32, P, SZ, C.POINTER(I32)]),
        "b200mppi_batch_run_trial_sequences": (C.c_int, [P, I32, C.POINTER(TrialDesc), P, I32, I32, P, P,
                                                         C.POINTER(TrialResult), C.POINTER(I32)]),
        "b200mppi_batch_run_trial_sequences_ex": (C.c_int, [P, I32, C.POINTER(TrialDesc), P, I32, I32, P, P,
                                                            C.POINTER(TrialResult), P, I32, P, SZ, C.POINTER(I32)]),
        "b200mppi_batch_loop_open": (C.c_int, [P, I32, P, P, C.POINTER(P)]),
        "b200mppi_loop_controls": (C.c_int, [P, C.POINTER(P), C.POINTER(P)]),
        "b200mppi_loop_solve": (C.c_int, [P, P]),
        "b200mppi_loop_shift_and_update": (C.c_int, [P, P, I32, I64]),
        "b200mppi_loop_stop": (C.c_int, [P, P, I32]),
        "b200mppi_loop_wait_stream": (C.c_int, [P, P]),
        "b200mppi_loop_active": (C.c_int, [P, C.POINTER(P)]),
        "b200mppi_loop_close": (C.c_int, [P, C.POINTER(LoopSummary)]),
        "b200mppi_batch_loop_open_ex": (C.c_int, [P, I32, P, P, I32, C.POINTER(P)]),
        "b200mppi_loop_obstacle_capacity": (C.c_int, [P, C.POINTER(I32)]),
        "b200mppi_loop_set_goals": (C.c_int, [P, P, I32, I64]),
        "b200mppi_loop_set_obstacles": (C.c_int, [P, P, I32, I32, I64, P]),
        "b200mppi_loop_close_ex": (C.c_int, [P, C.POINTER(LoopSummary), C.POINTER(LoopTask), P]),
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
    numba / cupy).  The memory belongs to the planner / TDM handle that created it.  ``stream`` (a cudaStream_t as
    int): the interface names it, so a consumer orders its work after the stream's (a device loop's controls)."""

    def __init__(self, owner, shape, dtype, reader, writer=None, dev_ptr=None, strides=None, stream=None):
        self._owner = owner           # keeps the handle alive
        self.shape = tuple(int(s) for s in shape)
        self.dtype = np.dtype(dtype)
        self._reader, self._writer = reader, writer
        self._dev_ptr, self._strides = dev_ptr, strides
        self._stream = stream

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
        cai = {"shape": self.shape, "typestr": self.dtype.str, "data": (int(self._dev_ptr()), False),
               "version": 3, "strides": self._strides}
        if self._stream is not None:
            cai["stream"] = int(self._stream) or 1      # the legacy default stream is 1 in the interface (0 is barred)
        return cai
