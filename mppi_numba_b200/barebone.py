"""Map-free "barebone" MPPI -- drop-in for the ``Config`` / ``MPPI_Numba`` pair defined inside the
reference's ``barebone_mppi_numba.ipynb`` (cells 2-3): nominal unicycle, quadratic distance cost,
circular obstacles, no traction maps.  Same engine, ``B200MPPI_MODE_BAREBONE``.

    from mppi_numba_b200.barebone import Config, MPPI_Numba
    planner = MPPI_Numba(Config(T=5.0, dt=0.1, num_control_rollouts=1000))
    planner.setup(mppi_params)          # dict as in the notebook (cell 5)
    useq = planner.solve()
"""
import copy
import ctypes as C
import time

import numpy as np

from . import _lib
from ._lib import DeviceArray, check, lib, ptr

DEFAULT_OBS_COST = 1e3           # notebook cell 3
DEFAULT_DIST_WEIGHT = 10

rec_max_control_rollouts = int(1e6)
rec_min_control_rollouts = 100


class Config:
    """Notebook cell 2: horizon, step, number of control sequences (clamped to [100, 1e6]), vis count, seed."""

    def __init__(self, T=10, dt=0.1, num_control_rollouts=1024, num_vis_state_rollouts=20, seed=1):
        assert T > 0 and dt > 0 and T > dt
        self.seed, self.T, self.dt = seed, T, dt
        self.num_steps = int(T / dt)
        assert self.num_steps > 0
        self.max_threads_per_block = 1024
        n = num_control_rollouts
        if n > rec_max_control_rollouts or n < rec_min_control_rollouts:
            n = min(rec_max_control_rollouts, max(rec_min_control_rollouts, n))
            print("MPPI Config: num_control_rollouts clipped to {}.".format(n))
        self.num_control_rollouts = n
        self.num_vis_state_rollouts = max(1, min(num_vis_state_rollouts, n))


class MPPI_Numba(object):
    """Planner object of the notebook (setup(params) / solve() / shift_and_update() / get_state_rollout())."""

    def __init__(self, cfg, device=0):
        self.cfg = cfg
        self.T, self.dt, self.num_steps = cfg.T, cfg.dt, cfg.num_steps
        self.num_control_rollouts = cfg.num_control_rollouts
        self.num_vis_state_rollouts = cfg.num_vis_state_rollouts
        self.seed = cfg.seed
        self.max_threads_per_block = cfg.max_threads_per_block
        self.device = int(device)
        self._handle = None
        self.noise_samples_d = self.u_cur_d = self.u_prev_d = None
        self.costs_d = self.weights_d = self.rng_states_d = self.state_rollout_batch_d = None
        self.device_var_initialized = False
        self.reset()

    def __del__(self):
        h, self._handle = getattr(self, "_handle", None), None
        if h:
            try:
                lib.b200mppi_planner_destroy(h)
            except Exception:
                pass

    def reset(self):
        self.u_seq0 = np.zeros((self.num_steps, 2), dtype=np.float32)
        self.params = None
        self.params_set = False
        self.u_prev_d = None
        self.init_device_vars_before_solving()

    def _buffer(self, buf_id, shape, dtype):
        h = self._handle
        return DeviceArray(self, shape, dtype,
                           lambda out: check(lib.b200mppi_planner_copy_out(h, buf_id, ptr(out), out.nbytes)),
                           lambda src: check(lib.b200mppi_planner_copy_in(h, buf_id, ptr(src), src.nbytes)))

    def init_device_vars_before_solving(self):
        if self.device_var_initialized:
            return
        t0 = time.time()
        N, T, V = self.num_control_rollouts, self.num_steps, self.num_vis_state_rollouts
        pod = _lib.ConfigPOD(num_steps=T, num_control_rollouts=N, num_grid_samples=1, max_map_rows=1, max_map_cols=1,
                             tdm_thread_x=1, tdm_thread_y=1, num_vis_state_rollouts=V, mode=_lib.MODE_BAREBONE,
                             device=self.device, rank=0, world_size=1, seed=int(self.seed) & (2 ** 64 - 1))
        h = C.c_void_p()
        check(lib.b200mppi_planner_create(C.byref(pod), C.byref(h)))
        self._handle = h
        self.noise_samples_d = self._buffer(_lib.BUF_NOISE, (N, T, 2), np.float32)
        self.u_cur_d = self._buffer(_lib.BUF_U_CUR, (T, 2), np.float32)
        self._u_prev_buf = self._buffer(_lib.BUF_U_PREV, (T, 2), np.float32)
        self.u_prev_d = self._u_prev_buf
        self.costs_d = self._buffer(_lib.BUF_COSTS, (N,), np.float32)
        self.weights_d = self._buffer(_lib.BUF_WEIGHTS, (N,), np.float32)
        self.rng_states_d = self._buffer(_lib.BUF_RNG, (N * T, 2), np.uint64)
        self.state_rollout_batch_d = self._buffer(_lib.BUF_STATE_ROLLOUT, (V, T + 1, 3), np.float32)
        self.device_var_initialized = True
        print("MPPI planner has initialized GPU memory after {} s".format(time.time() - t0))

    def setup(self, params):
        _lib.refuse_in_loop(self, "MPPI_Numba.setup")
        self.set_params(params)

    def set_params(self, params):
        _lib.refuse_in_loop(self, "MPPI_Numba.set_params")
        self.params = copy.deepcopy(params)
        self.params_set = True

    def check_solve_conditions(self):
        if not self.params_set:
            print("MPPI parameters are not set. Cannot solve")
            return False
        if not self.device_var_initialized:
            print("Device variables not initialized. Cannot solve.")
            return False
        return True

    def move_mppi_task_vars_to_device(self):
        p, f = self.params, np.float32
        pod = _lib.ParamsPOD()
        pod.dt = f(p['dt'])
        pod.x0 = _lib.c_floats(np.asarray(p['x0']).astype(f), 3)
        pod.xgoal = _lib.c_floats(np.asarray(p['xgoal']).astype(f), 2)
        pod.goal_tolerance = f(p['goal_tolerance'])
        pod.v_post_rollout = f(0.0)
        pod.cvar_alpha = f(1.0)
        pod.lambda_weight = f(p['lambda_weight'])
        pod.u_std = _lib.c_floats(np.asarray(p['u_std']).astype(f), 2)
        pod.vrange = _lib.c_floats(np.asarray(p['vrange']).astype(f), 2)
        pod.wrange = _lib.c_floats(np.asarray(p['wrange']).astype(f), 2)
        pod.obs_penalty = f(p.get('obs_penalty', DEFAULT_OBS_COST))
        pod.unknown_penalty = f(0.0)
        pod.dist_weight = f(p.get('dist_weight', DEFAULT_DIST_WEIGHT))
        pod.num_opt = int(p['num_opt'])
        pod.alpha_dyn = 1.0
        check(lib.b200mppi_planner_set_params(self._handle, C.byref(pod)))
        if "obstacle_positions" in p and len(p["obstacle_positions"]):
            pos = np.ascontiguousarray(np.asarray(p["obstacle_positions"]).astype(f).reshape(-1, 2))
            rad = np.ascontiguousarray(np.asarray(p["obstacle_radius"]).astype(f).reshape(-1))
            assert len(pos) == len(rad)
            check(lib.b200mppi_planner_set_obstacles(self._handle, ptr(pos), ptr(rad), len(rad)))
        else:
            check(lib.b200mppi_planner_set_obstacles(self._handle, None, None, 0))
        return pod

    def solve(self):
        _lib.refuse_in_loop(self, "MPPI_Numba.solve")
        if not self.check_solve_conditions():
            print("MPPI solve condition not met. Cannot solve. Return")
            return None
        return self.solve_with_nominal_dynamics()

    def solve_with_nominal_dynamics(self):
        self.move_mppi_task_vars_to_device()
        u = np.empty((self.num_steps, 2), dtype=np.float32)
        check(lib.b200mppi_planner_solve(self._handle, ptr(u)))
        self.u_prev_d = self._u_prev_buf
        return u

    def shift_and_update(self, new_x0, u_cur, num_shifts=1):
        _lib.refuse_in_loop(self, "MPPI_Numba.shift_and_update")
        self.params["x0"] = new_x0.copy()
        self.shift_optimal_control_sequence(u_cur, num_shifts)

    def shift_optimal_control_sequence(self, u_cur, num_shifts=1):
        shifted = u_cur.copy()
        shifted[:-num_shifts] = shifted[num_shifts:]
        shifted = np.ascontiguousarray(shifted, dtype=np.float32)
        check(lib.b200mppi_planner_set_u(self._handle, ptr(shifted)))

    def get_state_rollout(self):
        _lib.refuse_in_loop(self, "MPPI_Numba.get_state_rollout")
        assert self.params_set, "MPPI parameters are not set"
        if not self.device_var_initialized:
            print("Device variables not initialized. Cannot run mppi.")
            return None
        self.move_mppi_task_vars_to_device()
        out = np.empty(self.state_rollout_batch_d.shape, dtype=np.float32)
        check(lib.b200mppi_planner_get_state_rollout(self._handle, ptr(out), out.nbytes))
        return out
