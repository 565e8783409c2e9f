"""``MPPI_Numba`` -- the planner object, kept API-compatible with the reference class of the same
name (mppi_numba/mppi.py:39-608) but backed by libb200mppi.so (hand-written sm_90a CUDA behind the
C-ABI of include/b200mppi.h) instead of Numba-JIT kernels.

What a reference user keeps: ``MPPI_Numba(cfg)``, ``reset()``, ``setup(params, lin_tdm, ang_tdm)``,
``solve()`` -> ``np.float32[T, 2]`` (or ``None`` with a printed reason when preconditions fail),
``shift_and_update(x0, u, num_shifts)``, ``get_state_rollout()``, and the device attributes
``noise_samples_d, u_cur_d, u_prev_d, costs_d, weights_d, rng_states_d, state_rollout_batch_d``
(objects with ``.shape`` / ``.copy_to_host()``).

What is new: the work can be sharded over ranks (one process per GPU, ``torch.distributed``).
``use_tdm``: the M sampled MAPS are sharded -- each rank samples its M/G maps (bit-identical to the same
maps of a 1-rank run), rolls out all N control sequences on them, an all-to-all hands every rank the
per-(n,m) costs of its N/G slice for the CVaR, and one all-gather of 2T+2 floats (softmax baseline,
weight sum, weighted-noise sums) joins the update.  One-map modes shard N and need only the all-gather.  ``costs_d`` is NOT clobbered by the update (the reference reuses it as
scratch, SURVEY.md 9-Q1).
"""
import copy
import ctypes as C
import time

import numpy as np

from . import _lib
from ._lib import DeviceArray, check, lib, ptr

DEFAULT_UNKNOWN_COST = float(1e2)
DEFAULT_OBS_COST = float(1e5)
DEFAULT_DIST_WEIGHT = 1.0


class MPPI_Numba(object):
    """MPPI planner for a unicycle on a probabilistic traction map (GPU-resident state)."""

    def __init__(self, cfg, device=0, rank=0, world_size=1, process_group=None):
        self.cfg = cfg
        for name in ("T", "dt", "num_steps", "num_grid_samples", "num_control_rollouts",
                     "max_speed_padding", "tdm_sample_thread_dim", "num_vis_state_rollouts",
                     "max_map_dim", "seed", "use_tdm", "use_det_dynamics",
                     "use_nom_dynamics_with_speed_map", "use_costmap"):
            setattr(self, name, getattr(cfg, name))
        self.det_dyn = bool(self.use_det_dynamics or self.use_nom_dynamics_with_speed_map or self.use_costmap)
        self.max_threads_per_block = cfg.max_threads_per_block
        self.device, self.rank, self.world_size = int(device), int(rank), int(world_size)
        self.process_group = process_group
        self._handle = None
        self._pod = _lib.ParamsPOD()
        self._pod_f32 = np.frombuffer(self._pod, dtype=np.float32, count=19)     # dt .. dist_weight
        self._gathered = None            # torch tensor (world_size, 2T+2) for the exchange
        self._p2p = False                # peer-memory exchange connected (csrc/p2p.cu)
        self._partial_t = None
        self._stream = None

        self.noise_samples_d = self.u_cur_d = self.u_prev_d = None
        self.costs_d = self.weights_d = self.rng_states_d = self.state_rollout_batch_d = None
        self._u_prev_buf = None
        self.device_var_initialized = False
        self.reset()

    # ------------------------------------------------------------------ lifetime
    def __del__(self):
        h, self._handle = getattr(self, "_handle", None), None
        if h:
            try:
                lib.b200mppi_planner_destroy(h)
            except Exception:
                pass

    def reset(self):
        """Drop task state (params, TDM references).  Device buffers, the warm-start ``u_cur_d`` and
        the RNG streams persist, exactly like the reference (SURVEY.md 9-Q3)."""
        self.u_seq0 = np.zeros((self.num_steps, 2), dtype=np.float32)
        self.params = None
        self.params_set = False
        self.lin_tdm = self.ang_tdm = None
        self.tdm_set = False
        self.u_prev_d = None
        self.init_device_vars_before_solving()

    def _buffer(self, buf_id, shape, dtype, writable=True, raw_view=True):
        """raw_view=False: no ``__cuda_array_interface__`` (the device layout differs from ``shape``: the per-(n,m)
        costs are stored map-major, copy_to_host() returns the logical (n, m) array)."""
        h = self._handle

        def dev_ptr():
            p, n = C.c_void_p(), C.c_size_t()
            check(lib.b200mppi_planner_buffer(h, buf_id, C.byref(p), C.byref(n)))
            return p.value
        return DeviceArray(
            self, shape, dtype,
            lambda out: check(lib.b200mppi_planner_copy_out(h, buf_id, ptr(out), out.nbytes)),
            (lambda src: check(lib.b200mppi_planner_copy_in(h, buf_id, ptr(src), src.nbytes))) if writable else None,
            dev_ptr=dev_ptr if raw_view else None)

    def init_device_vars_before_solving(self):
        if self.device_var_initialized:
            return
        t0 = time.time()
        rows, cols = self.max_map_dim
        pod = _lib.ConfigPOD(num_steps=self.num_steps, num_control_rollouts=self.num_control_rollouts,
                             num_grid_samples=self.num_grid_samples, max_map_rows=rows, max_map_cols=cols,
                             tdm_thread_x=self.tdm_sample_thread_dim[0], tdm_thread_y=self.tdm_sample_thread_dim[1],
                             num_vis_state_rollouts=self.num_vis_state_rollouts, mode=self.cfg.mode,
                             device=self.device, rank=self.rank, world_size=self.world_size,
                             seed=int(self.seed) & (2 ** 64 - 1))
        h = C.c_void_p()
        check(lib.b200mppi_planner_create(C.byref(pod), C.byref(h)))
        self._handle = h
        N = self.num_control_rollouts
        self.n_begin = N * self.rank // self.world_size
        n_slice = N * (self.rank + 1) // self.world_size - self.n_begin
        T, M = self.num_steps, (self.num_grid_samples if self.use_tdm else 1)
        # use_tdm with several ranks shards the MAPS: every rank simulates all N control sequences on its
        # M/ws maps and reduces (CVaR, softmax) its N/ws slice; the one-map modes shard N instead.
        self.shard_maps = bool(self.use_tdm and self.world_size > 1)
        self.n_local = N if self.shard_maps else n_slice          # rows of noise / per-(n,m) costs
        self.n_reduce = n_slice                                   # rows of costs_d / weights_d
        if self.shard_maps:
            M //= self.world_size
        self.m_local = M
        self.noise_samples_d = self._buffer(_lib.BUF_NOISE, (self.n_local, T, 2), np.float32)
        self.u_cur_d = self._buffer(_lib.BUF_U_CUR, (T, 2), np.float32)
        self._u_prev_buf = self._buffer(_lib.BUF_U_PREV, (T, 2), np.float32)
        self.u_prev_d = self._u_prev_buf
        self.costs_d = self._buffer(_lib.BUF_COSTS, (self.n_reduce,), np.float32)
        self.weights_d = self._buffer(_lib.BUF_WEIGHTS, (self.n_reduce,), np.float32)
        self.costs_nm_d = self._buffer(_lib.BUF_COSTS_NM, (self.n_local, M), np.float32, raw_view=False)
        self.rng_states_d = self._buffer(_lib.BUF_RNG, (self.n_local * T, 2), np.uint64)
        self.partial_d = self._buffer(_lib.BUF_PARTIAL, (2 * T + 2,), np.float32, writable=False)
        self.state_rollout_batch_d = self._buffer(_lib.BUF_STATE_ROLLOUT,
                                                  (self.num_vis_state_rollouts, T + 1, 3), np.float32)
        self.device_var_initialized = True
        print("MPPI planner has initialized GPU memory after {} s".format(time.time() - t0))

    # ------------------------------------------------------------------ task set-up
    def setup(self, params, lin_tdm, ang_tdm):
        self.set_tdm(lin_tdm, ang_tdm)
        self.set_params(params)

    def is_within_bound(self, v, vbounds):
        return v >= vbounds[0] and v <= vbounds[1]

    def set_params(self, params):
        for axis, limits, label in ((0, self.lin_tdm.xlimits, "xlimits"), (1, self.lin_tdm.ylimits, "ylimits")):
            if not self.is_within_bound(params['x0'][axis], limits):
                print("ERROR: When setting mppi params, x0[{}] is not within {}!".format(axis, label))
                assert False
        self.params = copy.deepcopy(params)
        self.params_set = True

    def set_tdm(self, lin_tdm, ang_tdm):
        self.lin_tdm, self.ang_tdm = lin_tdm, ang_tdm
        self.tdm_set = True

    def check_solve_conditions(self):
        reasons = (
            (self.params_set, "MPPI parameters are not set. Cannot solve"),
            (self.tdm_set, "MPPI has not received TDMs. Cannot solve"),
            (self.device_var_initialized, "Device variables not initialized. Cannot solve."),
            (self.tdm_set and self.lin_tdm.pmf_grid_initialized, "Linear TDM's PMF not initialized. Cannot solve."),
            (self.tdm_set and self.ang_tdm.pmf_grid_initialized, "Angular TDM's PMF not initialized. Cannot solve."),
        )
        for ok, why in reasons:
            if not ok:
                print(why)
                return False
        if not self.is_within_bound(self.params["x0"][0], self.lin_tdm.padded_xlimits):
            print("Robot initial condition not within padded xlimits.")
            return False
        if not self.is_within_bound(self.params["x0"][1], self.lin_tdm.padded_ylimits):
            print("Robot initial condition not within padded ylimits.")
            return False
        return True

    def move_mppi_task_vars_to_device(self):
        """Pack the params dict into the POD the kernels take BY VALUE (one struct in kernel-argument
        space replaces the reference's seven cuda.to_device allocations per solve, mppi.py:214-234).
        Casts to float32 exactly where the reference casts."""
        p = self.params
        pod, v = self._pod, self._pod_f32          # persistent POD + float32 view of its 19 leading floats
        v[0] = p['dt']
        v[1:4] = p['x0']
        v[4:6] = p['xgoal']
        v[6] = p['goal_tolerance']
        v[7] = p['v_post_rollout']
        v[8] = p['cvar_alpha']
        v[9] = p['lambda_weight']
        v[10:12] = p['u_std']
        v[12:14] = p['vrange']
        v[14:16] = p['wrange']
        v[16] = p.get('obs_penalty', DEFAULT_OBS_COST)
        v[17] = p.get('unknown_penalty', DEFAULT_UNKNOWN_COST)
        v[18] = p.get('dist_weight', DEFAULT_DIST_WEIGHT)
        pod.num_opt = int(p['num_opt'])
        pod.alpha_dyn = float(p.get('alpha_dyn', 1.0))
        check(lib.b200mppi_planner_set_tdms(self._handle, self.lin_tdm._handle, self.ang_tdm._handle))
        check(lib.b200mppi_planner_set_params(self._handle, C.byref(pod)))
        return pod

    # ------------------------------------------------------------------ solve
    def solve(self):
        """One MPPI solve: sample both TDMs, then num_opt x (noise, rollouts, CVaR, update).
        Returns the optimised control sequence (T, 2) float32, or None if a precondition fails."""
        if not self.check_solve_conditions():
            print("MPPI solve condition not met. Cannot solve. Return")
            return None
        if self.use_det_dynamics:
            return self.solve_det_dyn()
        if self.use_nom_dynamics_with_speed_map:
            return self.solve_nom_dyn_w_speed_map()
        if self.use_tdm:
            if self.cfg.num_grid_samples > self.cfg.max_threads_per_block:
                return self.solve_stochastic_oversized()
            return self.solve_stochastic()
        print("None of the planner options are selected.")
        assert False

    def _solve_on_device(self):
        self.move_mppi_task_vars_to_device()
        u = np.empty((self.num_steps, 2), dtype=np.float32)
        if self.world_size == 1:
            check(lib.b200mppi_planner_solve(self._handle, ptr(u)))
        else:
            self._solve_sharded(u)
        if self.det_dyn:
            self.u_prev_d = self._u_prev_buf       # the reference aliases u_prev_d to u_cur_d here
        return u

    def solve_det_dyn(self):
        return self._solve_on_device()

    def solve_nom_dyn_w_speed_map(self):
        return self._solve_on_device()

    def solve_stochastic(self):
        return self._solve_on_device()

    def solve_stochastic_oversized(self):
        """num_grid_samples > 1024 (mppi.py:454-531).  The reference's oversized kernel swaps unconditionally
        instead of sorting (SURVEY.md 9-B1), so its result is meaningful only for cvar_alpha = 1 (the mean);
        the engine has no block-size limit on M and evaluates the same statistic as solve_stochastic:
        the mean of the ceil(M * cvar_alpha) largest costs."""
        assert self.num_grid_samples > self.cfg.max_threads_per_block
        return self._solve_on_device()

    # ---- multi-GPU: N sharded over ranks, one all-gather of 2T+2 floats per iteration
    def _ensure_exchange(self):
        if self._gathered is not None:
            return
        import torch
        import torch.distributed as dist
        assert dist.is_initialized(), "world_size > 1 needs an initialised torch.distributed process group"
        dev = torch.device("cuda", self.device)
        self._stream = torch.cuda.Stream(device=dev)
        # only the planner works on the exchange stream: solve() samples the TDMs' maps on the PLANNER's stream;
        # the TDMs keep their own streams for uploads and public sample_grids() calls (and may outlive the planner)
        check(lib.b200mppi_planner_set_stream(self._handle, C.c_void_p(self._stream.cuda_stream)))
        self._p2p = self._connect_peers()
        if self._p2p:
            self._gathered = True          # exchange buffers live inside the library
            return
        self._partial_t = torch.as_tensor(self.partial_d, device=dev)          # zero-copy view
        self._gathered = torch.empty((self.world_size * (2 * self.num_steps + 2),), dtype=torch.float32, device=dev)
        if self.shard_maps:
            # the device buffer itself: (ws, M/ws, N/ws) blocks by destination rank (include/b200mppi.h), zero-copy
            raw = self._buffer(_lib.BUF_COSTS_NM, (self.n_local * self.m_local,), np.float32)
            self._costs_send = torch.as_tensor(raw, device=dev)
            self._costs_recv = torch.empty_like(self._costs_send)                         # (ws, N/ws, M/ws)

    def _connect_peers(self):
        """Peer-memory exchange (csrc/p2p.cu): every rank exports the CUDA IPC handle of its exchange buffer,
        one all-gather of the 64-byte handles, every rank maps its peers' buffers.  Used when all ranks
        succeed; B200MPPI_EXCHANGE=nccl keeps the collective-library exchange, =p2p makes failure an error."""
        import os
        import sys
        import torch
        import torch.distributed as dist
        want = os.environ.get("B200MPPI_EXCHANGE", "auto").lower()
        if want == "nccl":
            return False
        with torch.cuda.device(self.device):
            h = (C.c_ubyte * 64)()
            rc = lib.b200mppi_planner_p2p_export(self._handle, h, 64)
            why = "" if rc == 0 else lib.b200mppi_last_error().decode()
            handles = [None] * self.world_size
            dist.all_gather_object(handles, bytes(h) if rc == 0 else None, group=self.process_group)
            ok = all(x is not None for x in handles)
            if ok:
                blob = b"".join(handles)
                buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
                ok = lib.b200mppi_planner_p2p_import(self._handle, buf, len(blob)) == 0
                if not ok:
                    why = lib.b200mppi_last_error().decode()
            votes = [None] * self.world_size
            dist.all_gather_object(votes, (bool(ok), why), group=self.process_group)
        ok = all(v[0] for v in votes)
        if not ok:
            reasons = "; ".join("rank %d: %s" % (r, v[1]) for r, v in enumerate(votes) if not v[0])
            if want == "p2p":
                raise RuntimeError("peer-memory exchange unavailable (%s)" % reasons)
            if self.rank == 0:
                print("mppi_numba_b200: peer-memory exchange unavailable (%s); using the NCCL exchange" % reasons,
                      file=sys.stderr)
        return ok

    def _solve_sharded(self, u_out):
        import torch
        import torch.distributed as dist
        self._ensure_exchange()
        num_opt = int(self.params['num_opt'])
        if self._p2p:
            check(lib.b200mppi_planner_solve_p2p(self._handle, ptr(u_out)))
            return
        with torch.cuda.stream(self._stream):
            for k in range(num_opt):
                check(lib.b200mppi_planner_solve_local(self._handle, 1 if k == 0 else 0))
                if self.shard_maps:
                    # exchange 1: per-(m,n) costs, equal contiguous blocks: rank d receives every rank's block d = its control sequences
                    dist.all_to_all_single(self._costs_recv, self._costs_send, group=self.process_group)
                    check(lib.b200mppi_planner_solve_reduce(self._handle, C.c_void_p(self._costs_recv.data_ptr())))
                # exchange 2: the (2T+2)-float softmax partial of every rank
                dist.all_gather_into_tensor(self._gathered, self._partial_t, group=self.process_group)
                last = k == num_opt - 1
                check(lib.b200mppi_planner_solve_finish(
                    self._handle, C.c_void_p(self._gathered.data_ptr()), ptr(u_out) if last else None))
        if num_opt == 0:
            self.u_cur_d.copy_to_host(u_out)

    # ------------------------------------------------------------------ receding horizon
    def shift_and_update(self, new_x0, u_cur, num_shifts=1):
        self.params["x0"] = new_x0.copy()
        self.shift_optimal_control_sequence(u_cur, num_shifts)

    def shift_optimal_control_sequence(self, u_cur, num_shifts=1):
        """u[:-s] = u[s:] on the host copy the caller passes in (the tail keeps its old values), then
        one 8*T-byte upload into the persistent buffer (the reference re-allocates, mppi.py:539-542)."""
        shifted = u_cur.copy()
        shifted[:-num_shifts] = shifted[num_shifts:]
        shifted = np.ascontiguousarray(shifted, dtype=np.float32)
        check(lib.b200mppi_planner_set_u(self._handle, ptr(shifted)))

    # ------------------------------------------------------------------ visualisation
    def get_state_rollout(self):
        """State sequences (V, T+1, 3) of the current optimal controls: over the first V sampled maps
        (use_tdm) or, for the deterministic modes, the optimal sequence plus V-1 noisy samples."""
        assert self.params_set, "MPPI parameters are not set"
        assert self.tdm_set, "MPPI has not received TDMs"
        if not self.device_var_initialized:
            print("Device variables not initialized. Cannot run mppi.")
            return None
        self.move_mppi_task_vars_to_device()
        out = np.empty(self.state_rollout_batch_d.shape, dtype=np.float32)
        check(lib.b200mppi_planner_get_state_rollout(self._handle, ptr(out), out.nbytes))
        return out

    # ------------------------------------------------------------------ tracing / checkpoint
    def set_profiling(self, enable=True):
        check(lib.b200mppi_planner_set_profiling(self._handle, 1 if enable else 0))

    def last_timings(self):
        """CUDA-event milliseconds of each stage of the last solve (needs set_profiling(True))."""
        ms = (C.c_float * len(_lib.T_NAMES))()
        check(lib.b200mppi_planner_last_timings(self._handle, ms))
        return dict(zip(_lib.T_NAMES, [float(v) for v in ms]))

    def sample_box(self):
        """How the last solve() sampled the traction maps: ``(mode, row_lo, row_hi, col_lo, col_hi)`` with mode
        0 = whole maps (what the reference does every solve), 1 / 2 = only the cells its rollouts could reach
        (bound from the speed limit / from this solve's own clipped controls); results are identical either way
        (include/b200mppi.h, b200mppi_planner_sample_box)."""
        out = (C.c_int32 * 5)()
        check(lib.b200mppi_planner_sample_box(self._handle, C.byref(out)))
        return tuple(int(v) for v in out)

    def launch_count(self):
        n = C.c_int64()
        check(lib.b200mppi_planner_launch_count(self._handle, C.byref(n)))
        return int(n.value)

    def get_state(self):
        """Checkpoint: warm-start controls + noise RNG streams (+ both TDM streams if attached)."""
        st = dict(u_cur=self.u_cur_d.copy_to_host(), rng=self.rng_states_d.copy_to_host())
        if self.tdm_set:
            st["lin_rng"] = self.lin_tdm.rng_states_d.copy_to_host()
            st["ang_rng"] = self.ang_tdm.rng_states_d.copy_to_host()
        return st

    def set_state(self, st):
        self.u_cur_d.copy_to_device(st["u_cur"])
        self.rng_states_d.copy_to_device(st["rng"])
        if self.tdm_set and "lin_rng" in st:
            self.lin_tdm.rng_states_d.copy_to_device(st["lin_rng"])
            self.ang_tdm.rng_states_d.copy_to_device(st["ang_rng"])
