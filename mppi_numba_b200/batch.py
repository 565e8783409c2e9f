"""``MPPI_Batch`` -- K independent one-map planners solved together, one kernel launch per stage for the whole batch.

    from mppi_numba_b200 import MPPI_Batch
    batch = MPPI_Batch([planner_0, planner_1, ...])     # MPPI_Numba (use_det_dynamics or
                                                         # use_nom_dynamics_with_speed_map) or barebone.MPPI_Numba
    u = batch.solve()                                    # np.float32 (K, T, 2) == [p.solve() for p in planners]
    for k, p in enumerate(planners):
        p.shift_and_update(new_x0[k], u[k])             # the per-planner closed-loop calls stay as they are

Each planner keeps its own params, TDMs, warm start and RNG streams; ``solve()`` leaves every one of them exactly as
``planner.solve()`` called on planners[0], planners[1], ... in that order would (include/b200mppi.h, batched one-map
solves).  The planners must share N, T, the device and the mode; their TDMs must not be shared between planners.
"""
import ctypes as C

import numpy as np

from ._lib import check, lib, ptr


def _kind(p):
    """('barebone' | 'det' | 'spd' | 'tdm', world_size) of a planner object."""
    from .barebone import MPPI_Numba as Barebone
    if isinstance(p, Barebone):
        return "barebone", 1
    if getattr(p, "use_tdm", False):
        return "tdm", p.world_size
    if getattr(p, "use_det_dynamics", False):
        return "det", p.world_size
    if getattr(p, "use_nom_dynamics_with_speed_map", False):
        return "spd", p.world_size
    return "other", getattr(p, "world_size", 1)


class MPPI_Batch(object):
    """Borrows ``planners`` (keeps them alive) and solves them with one launch per stage."""

    def __init__(self, planners):
        planners = list(planners)
        if not planners:
            raise ValueError("MPPI_Batch: no planners")
        kinds = [_kind(p) for p in planners]
        for i, (kind, ws) in enumerate(kinds):
            if kind == "tdm":
                raise ValueError("MPPI_Batch: planner %d uses use_tdm: the stochastic mode is not batched" % i)
            if kind == "other":
                raise ValueError("MPPI_Batch: planner %d is neither a det-dynamics, speed-map nor barebone planner" % i)
            if ws != 1:
                raise ValueError("MPPI_Batch: planner %d has world_size %d (a batch holds single-rank planners)" % (i, ws))
            if kind != kinds[0][0]:
                raise ValueError("MPPI_Batch: planner %d is a %s planner, planner 0 a %s planner (kinds cannot be mixed)"
                                 % (i, kind, kinds[0][0]))
        self.planners = planners
        self.kind = kinds[0][0]
        self.num_steps = planners[0].num_steps
        self._handle = None
        handles = (C.c_void_p * len(planners))(*[p._handle.value for p in planners])
        h = C.c_void_p()
        check(lib.b200mppi_batch_create(handles, len(planners), C.byref(h)))
        self._handle = h

    def __del__(self):
        h, self._handle = getattr(self, "_handle", None), None
        if h:
            try:
                lib.b200mppi_batch_destroy(h)
            except Exception:
                pass

    def __len__(self):
        return len(self.planners)

    def solve(self):
        """One solve() of every planner.  Returns np.float32 (K, T, 2), or None (with the planner's index and the
        reason printed) when a planner's preconditions fail -- then nothing is solved."""
        for i, p in enumerate(self.planners):
            if not p.check_solve_conditions():
                print("MPPI_Batch: planner {}: MPPI solve condition not met. Cannot solve. Return".format(i))
                return None
        for p in self.planners:
            p.move_mppi_task_vars_to_device()          # each planner's params POD (and TDMs / obstacles)
        u = np.empty((len(self.planners), self.num_steps, 2), dtype=np.float32)
        check(lib.b200mppi_batch_solve(self._handle, ptr(u)))
        for p in self.planners:                        # as each planner's own solve() does (mppi.py:292,362)
            p.u_prev_d = p._u_prev_buf
        return u

    def set_stream(self, cuda_stream):
        """Issue the batch's work on ``cuda_stream`` (a raw cudaStream_t as int, e.g. torch's ``stream.cuda_stream``)."""
        check(lib.b200mppi_batch_set_stream(self._handle, C.c_void_p(int(cuda_stream))))

    def launch_count(self):
        """Kernel launches issued by this batch since it was created."""
        n = C.c_int64()
        check(lib.b200mppi_batch_launch_count(self._handle, C.byref(n)))
        return int(n.value)

