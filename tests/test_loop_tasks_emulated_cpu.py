"""A device loop's task updates (csrc/reduce.cu, ``[emu:... loop_task]``: set_goals and set_obstacles) emulated on the
host against a numpy restatement, bit for bit, over a mix of one-map (RolloutArgs) and stochastic (RolloutWinArgs)
descriptors filled with random bytes:
  - goals: float64 -> float32 rounding at ties, +-0, +-inf and NaN, float32 goals taken exactly, strided and permuted
    rows; the descriptor's goal is float32 of the row, the task keeps the float64 value;
  - obstacles: counts 0, O', -1 and O' + 1 (the last two stop the planner once, with "bad_obstacles", and decrement the
    running count once), no counts (O' each), float32 and float64 triples, strided planner rows; each planner's float32
    slice, its float64 shadow and its descriptor's obstacle count;
  - planners gated out by their active flag left untouched, and every descriptor byte other than the goal and the
    obstacle count unchanged."""

import numpy as np
import pytest

from tests.emu_core import build as _build
from tests.emu_core import region

HARNESS = r'''
#include <cstddef>
#include <vector>
using namespace b200;
// planner k's rollout descriptor lies at descs + offs[k]: a RolloutArgs (kinds[k] 0) or a RolloutWinArgs (1), and its
// task record's descriptor pointers are staged from it, as trial_call_stage does.  op 0: set_goals from arg (dtype,
// rows stride bytes apart); op 1: set_obstacles from arg (n = O' triples per row, counts may be null)
extern "C" void emu_task(int op, int K, unsigned char* descs, const int* kinds, const long long* offs, void* state,
                         int* active, int* count, void* task, float* obs, double* obs64, int O, const void* arg,
                         int dtype, int n, long long stride, const int* counts) {
  std::vector<TrialDev> d(K);
  LoopArgs a{d.data(), reinterpret_cast<LoopState*>(state), active, count, K, 1};
  LoopTask* t = reinterpret_cast<LoopTask*>(task);
  for (int k = 0; k < K; ++k) {
    if (kinds[k] == 0) {
      RolloutArgs* r = reinterpret_cast<RolloutArgs*>(descs + offs[k]);
      t[k].xgoal_out = r->p.xgoal;
      t[k].num_obstacles_out = &r->num_obstacles;
    } else {
      t[k].xgoal_out = reinterpret_cast<RolloutWinArgs*>(descs + offs[k])->p.xgoal;
      t[k].num_obstacles_out = nullptr;
    }
  }
  LoopTaskArgs ta{t, obs, obs64, O};
  const unsigned char* x = reinterpret_cast<const unsigned char*>(arg);
  if (op == 0)
    emu::launch({(unsigned)((K + 127) / 128), 1, 1}, 128,
                [&] { loop_goal_body(a, ta, x, dtype, stride, (int)(blockIdx.x * blockDim.x + threadIdx.x)); });
  if (op == 1)
    emu::launch({(unsigned)K, 1, 1}, 32,
                [&] { loop_obstacles_body(a, ta, x, dtype, n, stride, counts, (int)blockIdx.x, (int)threadIdx.x); });
}
// 0: sizeof RolloutArgs, 1: its goal's offset, 2: its obstacle count's offset, 3: sizeof RolloutWinArgs, 4: its goal's
// offset, 5: sizeof LoopTask, 6: sizeof LoopState, 7: LOOP_BAD_OBSTACLES
extern "C" long long emu_layout(int what) {
  const long long v[] = {(long long)sizeof(RolloutArgs), (long long)(offsetof(RolloutArgs, p) + offsetof(RolloutParams, xgoal)),
                         (long long)offsetof(RolloutArgs, num_obstacles), (long long)sizeof(RolloutWinArgs),
                         (long long)(offsetof(RolloutWinArgs, p) + offsetof(RolloutParams, xgoal)),
                         (long long)sizeof(LoopTask), (long long)sizeof(LoopState), (long long)LOOP_BAD_OBSTACLES};
  return v[what];
}
'''

STATE = np.dtype([("x", "<f8", 3), ("pxlim", "<f8", 2), ("pylim", "<f8", 2), ("x0", "<f4", 3), ("solves", "<i4"),
                  ("shifts", "<i4"), ("status", "<i4"), ("bounded", "<i4"), ("row", "<i4")])
TASK = np.dtype([("goal", "<f8", 2), ("xgoal_out", "<u8"), ("num_obstacles_out", "<u8"), ("took_goal", "<i4"),
                 ("took_obstacles", "<i4"), ("num_obstacles", "<i4"), ("pad_", "<i4")])
BAD_OBSTACLES, STOPPED = 6, 5


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = _build(str(tmp_path_factory.mktemp("loop_task_emu")), "loop_task_emu",
                 [region("common.cuh", "params"), region("kernels.h", "cost_dst"), region("kernels.h", "rollout_args"),
                  region("kernels.h", "win_args"), region("kernels.h", "trial_args"), region("kernels.h", "loop_args"),
                  region("kernels.h", "loop_task_args"), region("reduce.cu", "loop_task")], HARNESS)
    assert lib.emu_layout(5) == TASK.itemsize and lib.emu_layout(6) == STATE.itemsize
    assert lib.emu_layout(7) == BAD_OBSTACLES
    return lib


class Tasks(object):
    """K planners' descriptors (random bytes), loop state and task records, and the same restated in numpy (ref_*)."""

    def __init__(self, emu, K, O, kinds, seed=0, rows=None):
        rng = np.random.default_rng(seed)
        self.emu, self.K, self.O = emu, K, O
        self.kinds = np.asarray(kinds, dtype=np.int32)
        size = [int(emu.emu_layout(0)), int(emu.emu_layout(3))]
        self.goal_at = [int(emu.emu_layout(1)), int(emu.emu_layout(4))]
        self.count_at = int(emu.emu_layout(2))
        self.offs = np.cumsum([0] + [(size[k] + 63) // 64 * 64 for k in self.kinds]).astype(np.int64)
        self.descs = rng.integers(0, 256, int(self.offs[-1]), dtype=np.uint8)
        self.offs = self.offs[:-1].copy()
        self.state = np.zeros(K, dtype=STATE)
        self.state["row"] = np.arange(K) if rows is None else rows
        self.active = np.ones(K, dtype=np.int32)
        self.count = np.array([K], dtype=np.int32)
        self.task = np.zeros(K, dtype=TASK)
        self.obs = rng.standard_normal(K * O * 3).astype(np.float32)
        self.obs64 = rng.standard_normal(K * O * 3)

    def copy(self):
        c = Tasks.__new__(Tasks)
        c.__dict__ = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in self.__dict__.items()}
        return c

    def call(self, op, arg, dtype, n=0, counts=None):
        e = self.emu
        e.emu_task(op, self.K, self.descs.ctypes.data, self.kinds.ctypes.data, self.offs.ctypes.data,
                   self.state.ctypes.data, self.active.ctypes.data, self.count.ctypes.data, self.task.ctypes.data,
                   self.obs.ctypes.data, self.obs64.ctypes.data, self.O, arg.ctypes.data, dtype, n, arg.strides[0],
                   None if counts is None else counts.ctypes.data)

    def desc_goal(self, k):
        at = int(self.offs[k]) + self.goal_at[self.kinds[k]]
        return self.descs[at:at + 8].view(np.float32)

    def desc_count(self, k):
        at = int(self.offs[k]) + self.count_at
        return self.descs[at:at + 4].view(np.int32)

    # ---- numpy restatements
    def ref_goals(self, g):
        for k in range(self.K):
            if not self.active[k]:
                continue
            r = g[self.state["row"][k]]
            v = r.astype(np.float64)                       # float32 widened exactly
            f = r if r.dtype == np.float32 else r.astype(np.float32)
            self.desc_goal(k)[:] = f
            self.task["goal"][k] = v
            self.task["took_goal"][k] = 1

    def ref_obstacles(self, obs, counts=None):
        Op = obs.shape[1]
        for k in range(self.K):
            if not self.active[k]:
                continue
            row = self.state["row"][k]
            n = Op if counts is None else int(counts[row])
            if n < 0 or n > Op:
                self.state["status"][k] = BAD_OBSTACLES
                self.active[k] = 0
                self.count[0] -= 1
                continue
            flat = np.ascontiguousarray(obs[row]).reshape(-1)[:3 * n]
            at = k * self.O * 3
            self.obs[at:at + 3 * n] = flat.astype(np.float32)
            self.obs64[at:at + 3 * n] = flat.astype(np.float64)
            if self.kinds[k] == 0:
                self.desc_count(k)[:] = n
            self.task["num_obstacles"][k] = n
            self.task["took_obstacles"][k] = 1


def same(a, b):
    assert a.descs.tobytes() == b.descs.tobytes(), "descriptor bytes"
    assert a.state.tobytes() == b.state.tobytes(), "loop state"
    assert a.active.tolist() == b.active.tolist() and a.count.tolist() == b.count.tolist()
    for f in ("goal", "took_goal", "took_obstacles", "num_obstacles"):
        assert a.task[f].tobytes() == b.task[f].tobytes(), "task field " + f
    assert a.obs.tobytes() == b.obs.tobytes(), "float32 obstacle slices"
    assert a.obs64.tobytes() == b.obs64.tobytes(), "float64 shadow"


def goals_both(L, g, strided=False):
    R = L.copy()
    R.ref_goals(g)
    arg = g
    if strided:                                            # rows 5 elements apart
        arg = np.zeros((g.shape[0], 5), dtype=g.dtype)
        arg[:, :2] = g
    L.call(0, np.ascontiguousarray(arg), 1 if g.dtype == np.float32 else 0)
    R.task["xgoal_out"], R.task["num_obstacles_out"] = L.task["xgoal_out"], L.task["num_obstacles_out"]
    same(L, R)


def obstacles_both(L, obs, counts=None, pad=0):
    R = L.copy()
    R.ref_obstacles(obs, counts)
    K, Op = obs.shape[:2]
    arg = np.zeros((K, Op * 3 + pad), dtype=obs.dtype)     # planner rows pad elements longer than their triples
    arg[:, :Op * 3] = obs.reshape(K, -1)
    L.call(1, arg, 1 if obs.dtype == np.float32 else 0, Op, counts)
    same(L, R)


def test_goal_rounding(emu):
    one = 1.0
    tie_down, tie_up = one + 2.0 ** -24, one + 3 * 2.0 ** -24
    big = float(np.float32(3.4e38)) * 1.0000001            # rounds to float32 +inf
    g = np.array([[tie_down, tie_up], [-0.0, 0.0], [np.inf, -np.inf], [np.nan, big], [1e-46, -1e-46],
                  [0.1, -2.75]])
    L = Tasks(emu, 6, 2, [0, 1, 0, 1, 1, 0], seed=1, rows=np.array([3, 0, 5, 1, 4, 2]))
    goals_both(L, g)
    got = np.stack([L.desc_goal(k) for k in range(6)])
    want = g[L.state["row"]].astype(np.float32)
    assert got.view(np.uint32).tolist() == want.view(np.uint32).tolist()
    k = int(np.flatnonzero(L.state["row"] == 0)[0])
    assert L.desc_goal(k)[0] == 1.0 and L.desc_goal(k)[1] == np.float32(1 + 2.0 ** -22)
    assert L.task["goal"].view(np.uint64).tolist() == g[L.state["row"]].view(np.uint64).tolist()
    assert L.task["took_goal"].tolist() == [1] * 6
    goals_both(L, g[::-1].copy(), strided=True)            # a second set, rows 5 elements apart


def test_float32_goals_taken_exactly(emu):
    g = np.array([[0.1, 0.2], [np.float32(1e-40), -3.5], [-0.0, 7.0]], dtype=np.float32)
    L = Tasks(emu, 3, 0, [1, 0, 1], seed=2)
    goals_both(L, g, strided=True)
    assert L.task["goal"].tolist() == g.astype(np.float64).tolist()


def test_inactive_planners_untouched(emu):
    L = Tasks(emu, 5, 4, [0, 0, 1, 0, 0], seed=3)         # obstacles: barebone (one-map) descriptors only
    L.active[[1, 2]] = 0
    L.count[0] = 3
    before = L.copy()
    goals_both(L, np.full((5, 2), 4.5))
    obstacles_both(L, np.full((5, 4, 3), 0.25), np.array([1, 2, 3, 4, 0], np.int32))
    for k in (1, 2):
        assert L.desc_goal(k).tobytes() == before.desc_goal(k).tobytes()
        for f in ("goal", "took_goal", "took_obstacles", "num_obstacles"):
            assert L.task[f][k].tobytes() == before.task[f][k].tobytes()
        at = k * 4 * 3
        assert L.obs[at:at + 12].tobytes() == before.obs[at:at + 12].tobytes()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_obstacle_counts(emu, dtype):
    O, Op, K = 6, 4, 6
    rng = np.random.default_rng(4)
    L = Tasks(emu, K, O, [0] * K, seed=5, rows=np.array([5, 4, 3, 2, 1, 0]))
    obs = rng.uniform(-5, 5, (K, Op, 3)).astype(dtype)
    obs[0, 0] = [np.nan, np.inf, 0.0]                      # passed through as they are
    obs[1, 1] = [1.0 + 2.0 ** -24, -0.0, 1e-46]
    counts = np.array([0, Op, -1, Op + 1, 2, 1], dtype=np.int32)     # by row
    obstacles_both(L, obs, counts, pad=5)
    by_row = L.state["status"][np.argsort(L.state["row"])]
    assert by_row.tolist() == [0, 0, BAD_OBSTACLES, BAD_OBSTACLES, 0, 0] and L.count[0] == K - 2
    assert [int(L.desc_count(k)[0]) for k in range(K) if L.active[k]] == [1, 2, Op, 0]
    # the stopped planners keep their last set and are not counted again; no counts: O' each
    obstacles_both(L, obs[:, :3].copy(), np.array([-1, 3, 9, 9, 0, 0], dtype=np.int32))
    assert L.count[0] == K - 2 - 1
    obstacles_both(L, obs[:, :3].copy())
    assert [int(L.desc_count(k)[0]) for k in range(K) if L.active[k]] == [3, 3, 3]
    assert L.task["took_obstacles"].tolist() == [1, 1, 0, 0, 1, 1]


def test_no_obstacles_and_full_capacity(emu):
    K, O = 3, 5
    L = Tasks(emu, K, O, [0, 0, 0], seed=6)
    obstacles_both(L, np.zeros((K, 0, 3)))                 # O' 0: every planner takes no obstacles
    assert [int(L.desc_count(k)[0]) for k in range(K)] == [0, 0, 0] and L.task["took_obstacles"].tolist() == [1] * 3
    rng = np.random.default_rng(7)
    obstacles_both(L, rng.standard_normal((K, O, 3)))
    assert [int(L.desc_count(k)[0]) for k in range(K)] == [O] * K
    L.call(1, np.zeros((K, 3)), 0, 1, np.array([2, 0, 1], np.int32))      # count 2 > O' 1: planner 0 stops
    assert L.state["status"].tolist() == [BAD_OBSTACLES, 0, 0] and L.count[0] == 2
