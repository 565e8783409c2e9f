"""The device-loop kernels (csrc/reduce.cu, ``[emu:... loop]``: export, ingest and stop) emulated on the host against a
numpy restatement of each, bit for bit: the in-place one-row shift of u_cur (T = 1, 2, 33), float32 rounding of
float64 poses at ties, +-0, +-inf and NaN, the padded-limit rule at lo, hi and one ulp outside, the stochastic window
origin, NaN rows of planners that no longer run, the solve and shift counters, one-way stop, and planners gated out
by their active flag left untouched."""
import ctypes as C

import numpy as np
import pytest

from tests.emu_core import build as _build
from tests.emu_core import region

HARNESS = r'''
using namespace b200;
// planner i: u_cur[i] (T, 2), x0_out[i] (3 floats), win[i] (6 ints: WW, WH, wx0, wy0, ww, wh; null: no window) over a
// map of geo[3 i ..] = pxl, pyl, res and dims[2 i ..] = rows, cols.  op 0: export into out; 1: ingest the poses at arg
// (dtype kind, rows stride bytes apart); 2: stop with the mask at arg (kind: element bytes)
extern "C" void emu_loop(int op, int K, int T, float** u_cur, float** x0_out, int** win, const float* geo,
                         const int* dims, void* state, int* active, int* count, const void* arg, int kind,
                         long long stride, float* out) {
  std::vector<TrialDev> d(K);
  for (int i = 0; i < K; ++i) {
    d[i] = TrialDev{};
    d[i].u_cur = u_cur[i]; d[i].x0_out = x0_out[i]; d[i].win = win[i];
    d[i].win_pxl = geo[3 * i]; d[i].win_pyl = geo[3 * i + 1]; d[i].win_res = geo[3 * i + 2];
    d[i].win_rows = dims[2 * i]; d[i].win_cols = dims[2 * i + 1];
  }
  LoopArgs a{d.data(), reinterpret_cast<LoopState*>(state), active, count, K, T};
  if (op == 0) emu::launch({(unsigned)K, 1, 1}, 128, [&] { loop_export_body(a, out, (int)blockIdx.x); });
  if (op == 1)
    emu::launch({(unsigned)K, 1, 1}, 32, [&] {
      loop_ingest_body(a, reinterpret_cast<const unsigned char*>(arg), kind, stride, (int)blockIdx.x, (int)threadIdx.x);
    });
  if (op == 2)
    emu::launch({(unsigned)((K + 127) / 128), 1, 1}, 128,
                [&] { loop_stop_body(a, arg, kind, (int)(blockIdx.x * blockDim.x + threadIdx.x)); });
}
extern "C" int emu_loop_state_bytes() { return (int)sizeof(b200::LoopState); }
'''

STATE = np.dtype([("x", "<f8", 3), ("pxlim", "<f8", 2), ("pylim", "<f8", 2), ("x0", "<f4", 3), ("solves", "<i4"),
                  ("shifts", "<i4"), ("status", "<i4"), ("bounded", "<i4"), ("row", "<i4")])
RUNNING, LEFT_MAP, STOPPED = 0, 3, 5


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = _build(str(tmp_path_factory.mktemp("loop_emu")), "loop_emu",
                 [region("kernels.h", "trial_args"), region("kernels.h", "loop_args"), region("reduce.cu", "trial"),
                  region("reduce.cu", "loop")], HARNESS)
    assert lib.emu_loop_state_bytes() == STATE.itemsize
    return lib


class Loop(object):
    """K planners' device-side loop state, and the same restated in numpy (``ref_*``)."""

    def __init__(self, K, T, seed=0, rows=None, windows=False):
        rng = np.random.default_rng(seed)
        self.K, self.T = K, T
        self.u = [rng.standard_normal((T, 2)).astype(np.float32) for _ in range(K)]
        self.x0 = [rng.standard_normal(3).astype(np.float32) for _ in range(K)]
        self.geo = np.array([[-1.5, -2.25, 0.2]] * K, dtype=np.float32)
        self.dims = np.array([[64, 80]] * K, dtype=np.int32)
        self.win = [np.array([32, 24, -7, -7, -7, -7], dtype=np.int32) if windows else None for _ in range(K)]
        self.state = np.zeros(K, dtype=STATE)
        self.state["pxlim"] = (-1.5, 14.5)
        self.state["pylim"] = (-2.25, 10.55)
        self.state["bounded"] = 1
        self.state["row"] = np.arange(K) if rows is None else rows
        self.active = np.ones(K, dtype=np.int32)
        self.count = np.array([K], dtype=np.int32)

    def copy(self):
        c = Loop.__new__(Loop)
        c.__dict__ = {k: ([None if a is None else a.copy() for a in v] if isinstance(v, list) else
                          (v.copy() if isinstance(v, np.ndarray) else v)) for k, v in self.__dict__.items()}
        return c

    def call(self, emu, op, arg=None, kind=0, stride=0, out=None):
        P = lambda arrs: (C.c_void_p * self.K)(*[None if a is None else a.ctypes.data for a in arrs])   # noqa: E731
        emu.emu_loop(op, self.K, self.T, P(self.u), P(self.x0), P(self.win), self.geo.ctypes.data,
                     self.dims.ctypes.data, self.state.ctypes.data, self.active.ctypes.data, self.count.ctypes.data,
                     None if arg is None else arg.ctypes.data, kind, stride, None if out is None else out.ctypes.data)

    # ---- numpy restatements
    def ref_export(self, out):
        for k in range(self.K):
            s = self.state[k]
            if self.active[k]:
                out[s["row"]] = self.u[k]
                s["solves"] += 1
                s["x0"] = self.x0[k]
            else:
                out[s["row"]] = np.float32(np.nan)

    def ref_ingest(self, x):
        for k in range(self.K):
            if not self.active[k]:
                continue
            s = self.state[k]
            u = self.u[k]
            u[:-1] = u[1:].copy()
            p = np.asarray(x[s["row"]], dtype=np.float64)
            s["x"] = p
            s["shifts"] += 1
            inside = s["pxlim"][0] <= p[0] <= s["pxlim"][1] and s["pylim"][0] <= p[1] <= s["pylim"][1]
            if s["bounded"] and not inside:
                s["status"] = LEFT_MAP
                self.active[k] = 0
                self.count[0] -= 1
                continue
            self.x0[k][:] = p.astype(np.float32)
            if self.win[k] is not None:
                self.win[k][:] = win_origin(self.x0[k], self.geo[k], self.dims[k], self.win[k])

    def ref_stop(self, mask):
        for k in range(self.K):
            s = self.state[k]
            if self.active[k] and mask[s["row"]]:
                s["status"] = STOPPED
                self.active[k] = 0
                self.count[0] -= 1


def win_origin(x0, geo, dims, f):
    """kernels.h win_origin: the window of WW x WH cells around the robot's cell, inside the map, x origin a multiple of
    16."""
    pxl, pyl, res = (float(v) for v in geo)
    rows, cols = int(dims[0]), int(dims[1])
    xi0 = int(np.floor((float(x0[0]) - pxl) / res))
    yi0 = int(np.floor((float(x0[1]) - pyl) / res))
    WW, WH = int(f[0]), int(f[1])
    cx, cy = min(xi0 - WW // 2, cols - WW), min(yi0 - WH // 2, rows - WH)
    cx, cy = max(cx, 0), max(cy, 0)
    ox = cx & ~15
    return np.array([WW, WH, ox, cy, min(WW, cols - ox), min(WH, rows - cy)], dtype=np.int32)


def same(a, b):
    assert len(a.u) == len(b.u)
    for k in range(a.K):
        assert a.u[k].tobytes() == b.u[k].tobytes(), "u_cur of planner %d" % k
        assert a.x0[k].tobytes() == b.x0[k].tobytes(), "x0_out of planner %d" % k
        if a.win[k] is not None:
            assert a.win[k].tolist() == b.win[k].tolist(), "window of planner %d" % k
    assert a.state.tobytes() == b.state.tobytes()
    assert a.active.tolist() == b.active.tolist() and a.count.tolist() == b.count.tolist()


def ingest_both(emu, L, x, strided=False):
    R = L.copy()
    R.ref_ingest(x.astype(np.float64) if x.dtype == np.float32 else x)
    if strided:                                            # rows 5 elements apart
        wide = np.zeros((x.shape[0], 5), dtype=x.dtype)
        wide[:, :3] = x
        L.call(emu, 1, wide, 1 if x.dtype == np.float32 else 0, wide.strides[0])
    else:
        x = np.ascontiguousarray(x)
        L.call(emu, 1, x, 1 if x.dtype == np.float32 else 0, x.strides[0])
    same(L, R)


@pytest.mark.parametrize("T", [1, 2, 33])
def test_shift_and_counters(emu, T):
    L = Loop(3, T, seed=T, rows=np.array([2, 0, 1]))
    x = np.array([[0.5, 0.5, 0.1], [1.0, 2.0, -0.3], [3.0, 0.25, 1e-9]])
    for strided in (False, True):
        ingest_both(emu, L, x, strided)
    assert L.state["shifts"].tolist() == [2, 2, 2]
    out = np.full((3, T, 2), -7.0, np.float32)
    R = L.copy()
    ref = out.copy()
    R.ref_export(ref)
    L.call(emu, 0, out=out)
    same(L, R)
    assert out.tobytes() == ref.tobytes()
    assert L.state["solves"].tolist() == [1, 1, 1]


def test_float32_rounding_of_poses(emu):
    one = 1.0
    tie_even_down = one + 2.0 ** -24                       # halfway between 1 and 1 + 2^-23: to even, 1
    tie_even_up = one + 3 * 2.0 ** -24                     # halfway between 1 + 2^-23 and 1 + 2^-22: 1 + 2^-22
    big = float(np.float32(3.4e38)) * 1.0000001            # rounds to float32 +inf
    poses = np.array([[tie_even_down, tie_even_up, -0.0], [-tie_even_up, 0.0, np.inf], [1e-46, -1e-46, -np.inf],
                      [big, 2.5, np.nan]])
    L = Loop(4, 5, seed=4)
    L.state["bounded"] = 0                                 # barebone: no limits, every pose taken
    ingest_both(emu, L, poses)
    got = np.stack(L.x0)
    assert got.view(np.uint32).tolist() == poses.astype(np.float32).view(np.uint32).tolist()
    assert got[0, 0] == 1.0 and got[0, 1] == np.float32(1 + 2.0 ** -22) and np.signbit(got[0, 2])
    L32 = Loop(2, 4, seed=5)
    ingest_both(emu, L32, np.array([[0.1, 0.2, -0.0], [np.float32(1e-40), 3.0, 1.5]], dtype=np.float32))
    assert L32.state["x"][0].tolist() == [float(np.float32(0.1)), float(np.float32(0.2)), -0.0]


def test_padded_limit_rule(emu):
    lo, hi = -1.5, 14.5
    down, up = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
    ylo, yhi = -2.25, 10.55
    xs = [(lo, 0.0), (hi, 0.0), (down, 0.0), (up, 0.0), (0.0, ylo), (0.0, yhi), (0.0, np.nextafter(ylo, -np.inf)),
          (0.0, np.nextafter(yhi, np.inf)), (np.nan, 0.0), (0.0, np.nan)]
    L = Loop(len(xs), 6, seed=6, windows=True)
    x = np.array([[a, b, 0.3] for a, b in xs])
    ingest_both(emu, L, x)
    assert L.state["status"].tolist() == [0, 0, 3, 3, 0, 0, 3, 3, 3, 3]
    assert L.active.tolist() == [1, 1, 0, 0, 1, 1, 0, 0, 0, 0] and L.count[0] == 4
    # the planners that left are untouched by every later call
    before = L.copy()
    ingest_both(emu, L, np.zeros((len(xs), 3)))
    for k in (2, 3, 6, 7, 8, 9):
        assert L.u[k].tobytes() == before.u[k].tobytes() and L.x0[k].tobytes() == before.x0[k].tobytes()
        assert L.state[k].tobytes() == before.state[k].tobytes()


def test_window_origins(emu):
    rng = np.random.default_rng(9)
    x = np.column_stack([rng.uniform(-1.5, 14.5, 40), rng.uniform(-2.25, 10.55, 40), rng.uniform(-3, 3, 40)])
    x[:4, :2] = [[-1.5, -2.25], [14.5, 10.55], [-1.49, 10.5], [14.49, -2.2]]     # the corners: clamped windows
    L = Loop(40, 8, seed=10, windows=True)
    ingest_both(emu, L, x)
    assert all(w[2] % 16 == 0 for w in L.win)


def test_nan_rows_and_one_way_stop(emu):
    L = Loop(5, 7, seed=11, rows=np.array([4, 3, 2, 1, 0]))
    mask = np.array([0, 1, 0, 0, 1], dtype=np.int32)       # by row: planners 3 and 0
    R = L.copy()
    R.ref_stop(mask)
    L.call(emu, 2, mask, 4)
    same(L, R)
    assert L.state["status"].tolist() == [STOPPED, 0, 0, STOPPED, 0] and L.count[0] == 3
    # a bool mask, and a planner stopped twice: stays stopped, counted once
    bmask = np.array([1, 1, 0, 0, 0], dtype=np.bool_)
    R = L.copy()
    R.ref_stop(bmask)
    L.call(emu, 2, bmask, 1)
    same(L, R)
    assert L.state["status"].tolist() == [STOPPED, 0, 0, STOPPED, STOPPED] and L.count[0] == 2
    out = np.zeros((5, 7, 2), np.float32)
    R = L.copy()
    ref = out.copy()
    R.ref_export(ref)
    L.call(emu, 0, out=out)
    same(L, R)
    assert out.tobytes() == ref.tobytes()
    assert np.isnan(out[[4, 1, 0]]).all() and not np.isnan(out[[3, 2]]).any()
    assert L.state["solves"].tolist() == [0, 1, 1, 0, 0]
    ingest_both(emu, L, np.full((5, 3), 1.0))
    assert L.state["shifts"].tolist() == [0, 1, 1, 0, 0]
    R = L.copy()
    L.call(emu, 2, np.zeros(5, np.int32), 4)               # an all-zero mask changes nothing
    same(L, R)
