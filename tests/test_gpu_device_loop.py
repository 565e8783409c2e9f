"""Device loops on the GPU (run with ``-m gpu``): a torch plant drives ``batch.device_loop()`` and every pose fed and
every u returned is kept; replaying the same calls with those poses on identical twins through the host calls (u =
p.solve(), or MPPI_StochasticBatch([p]).solve() for use_tdm planners; p.shift_and_update(x[k], u_cur, 1)) gives u bit
for bit at every solve, and after close the same snapshot(), params['x0'] and next solve.  Covered: det, speed-map,
use_tdm (num_opt 1 and 2), barebone with obstacles, MPPI_MixedBatch, share_tdms with members that stop at different
steps, maps of mixed geometry, float32 / float64 / row-strided poses, a planner leaving its padded map, stop() between
a solve and its shift, two solves and two shifts in a row and a close right after a solve.  Also: the launches per
call, and that solve() and shift_and_update() return while the stream is still busy (no host wait)."""
import functools

import numpy as np
import pytest

from tests import gpu_harness as H
from tests import test_gpu_mixed_geometry_trials as MG
from tests import test_gpu_shared_tdm as SH
from tests.gpu_harness import assert_same, eng, quiet, snapshot, solve_in_batch_of_one  # noqa: F401
from tests.scenarios import make_scenario
from tests.test_gpu_barebone_trials import bb_setup
from tests.test_gpu_mixed_batch import planner as mixed_planner
from tests.test_gpu_trials import trial_setup

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def is_tdm(p):
    return bool(getattr(p, "use_tdm", False))


def solve_one(p):
    return solve_in_batch_of_one(p) if is_tdm(p) else p.solve()


def padded_ok(p, x):
    """check_solve_conditions' padded-limit test of pose x (float64)."""
    if getattr(p, "lin_tdm", None) is None:
        return True
    xl, yl = p.lin_tdm.padded_xlimits, p.lin_tdm.padded_ylimits
    return bool(xl[0] <= x[0] <= xl[1] and yl[0] <= x[1] <= yl[1])


class Driver(object):
    """Runs a device loop with a torch unicycle plant (dt per planner, float64 on the device) and keeps the calls."""

    def __init__(self, batch, A, dtype=torch.float64, strided=False):
        # the loop runs on torch's stream, so the plant, the loop's calls and torch's reads of u are ordered (torch's
        # array interface names no stream)
        batch.set_stream(torch.cuda.current_stream().cuda_stream)
        self.batch, self.A = batch, A
        self.dtype, self.strided = dtype, strided
        self.K = len(A)
        self.dt = torch.tensor([float(p.params["dt"]) for p in A], dtype=torch.float64, device="cuda")
        self.x = torch.tensor(np.stack([np.asarray(p.params["x0"], np.float64)[:3] for p in A]), device="cuda")
        self.calls = []
        self.u = None

    def pose(self):
        x = self.x.to(self.dtype)
        if self.strided:                                  # x[:, :3] of a (K, 4) tensor: rows 4 elements apart
            wide = torch.zeros((self.K, 4), dtype=self.dtype, device="cuda")
            wide[:, :3] = x
            return wide[:, :3]
        return x.contiguous()

    def solve(self, loop):
        self.u = torch.as_tensor(loop.solve(), device="cuda")
        self.calls.append(("solve", self.u.cpu().numpy().copy()))

    def step(self, kick=None):
        """The plant step with u[:, 0] of the last solve (NaN rows: no motion); kick: {k: (dx, dy)} added after."""
        v = torch.nan_to_num(self.u[:, 0, 0].double())
        w = torch.nan_to_num(self.u[:, 0, 1].double())
        th = self.x[:, 2]
        self.x = torch.stack([self.x[:, 0] + self.dt * torch.cos(th) * v, self.x[:, 1] + self.dt * torch.sin(th) * v,
                              th + self.dt * w], dim=1)
        for k, d in (kick or {}).items():
            self.x[k, :2] += torch.tensor(d, dtype=torch.float64, device="cuda")

    def shift(self, loop):
        x = self.pose()
        loop.shift_and_update(x)
        self.calls.append(("shift", x.cpu().numpy().astype(np.float64)))

    def stop(self, loop, ks):
        mask = torch.zeros(self.K, dtype=torch.bool, device="cuda")
        mask[list(ks)] = True
        loop.stop(mask)
        self.calls.append(("stop", mask.cpu().numpy()))


def replay(D, B, loop):
    """The recorded calls on the twins B through the host calls: u bit for bit at every solve (NaN once stopped), then
    every planner's snapshot, params['x0'] and one more solve against the loop's planners D.A."""
    A = D.A
    for k, p in enumerate(B):
        running, solves, shifts = True, 0, 0
        with quiet():
            for what, v in D.calls:
                if what == "solve":
                    if running:
                        u = solve_one(p)
                        solves += 1
                        assert_same(dict(u=v[k]), dict(u=u), "planner %d solve %d" % (k, solves))
                    else:
                        assert np.isnan(v[k]).all(), "planner %d: a stopped planner's row is not NaN" % k
                elif what == "shift" and running:
                    p.shift_and_update(v[k].copy(), p.u_cur_d.copy_to_host(), 1)
                    shifts += 1
                    running = padded_ok(p, v[k])
                elif what == "stop" and running and v[k]:
                    running = False
        assert loop.solves[k] == solves and loop.shifts[k] == shifts, (k, loop.solves[k], solves, loop.shifts[k], shifts)
        assert_same(snapshot(A[k]), snapshot(p), "planner %d" % k)
        assert np.asarray(A[k].params["x0"]).dtype == np.float64
        assert_same(dict(x0=np.asarray(A[k].params["x0"], np.float64)),
                    dict(x0=np.asarray(p.params["x0"], np.float64)), "planner %d x0" % k)
        if not is_tdm(p):
            assert (A[k].u_prev_d is A[k]._u_prev_buf) == (p.u_prev_d is p._u_prev_buf)
    with quiet():
        for k in range(len(A)):
            if loop.status[k] == "left_map":
                assert A[k].solve() is None and B[k].solve() is None
            else:
                ua, ub = solve_one(A[k]), solve_one(B[k])
                assert_same(dict(u=ua), dict(u=ub), "planner %d: the next solve" % k)
                assert_same(snapshot(A[k]), snapshot(B[k]), "planner %d after one more solve" % k)


def run(batch, A, steps, dtype=torch.float64, strided=False, kick=None, stops=None):
    """``steps`` rounds of solve, plant, shift; kick: {step: {k: (dx, dy)}}; stops: {step: ks} issued between the
    solve and the shift.  Returns (driver, loop)."""
    D = Driver(batch, A, dtype, strided)
    with batch.device_loop() as loop:
        for t in range(steps):
            D.solve(loop)
            D.step((kick or {}).get(t))
            if t in (stops or {}):
                D.stop(loop, stops[t])
            D.shift(loop)
    return D, loop


def onemap_twins(E, mode, K=5):
    return H.twins(functools.partial(trial_setup, E, mode), K)[:2]


@pytest.mark.parametrize("mode", ["det", "spd"])
def test_onemap_loop(eng, mode):
    E = eng
    A, B = onemap_twins(E, mode)
    batch = E.MPPI_Batch(A)
    D, loop = run(batch, A, 8, kick={3: {4: (100.0, 0.0)}}, stops={5: [1]})
    assert loop.status[4] == "left_map" and loop.status[1] == "stopped", loop.status
    replay(D, B, loop)


@pytest.mark.parametrize("num_opt", [1, 2])
def test_stochastic_loop(eng, num_opt):
    E = eng
    A, B, _ = H.twins(functools.partial(H.tdm_trial_setup, E, num_opt=num_opt), 5)
    batch = E.MPPI_StochasticBatch(A)
    D, loop = run(batch, A, 6, dtype=torch.float32, kick={2: {4: (0.0, -100.0)}}, stops={3: [0]})
    assert loop.status[4] == "left_map" and loop.status[0] == "stopped", loop.status
    replay(D, B, loop)


def test_barebone_loop_with_obstacles(eng):
    E = eng
    A, B, _ = H.twins(functools.partial(bb_setup, E), 6)
    batch = E.MPPI_Batch(A)
    D, loop = run(batch, A, 8, strided=True, kick={2: {0: (1e9, 0.0)}}, stops={4: [2, 5]})
    assert loop.status[0] == "running", "barebone planners have no map to leave"
    replay(D, B, loop)


def test_mixed_batch_loop(eng):
    E = eng
    order = [("tdm", 0), ("det", 2), ("spd", 4), ("tdm", 2), ("det", 0)]
    with quiet():
        A = [mixed_planner(E, kind, j)[0] for kind, j in order]
        B = [mixed_planner(E, kind, j)[0] for kind, j in order]
    batch = E.MPPI_MixedBatch(A)
    D, loop = run(batch, A, 6, kick={2: {1: (-100.0, 0.0)}}, stops={4: [3]})
    replay(D, B, loop)


@pytest.mark.parametrize("mode", ["det", "tdm"])
def test_share_tdms_members_stop_at_different_steps(eng, mode):
    E = eng
    if mode == "tdm":
        sc = H.tdm_scenario(0)
    else:
        sc = make_scenario(mode, N=200, M=1, T=20, H=64, W=64, res=0.2, B=5, seed=3, warm_start=True)
    K = 5
    A = SH.build(E, sc, K, shared=True)
    B = SH.build(E, sc, K, shared=False)
    SH.same_start(A, B)
    batch = (E.MPPI_StochasticBatch if mode == "tdm" else E.MPPI_Batch)(A, share_tdms=True)
    D, loop = run(batch, A, 7, stops={1: [0], 3: [2], 5: [4]})
    # the twins run on private pairs: compare each planner without its pair, and the shared pair with the copy of its
    # longest-running member (planners 0 .. K-2 share it; planner 1 and 3 run to the end, 1 first)
    saved = {}
    for k in range(K):
        saved[k] = SH.pair_state(A[k])
    with quiet():
        for k, p in enumerate(B):
            running = True
            for what, v in D.calls:
                if what == "solve" and running:
                    assert_same(dict(u=v[k]), dict(u=solve_one(p)), "planner %d" % k)
                elif what == "shift" and running:
                    p.shift_and_update(v[k].copy(), p.u_cur_d.copy_to_host(), 1)
                elif what == "stop" and v[k]:
                    running = False
    for k in range(K):
        assert_same(SH.planner_state(A[k]), SH.planner_state(B[k]), "planner %d" % k)
    assert_same(saved[0], SH.pair_state(B[1]), "the shared pair")
    assert_same(saved[K - 1], SH.pair_state(B[K - 1]), "the private pair")


def test_mixed_geometry_loop(eng):
    E = eng
    A, B = MG.build(E, "tdm", MG.SPECS), MG.build(E, "tdm", MG.SPECS)
    D, loop = run(E.MPPI_StochasticBatch(A), A, 5)
    replay(D, B, loop)
    A, B = MG.build(E, "det", MG.SPECS), MG.build(E, "det", MG.SPECS)
    D, loop = run(E.MPPI_Batch(A), A, 5)
    replay(D, B, loop)


def test_call_orders(eng):
    """Two solves in a row, two shifts in a row, a shift first, and a close right after a solve."""
    E = eng
    A, B = onemap_twins(E, "det", K=3)
    batch = E.MPPI_Batch(A)
    D = Driver(batch, A)
    with batch.device_loop() as loop:
        D.shift(loop)
        D.solve(loop)
        D.solve(loop)
        D.step()
        D.shift(loop)
        D.step()
        D.shift(loop)
        D.solve(loop)
    replay(D, B, loop)
    A2, B2, _ = H.twins(functools.partial(H.tdm_trial_setup, E), 3)
    D = Driver(E.MPPI_StochasticBatch(A2), A2)
    with D.batch.device_loop() as loop:
        D.solve(loop)
        D.solve(loop)
        D.step()
        D.shift(loop)
        D.shift(loop)
        D.solve(loop)
    replay(D, B2, loop)


def test_commit_on_exception_and_refusals(eng):
    E = eng
    A, B = onemap_twins(E, "spd", K=3)
    batch = E.MPPI_Batch(A)
    D = Driver(batch, A)
    with pytest.raises(RuntimeError, match="plant failed"):
        with batch.device_loop() as loop:
            D.solve(loop)
            D.step()
            D.shift(loop)
            with pytest.raises(ValueError, match="planner 1"):
                A[1].solve()
            with pytest.raises(ValueError, match="device loop"):
                batch.solve()
            with pytest.raises(ValueError, match="strides"):
                loop.shift_and_update(torch.zeros((3, 6), dtype=torch.float64, device="cuda")[:, ::2])
            with pytest.raises(ValueError, match="dtype"):
                loop.shift_and_update(torch.zeros((3, 3), dtype=torch.int32, device="cuda"))
            with pytest.raises(ValueError, match="shape"):
                loop.solve(out=torch.zeros((3, 5, 2), dtype=torch.float32, device="cuda"))
            with pytest.raises(TypeError, match="cuda_array_interface"):
                loop.stop(np.zeros(3, dtype=np.int32))
            raise RuntimeError("plant failed")
    assert batch._loop is None and loop.solves.tolist() == [1, 1, 1]
    with pytest.raises(ValueError, match="closed"):
        loop.solve()
    replay(D, B, loop)


def launches_per_solve(kind, num_opt, C1=1, C2=1):
    return {"onemap": 3 * num_opt + C1, "barebone": 3 * num_opt, "tdm": 4 * num_opt + 2 * C2,
            "mixed": 6 * num_opt + C1 + 2 * C2}[kind] + 1


@pytest.mark.parametrize("kind", ["onemap", "barebone", "tdm", "mixed"])
def test_launches_per_call(eng, kind):
    E = eng
    with quiet():
        if kind == "onemap":
            batch = E.MPPI_Batch(onemap_twins(E, "det", K=2)[0])
        elif kind == "barebone":
            batch = E.MPPI_Batch(H.twins(functools.partial(bb_setup, E, num_opt=2), 2)[0])
        elif kind == "tdm":
            batch = E.MPPI_StochasticBatch(H.twins(functools.partial(H.tdm_trial_setup, E), 2)[0])
        else:
            batch = E.MPPI_MixedBatch([mixed_planner(E, k, 2)[0] for k in ("det", "tdm")])
    num_opt = 2 if kind == "barebone" else 1
    D = Driver(batch, batch.planners)
    n0 = batch.launch_count()
    with batch.device_loop() as loop:
        assert batch.launch_count() == n0
        for _ in range(2):
            n = batch.launch_count()
            D.solve(loop)
            assert batch.launch_count() - n == launches_per_solve(kind, num_opt)
            D.step()
            n = batch.launch_count()
            D.shift(loop)
            assert batch.launch_count() - n == 1
            n = batch.launch_count()
            D.stop(loop, [])
            assert batch.launch_count() - n == 1


def test_no_host_wait(eng):
    E = eng
    A = onemap_twins(E, "det", K=2)[0]
    batch = E.MPPI_Batch(A)
    stream = torch.cuda.current_stream()
    batch.set_stream(stream.cuda_stream)
    x = torch.tensor(np.stack([np.asarray(p.params["x0"], np.float64)[:3] for p in A]), device="cuda")
    with batch.device_loop() as loop:
        loop.solve()                                    # every kernel loaded before the stream is held up
        loop.shift_and_update(x)
        torch.cuda.synchronize()
        for call in (lambda: loop.solve(), lambda: loop.shift_and_update(x)):
            torch.cuda._sleep(int(2e9))                 # about a second of GPU time queued first
            call()
            ev = torch.cuda.Event()
            ev.record(stream)
            assert not ev.query(), "the call waited for the stream"
            torch.cuda.synchronize()
    assert loop.solves.tolist() == [2, 2] and loop.shifts.tolist() == [2, 2]
