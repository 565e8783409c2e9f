"""Device-loop task updates on the GPU (run with ``-m gpu``): ``set_goals`` and ``set_obstacles`` calls recorded beside
the solves, shifts and stops of a torch-driven loop are replayed on identical twins through the host calls
(``p.params['xgoal'] = g[k]``; ``p.params['obstacle_positions'] = obs[k, :n, :2]``, ``['obstacle_radius'] =
obs[k, :n, 2]``).  u must match bit for bit at every solve, and after close every planner's snapshot(), params (x0,
xgoal, obstacles as float64) and one more solve.  Covered: det, speed-map and use_tdm (num_opt 1 and 2), a mixed batch,
share_tdms and mixed map geometries; a goal set between a solve and its shift, two sets in a row and a set after a
stop; barebone robots whose obstacles are the other robots' torch-computed positions with counts 0, between and the
capacity, row-strided and float32 sets; a bad count stopping one planner; the C-side commit (a direct batch solve after
close, without set_params); the launches (+1 per call, and a loop without task calls as before); no host wait; and a
graph-captured step with a torch waypoint switch and swarm obstacles, replayed and mixed with eager steps."""
import functools

import numpy as np
import pytest

from tests import gpu_harness as H
from tests import test_gpu_mixed_geometry_trials as MG
from tests import test_gpu_shared_tdm as SH
from tests.gpu_harness import assert_same, eng, quiet, snapshot  # noqa: F401
from tests.scenarios import make_scenario
from tests.test_gpu_barebone_trials import bb_setup
from tests.test_gpu_device_loop import Driver, launches_per_solve, onemap_twins, padded_ok, solve_one
from tests.test_gpu_loop_graphs import GraphDriver
from tests.test_gpu_mixed_batch import planner as mixed_planner

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

STATIC = [[5.0, 4.5, 1.5], [2.0, 1.0, 1.0]]           # bb_setup's two obstacles
ROBOT_R = 0.3


class TaskDriver(Driver):
    """Driver that also sets goals and obstacles and keeps those calls."""

    def goals(self, loop, g):
        loop.set_goals(g)
        self.calls.append(("goals", g.cpu().numpy().copy()))

    def obstacles(self, loop, obs, counts=None):
        loop.set_obstacles(obs, counts)
        self.calls.append(("obstacles", obs.cpu().numpy().copy(), None if counts is None else counts.cpu().numpy()))

    def base_goals(self):
        return torch.tensor(np.stack([np.asarray(p.params["xgoal"], np.float64)[:2] for p in self.A]), device="cuda")


@functools.lru_cache(maxsize=None)
def _swarm_tables(K):
    """The others' indices (K, K - 1) and the static obstacles (K, 2, 3), made once (a capture may not upload them)."""
    idx = torch.tensor([[j for j in range(K) if j != k] for k in range(K)], device="cuda")
    return idx, torch.tensor(STATIC, dtype=torch.float64, device="cuda").expand(K, 2, 3)


def swarm_obstacles(x, dtype=torch.float64):
    """(K, 2 + K - 1, 3): the two static obstacles, then every other robot at its current position (radius ROBOT_R)."""
    K = x.shape[0]
    idx, static = _swarm_tables(K)
    others = torch.cat([x[idx, :2], torch.full((K, K - 1, 1), ROBOT_R, dtype=x.dtype, device=x.device)], dim=2)
    return torch.cat([static, others], dim=1).to(dtype)


def replay_tasks(D, B, loop, next_solve=True):
    """The recorded calls on the twins B through the host calls: u bit for bit at every solve, then every planner's
    snapshot, params and (next_solve) one more solve, against the loop's planners D.A."""
    A = D.A
    for k, p in enumerate(B):
        running, solves, shifts, status = True, 0, 0, "running"
        with quiet():
            for call in D.calls:
                what, v = call[0], call[1]
                if what == "solve":
                    if running:
                        u = solve_one(p)
                        solves += 1
                        assert_same(dict(u=v[k]), dict(u=u), "planner %d solve %d" % (k, solves))
                    else:
                        assert np.isnan(v[k]).all(), "planner %d: a stopped planner's row is not NaN" % k
                elif not running:
                    continue
                elif what == "shift":
                    p.shift_and_update(v[k].copy(), p.u_cur_d.copy_to_host(), 1)
                    shifts += 1
                    if not padded_ok(p, v[k]):
                        running, status = False, "left_map"
                elif what == "stop" and v[k]:
                    running, status = False, "stopped"
                elif what == "goals":
                    p.params["xgoal"] = v[k].copy()
                elif what == "obstacles":
                    n = v.shape[1] if call[2] is None else int(call[2][k])
                    if n < 0 or n > v.shape[1]:
                        running, status = False, "bad_obstacles"
                    else:
                        p.params["obstacle_positions"] = v[k, :n, :2].copy()
                        p.params["obstacle_radius"] = v[k, :n, 2].copy()
        assert (loop.solves[k], loop.shifts[k], loop.status[k]) == (solves, shifts, status), (k, loop.status[k])
        assert_same(snapshot(A[k]), snapshot(p), "planner %d" % k)
        for key in ("x0", "xgoal", "obstacle_positions", "obstacle_radius"):
            a, b = A[k].params.get(key), p.params.get(key)
            assert (a is None) == (b is None), (k, key)
            if a is not None:
                if np.asarray(b).dtype == np.float32:  # a float32 goal widened exactly
                    assert np.asarray(a).dtype == np.float64, (k, key)
                assert_same({key: np.asarray(a, np.float64)}, {key: np.asarray(b, np.float64)}, "planner %d" % k)
    if not next_solve:
        return
    with quiet():
        for k in range(len(A)):
            if loop.status[k] == "left_map":
                assert A[k].solve() is None and B[k].solve() is None
            else:
                ua, ub = solve_one(A[k]), solve_one(B[k])
                assert_same(dict(u=ua), dict(u=ub), "planner %d: the next solve" % k)
                assert_same(snapshot(A[k]), snapshot(B[k]), "planner %d after one more solve" % k)


def goal_schedule(D, loop, steps, kick=None, stops=None, dtype=torch.float64):
    """``steps`` rounds of solve, plant, shift, with goals set between a solve and its shift (step 1), twice in a row
    (step 2: float32, then rows 3 elements apart), and after the stops (step 5 and the last step)."""
    rng = np.random.default_rng(11)
    base = D.base_goals()
    K = D.K

    def near():
        return base + torch.tensor(rng.uniform(-0.6, 0.6, (K, 2)), device="cuda")

    for t in range(steps):
        D.solve(loop)
        if t == 1:
            D.goals(loop, near())
        D.step((kick or {}).get(t))
        if t in (stops or {}):
            D.stop(loop, stops[t])
        D.shift(loop)
        if t == 2:
            D.goals(loop, near().float())
            wide = torch.zeros((K, 3), dtype=torch.float64, device="cuda")
            wide[:, :2] = near()
            D.goals(loop, wide[:, :2])
        if t in (5, steps - 1):
            D.goals(loop, near().to(dtype))


@pytest.mark.parametrize("mode", ["det", "spd"])
def test_onemap_goals(eng, mode):
    E = eng
    A, B = onemap_twins(E, mode)
    D = TaskDriver(E.MPPI_Batch(A), A)
    with D.batch.device_loop() as loop:
        goal_schedule(D, loop, 8, kick={3: {4: (100.0, 0.0)}}, stops={4: [1]})
    assert loop.status[4] == "left_map" and loop.status[1] == "stopped", loop.status
    replay_tasks(D, B, loop)


@pytest.mark.parametrize("num_opt", [1, 2])
def test_stochastic_goals(eng, num_opt):
    E = eng
    A, B, _ = H.twins(functools.partial(H.tdm_trial_setup, E, num_opt=num_opt), 4)
    D = TaskDriver(E.MPPI_StochasticBatch(A), A, dtype=torch.float32)
    with D.batch.device_loop() as loop:
        goal_schedule(D, loop, 7, stops={3: [0]}, dtype=torch.float32)
    replay_tasks(D, B, loop)


def test_mixed_batch_goals(eng):
    E = eng
    order = [("tdm", 0), ("det", 2), ("spd", 4), ("tdm", 2), ("det", 0)]
    with quiet():
        A = [mixed_planner(E, kind, j)[0] for kind, j in order]
        B = [mixed_planner(E, kind, j)[0] for kind, j in order]
    D = TaskDriver(E.MPPI_MixedBatch(A), A)
    with D.batch.device_loop() as loop:
        goal_schedule(D, loop, 6, stops={4: [3]})
    replay_tasks(D, B, loop)


def test_mixed_geometry_goals(eng):
    E = eng
    for mode, Batch in (("tdm", E.MPPI_StochasticBatch), ("det", E.MPPI_Batch)):
        A, B = MG.build(E, mode, MG.SPECS), MG.build(E, mode, MG.SPECS)
        D = TaskDriver(Batch(A), A)
        with D.batch.device_loop() as loop:
            goal_schedule(D, loop, 5)
        replay_tasks(D, B, loop)


@pytest.mark.parametrize("mode", ["det", "tdm"])
def test_share_tdms_goals(eng, mode):
    """Members of shared pairs that take different goals and stop at different steps, each against its private twin,
    the shared pair against the copy of its longest-running member (planners 0 .. K-2 share it, 1 and 3 run on)."""
    E = eng
    sc = H.tdm_scenario(0) if mode == "tdm" else make_scenario(mode, N=200, M=1, T=20, H=64, W=64, res=0.2, B=5,
                                                               seed=3, warm_start=True)
    K = 5
    A, B = SH.build(E, sc, K, shared=True), SH.build(E, sc, K, shared=False)
    SH.same_start(A, B)
    D = TaskDriver((E.MPPI_StochasticBatch if mode == "tdm" else E.MPPI_Batch)(A, share_tdms=True), A)
    with D.batch.device_loop() as loop:
        goal_schedule(D, loop, 7, stops={1: [0], 3: [2], 5: [4]})
    saved = {k: SH.pair_state(A[k]) for k in range(K)}
    with quiet():
        for k, p in enumerate(B):
            running = True
            for call in D.calls:
                what, v = call[0], call[1]
                if what == "solve" and running:
                    assert_same(dict(u=v[k]), dict(u=solve_one(p)), "planner %d" % k)
                elif what == "shift" and running:
                    p.shift_and_update(v[k].copy(), p.u_cur_d.copy_to_host(), 1)
                elif what == "goals" and running:
                    p.params["xgoal"] = v[k].copy()
                elif what == "stop" and v[k]:
                    running = False
    for k in range(K):
        assert_same(SH.planner_state(A[k]), SH.planner_state(B[k]), "planner %d" % k)
        assert_same(dict(g=np.asarray(A[k].params["xgoal"])), dict(g=np.asarray(B[k].params["xgoal"], np.float64)),
                    "planner %d goal" % k)
    assert_same(saved[0], SH.pair_state(B[1]), "the shared pair")
    assert_same(saved[K - 1], SH.pair_state(B[K - 1]), "the private pair")


def swarm(D, loop, steps, bad_at=None, with_goals=True):
    """Barebone robots that avoid each other: after each plant step every robot's obstacles are the statics and the
    others' positions, with counts cycling through 0, between and the capacity (None: all), float32 and row-strided
    sets on some steps; bad_at: the step at which robot 2's count is -1."""
    K = D.K
    Op = 2 + K - 1
    cycle = [None, [0, 3, Op, 5, 2, Op], [Op, 0, 1, Op, 4, 0][:K], None]
    for t in range(steps):
        D.solve(loop)
        D.step()
        D.shift(loop)
        obs = swarm_obstacles(D.x, torch.float32 if t == 2 else torch.float64)
        if t == 3:                                      # planner rows 9 triples apart
            wide = torch.zeros((K, Op + 2, 3), dtype=obs.dtype, device="cuda")
            wide[:, :Op] = obs
            obs = wide[:, :Op]
        c = cycle[t % len(cycle)]
        counts = None if c is None else torch.tensor(c[:K], dtype=torch.int32, device="cuda")
        if t == bad_at:
            counts = torch.full((K,), Op, dtype=torch.int32, device="cuda")
            counts[2] = -1
        D.obstacles(loop, obs, counts)
        if with_goals and t == 1:
            D.goals(loop, D.base_goals() + 0.5)
    D.solve(loop)


def test_barebone_swarm_obstacles(eng):
    E = eng
    K = 6
    A, B, _ = H.twins(functools.partial(bb_setup, E), K)
    D = TaskDriver(E.MPPI_Batch(A), A)
    with D.batch.device_loop(max_obstacles=2 + K - 1) as loop:
        assert loop.max_obstacles == 2 + K - 1
        swarm(D, loop, 7, bad_at=4)
    assert loop.status[2] == "bad_obstacles", loop.status
    replay_tasks(D, B, loop)


def test_c_side_commit(eng):
    """After close, a direct b200mppi_batch_solve (no set_params) plans toward the committed goal and obstacles: the
    same u and state as the twins' batch after their host loop, whose last solve uploaded the same params."""
    E = eng
    from mppi_numba_b200._lib import check, lib, ptr
    for barebone in (True, False):
        if barebone:
            K = 4
            A, B, _ = H.twins(functools.partial(bb_setup, E), K)
        else:
            K = 3
            A, B = onemap_twins(E, "det", K=K)
        D = TaskDriver(E.MPPI_Batch(A), A)
        with D.batch.device_loop(max_obstacles=8 if barebone else 0) as loop:
            if barebone:
                swarm(D, loop, 3)
                D.obstacles(loop, swarm_obstacles(D.x)[:, :4].contiguous(),
                            torch.tensor([4, 1, 0, 3], dtype=torch.int32, device="cuda"))
            D.goals(loop, D.base_goals() - 0.25)
            D.solve(loop)
        replay_tasks(D, B, loop, next_solve=False)
        u = {}
        for name, batch in (("loop", D.batch), ("twins", E.MPPI_Batch(B))):
            u[name] = np.empty((K, A[0].num_steps, 2), np.float32)
            check(lib.b200mppi_batch_solve(batch._handle, ptr(u[name])))
        assert_same(dict(u=u["loop"]), dict(u=u["twins"]), "direct batch solve after close")
        for k in range(K):
            assert_same(snapshot(A[k]), snapshot(B[k]), "planner %d after the direct solve" % k)


@pytest.mark.parametrize("kind", ["onemap", "barebone", "tdm", "mixed"])
def test_launches(eng, kind):
    """+1 per set_goals / set_obstacles call; a loop that never calls them issues what it issued before, also with an
    obstacle capacity."""
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
    D = TaskDriver(batch, batch.planners)
    for tasks in (False, True):
        with batch.device_loop(max_obstacles=5 if kind == "barebone" else 0) as loop:
            for _ in range(2):
                n = batch.launch_count()
                D.solve(loop)
                assert batch.launch_count() - n == launches_per_solve(kind, num_opt)
                D.step()
                n = batch.launch_count()
                D.shift(loop)
                assert batch.launch_count() - n == 1
                if not tasks:
                    continue
                n = batch.launch_count()
                D.goals(loop, D.base_goals())
                assert batch.launch_count() - n == 1
                if kind == "barebone":
                    n = batch.launch_count()
                    D.obstacles(loop, torch.zeros((2, 5, 3), dtype=torch.float64, device="cuda"))
                    assert batch.launch_count() - n == 1


def test_no_host_wait(eng):
    E = eng
    A = H.twins(functools.partial(bb_setup, E), 3)[0]
    batch = E.MPPI_Batch(A)
    stream = torch.cuda.current_stream()
    batch.set_stream(stream.cuda_stream)
    g = torch.zeros((3, 2), dtype=torch.float64, device="cuda")
    obs = torch.zeros((3, 4, 3), dtype=torch.float64, device="cuda")
    with batch.device_loop(max_obstacles=4) as loop:
        loop.set_goals(g)                               # every kernel loaded before the stream is held up
        loop.set_obstacles(obs)
        torch.cuda.synchronize()
        for call in (lambda: loop.set_goals(g), lambda: loop.set_obstacles(obs)):
            torch.cuda._sleep(int(2e9))                 # about a second of GPU time queued first
            call()
            ev = torch.cuda.Event()
            ev.record(stream)
            assert not ev.query(), "the call waited for the stream"
            torch.cuda.synchronize()


class TaskGraphDriver(GraphDriver):
    """GraphDriver whose step also switches waypoints in torch (a robot within 0.4 of its goal moves on to its next
    waypoint) and sets the goals, and (barebone) sets the swarm's obstacles with counts from a table indexed by the
    step counter; every tensor static, one set per unrolled step."""

    def __init__(self, batch, A, steps, obstacles=False, **kw):
        GraphDriver.__init__(self, batch, A, steps, **kw)
        K, P = self.K, 3
        with torch.cuda.stream(self.stream):
            base = torch.tensor(np.stack([np.asarray(p.params["xgoal"], np.float64)[:2] for p in A]), device="cuda")
            step = torch.tensor([[0.3, 0.2], [0.2, -0.3], [-0.1, 0.4]], dtype=torch.float64, device="cuda")
            self.way = base[:, None, :] + step[None, :P, :]          # (K, P, 2) waypoints
            self.widx = torch.zeros(K, dtype=torch.int64, device="cuda")
            self.G = [torch.zeros((K, 2), dtype=torch.float64, device="cuda") for _ in range(self.unroll)]
            self.obstacles = obstacles
            if obstacles:
                Op = 2 + K - 1
                self.OBS = [torch.zeros((K, Op, 3), dtype=torch.float64, device="cuda") for _ in range(self.unroll)]
                self.CNT = [torch.zeros(K, dtype=torch.int32, device="cuda") for _ in range(self.unroll)]
                rng = np.random.default_rng(5)
                self.cnt_table = torch.tensor(rng.integers(0, Op + 1, (steps, K)), dtype=torch.int32, device="cuda")

    def body(self, loop, j):
        t = self.t.clamp(max=self.steps - 1)           # the step counter before GraphDriver.body advances it
        GraphDriver.body(self, loop, j)
        x = self.x
        K = self.K
        near = torch.linalg.norm(x[:, :2] - self.way[torch.arange(K, device="cuda"), self.widx], dim=1) <= 0.4
        self.widx.copy_((self.widx + near.long()) % self.way.shape[1])
        self.G[j].copy_(self.way[torch.arange(K, device="cuda"), self.widx])
        loop.set_goals(self.G[j])
        if self.obstacles:
            self.OBS[j].copy_(swarm_obstacles(x))
            self.CNT[j].copy_(torch.index_select(self.cnt_table, 0, t)[0])
            loop.set_obstacles(self.OBS[j], self.CNT[j])

    def record(self, n):
        for j in range(n):
            self.calls.append(("solve", self.U[j].cpu().numpy().copy()))
            self.calls.append(("stop", self.M[j].cpu().numpy().copy()))
            self.calls.append(("shift", self.X[j].cpu().numpy().astype(np.float64)))
            self.calls.append(("goals", self.G[j].cpu().numpy().copy()))
            if self.obstacles:
                self.calls.append(("obstacles", self.OBS[j].cpu().numpy().copy(), self.CNT[j].cpu().numpy().copy()))
        self.done += n


@pytest.mark.parametrize("kind", ["det", "tdm", "barebone"])
def test_graph_with_goals_and_obstacles(eng, kind):
    """One eager step, a capture, then replays mixed with eager steps (e r r e r), against the host loop on twins."""
    E = eng
    if kind == "det":
        A, B = onemap_twins(E, "det", K=4)
        batch = E.MPPI_Batch(A)
    elif kind == "tdm":
        A, B, _ = H.twins(functools.partial(H.tdm_trial_setup, E, num_opt=2), 4)
        batch = E.MPPI_StochasticBatch(A)
    else:
        A, B, _ = H.twins(functools.partial(bb_setup, E), 5)
        batch = E.MPPI_Batch(A)
    schedule = "errer"
    total = 1 + len(schedule)
    bb = kind == "barebone"
    D = TaskGraphDriver(batch, A, total, obstacles=bb, stops={3: [1]})
    with batch.device_loop(max_obstacles=2 + len(A) - 1 if bb else 0) as loop:
        per_step = D.eager(loop)
        assert per_step == launches_per_solve("barebone" if bb else "onemap" if kind == "det" else "tdm",
                                              2 if kind == "tdm" else 1) + 3 + (1 if bb else 0)
        assert D.capture(loop) == per_step
        for c in schedule:
            if c == "r":
                D.replay()
            else:
                assert D.eager(loop) == per_step
    assert D.done == total and loop.status[1] == "stopped"
    replay_tasks(D, B, loop)
