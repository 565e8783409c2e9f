"""Device loops under CUDA graph capture on the GPU (run with ``-m gpu``): a loop step -- solve into a static ``out``,
the torch plant, a device-computed ``stop`` and ``shift_and_update`` -- is captured with ``torch.cuda.graph`` on the
batch's stream after one eager step and replayed.  Kicks off the map and stops come from tables indexed by a step
counter on the device, so every replay is a different step.  After each step the controls, stop mask and pose are read
back, and the host loop replayed on twins (tests/test_gpu_device_loop.py ``replay``) must give every solve's u, and
after close every planner's snapshot, params['x0'], solves, shifts and status, bit for bit.  Covered: det, speed-map,
use_tdm (num_opt 1 and 2), barebone with obstacles, MPPI_MixedBatch, share_tdms with members that stop at different
steps, maps of mixed geometry, a graph of 3 unrolled steps replayed to an odd total, eager steps interleaved with
replays, the launch count of captures and replays, and the refusals: close() while the batch's stream captures (the
loop stays usable), a call while torch captures on another stream, and a wait on a stream outside the capture."""
import functools

import numpy as np
import pytest

from tests import gpu_harness as H
from tests import test_gpu_mixed_geometry_trials as MG
from tests import test_gpu_shared_tdm as SH
from tests.gpu_harness import assert_same, eng, quiet  # noqa: F401
from tests.scenarios import make_scenario
from tests.test_gpu_barebone_trials import bb_setup
from tests.test_gpu_device_loop import Driver, onemap_twins, replay, solve_one
from tests.test_gpu_mixed_batch import planner as mixed_planner

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


class GraphDriver(Driver):
    """A device loop whose steps run eagerly ("e") or as replays ("r") of one captured graph of ``unroll`` steps, each
    step the body of test_gpu_device_loop.run with every tensor static: kick[t] (K, 2) is added to the poses after the
    plant step and stop[t] (K,) is the stop mask, t the step counter on the device."""

    def __init__(self, batch, A, steps, dtype=torch.float64, strided=False, kick=None, stops=None, unroll=1):
        self.stream = torch.cuda.Stream()
        with torch.cuda.stream(self.stream):
            Driver.__init__(self, batch, A, dtype, strided)     # the batch's stream: the capturing one
            K, dev = self.K, "cuda"
            self.kick = torch.zeros((steps, K, 2), dtype=torch.float64, device=dev)
            self.stops = torch.zeros((steps, K), dtype=torch.bool, device=dev)
            for t, d in (kick or {}).items():
                for k, v in d.items():
                    self.kick[t, k] = torch.tensor(v, dtype=torch.float64)
            for t, ks in (stops or {}).items():
                self.stops[t, list(ks)] = True
            self.t = torch.zeros(1, dtype=torch.int64, device=dev)
            self.steps, self.unroll = steps, unroll
            self.U = [torch.zeros((K, self.T, 2), dtype=torch.float32, device=dev) for _ in range(unroll)]
            self.M = [torch.zeros(K, dtype=torch.bool, device=dev) for _ in range(unroll)]
            if strided:                                  # x[:, :3] of a (K, 4) tensor: rows 4 elements apart
                self.X = [torch.zeros((K, 4), dtype=dtype, device=dev)[:, :3] for _ in range(unroll)]
            else:
                self.X = [torch.zeros((K, 3), dtype=dtype, device=dev) for _ in range(unroll)]
        self.graph = None
        self.done = 0                                    # steps run

    @property
    def T(self):
        return self.batch.num_steps

    def body(self, loop, j):
        u, mask, xin = self.U[j], self.M[j], self.X[j]
        loop.solve(out=u)
        v = torch.nan_to_num(u[:, 0, 0].double())
        w = torch.nan_to_num(u[:, 0, 1].double())
        x = self.x
        th = x[:, 2]
        t = self.t.clamp(max=self.steps - 1)
        nx = torch.stack([x[:, 0] + self.dt * torch.cos(th) * v, x[:, 1] + self.dt * torch.sin(th) * v,
                          th + self.dt * w], dim=1)
        nx[:, :2] += torch.index_select(self.kick, 0, t)[0]
        x.copy_(nx)
        mask.copy_(torch.index_select(self.stops, 0, t)[0])
        loop.stop(mask)
        xin.copy_(x.to(self.dtype))
        loop.shift_and_update(xin)
        self.t += 1

    def record(self, n):
        """The calls of the last n steps (buffers 0 .. n-1), as Driver records them."""
        for j in range(n):
            self.calls.append(("solve", self.U[j].cpu().numpy().copy()))
            self.calls.append(("stop", self.M[j].cpu().numpy().copy()))
            self.calls.append(("shift", self.X[j].cpu().numpy().astype(np.float64)))
        self.done += n

    def eager(self, loop):
        with torch.cuda.stream(self.stream):
            n = self.batch.launch_count()
            self.body(loop, 0)
            per_step = self.batch.launch_count() - n
            self.record(1)
        return per_step

    def capture(self, loop):
        self.graph = torch.cuda.CUDAGraph()
        n = self.batch.launch_count()
        with torch.cuda.graph(self.graph, stream=self.stream):
            for j in range(self.unroll):
                self.body(loop, j)
        return self.batch.launch_count() - n

    def replay(self):
        with torch.cuda.stream(self.stream):
            n = self.batch.launch_count()
            self.graph.replay()
            assert self.batch.launch_count() == n, "a replay issued launches from the host"
            self.record(self.unroll)


def graph_run(batch, A, steps, schedule=None, unroll=1, **kw):
    """One eager step, a capture of ``unroll`` steps, then ``schedule`` ("e": an eager step, "r": a replay; default:
    replays up to ``steps``).  Returns (driver, loop)."""
    if schedule is None:
        schedule = "r" * -(-(steps - 1) // unroll)
    total = 1 + sum(unroll if c == "r" else 1 for c in schedule)
    D = GraphDriver(batch, A, total, unroll=unroll, **kw)
    with batch.device_loop() as loop:
        per_step = D.eager(loop)
        assert D.capture(loop) == unroll * per_step, "a capture issues what its steps issue eagerly"
        for c in schedule:
            if c == "r":
                D.replay()
            else:
                assert D.eager(loop) == per_step
    assert D.done == total
    return D, loop


@pytest.mark.parametrize("mode", ["det", "spd"])
def test_onemap_graph(eng, mode):
    E = eng
    A, B = onemap_twins(E, mode)
    D, loop = graph_run(E.MPPI_Batch(A), A, 8, kick={3: {4: (100.0, 0.0)}}, stops={5: [1]})
    assert loop.status[4] == "left_map" and loop.status[1] == "stopped", loop.status
    replay(D, B, loop)


@pytest.mark.parametrize("num_opt", [1, 2])
def test_stochastic_graph(eng, num_opt):
    E = eng
    A, B, _ = H.twins(functools.partial(H.tdm_trial_setup, E, num_opt=num_opt), 5)
    D, loop = graph_run(E.MPPI_StochasticBatch(A), A, 7, dtype=torch.float32, kick={2: {4: (0.0, -100.0)}},
                        stops={3: [0]})
    assert loop.status[4] == "left_map" and loop.status[0] == "stopped", loop.status
    replay(D, B, loop)


def test_barebone_graph_with_obstacles(eng):
    E = eng
    A, B, _ = H.twins(functools.partial(bb_setup, E), 6)
    D, loop = graph_run(E.MPPI_Batch(A), A, 8, strided=True, kick={2: {0: (1e9, 0.0)}}, stops={4: [2, 5]})
    assert loop.status[0] == "running", "barebone planners have no map to leave"
    replay(D, B, loop)


def test_mixed_batch_graph(eng):
    E = eng
    order = [("tdm", 0), ("det", 2), ("spd", 4), ("tdm", 2), ("det", 0)]
    with quiet():
        A = [mixed_planner(E, kind, j)[0] for kind, j in order]
        B = [mixed_planner(E, kind, j)[0] for kind, j in order]
    D, loop = graph_run(E.MPPI_MixedBatch(A), A, 6, kick={2: {1: (-100.0, 0.0)}}, stops={4: [3]})
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
    D, loop = graph_run(batch, A, 7, stops={1: [0], 3: [2], 5: [4]})
    # as test_gpu_device_loop: each planner against its private twin, the shared pair against the copy of its
    # longest-running member (planners 0 .. K-2 share it; 1 and 3 run to the end)
    saved = {k: SH.pair_state(A[k]) for k in range(K)}
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
    assert loop.solves.tolist() == [2, 7, 4, 7, 6], loop.solves


def test_mixed_geometry_graph(eng):
    E = eng
    A, B = MG.build(E, "tdm", MG.SPECS), MG.build(E, "tdm", MG.SPECS)
    D, loop = graph_run(E.MPPI_StochasticBatch(A), A, 5)
    replay(D, B, loop)
    A, B = MG.build(E, "det", MG.SPECS), MG.build(E, "det", MG.SPECS)
    D, loop = graph_run(E.MPPI_Batch(A), A, 5)
    replay(D, B, loop)


@pytest.mark.parametrize("kind", ["det", "tdm"])
def test_unrolled_graph_and_interleaved_eager_steps(eng, kind):
    """A graph of 3 steps replayed twice (7 steps with the warm-up: an odd total), and eager steps between replays
    (eager, replay x2, eager, replay), against the host loop; use_tdm with num_opt 2, so a solve toggles the reach slot
    twice and the sampler parity once."""
    E = eng
    for unroll, schedule in ((3, "rr"), (1, "errer")):
        if kind == "det":
            A, B = onemap_twins(E, "det", K=4)
            batch = E.MPPI_Batch(A)
        else:
            A, B, _ = H.twins(functools.partial(H.tdm_trial_setup, E, num_opt=2), 4)
            batch = E.MPPI_StochasticBatch(A)
        D, loop = graph_run(batch, A, 0, schedule=schedule, unroll=unroll, stops={4: [1]})
        assert loop.solves.tolist()[1] == 5 and loop.status[1] == "stopped", (loop.solves, loop.status)
        replay(D, B, loop)


def test_refusals_during_capture(eng):
    E = eng
    A, B = onemap_twins(E, "det", K=3)
    batch = E.MPPI_Batch(A)
    D = GraphDriver(batch, A, 4)
    other = torch.cuda.Stream()

    class OnStream(object):
        """D.U[0] whose array interface names ``other``."""
        def __init__(self, t):
            self.__cuda_array_interface__ = dict(t.__cuda_array_interface__, version=3, stream=other.cuda_stream)

    with batch.device_loop() as loop:
        D.eager(loop)
        # torch captures on a stream other than the loop's: every call is refused before anything is enqueued
        g = torch.cuda.CUDAGraph()
        n = batch.launch_count()
        with torch.cuda.graph(g, stream=other):
            torch.zeros(1, device="cuda").add_(1)
            for call in (lambda: loop.solve(out=D.U[0]), lambda: loop.shift_and_update(D.X[0]),
                         lambda: loop.stop(D.M[0]), loop.close):
                with pytest.raises(ValueError, match="capturing"):
                    call()
        assert batch.launch_count() == n and batch._loop is loop
        # the loop's own stream captures: close and a wait on a stream outside the capture are refused
        D.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(D.graph, stream=D.stream):
            with pytest.raises(RuntimeError, match="capturing"):       # B200MPPIError
                loop.close()
            with pytest.raises(RuntimeError, match="not part of that capture"):
                loop.solve(out=OnStream(D.U[0]))
            assert batch.launch_count() == n
            D.body(loop, 0)
        assert batch._loop is loop
        D.replay()
        D.eager(loop)
        D.replay()
    assert batch._loop is None and loop.solves.tolist() == [4, 4, 4]
    replay(D, B, loop)
