"""The mode-dispatching one-map rollout of mixed batches (rollout_batch_mixed_kernel, rollout.cu's ``[emu:begin
rollout_batch]`` region) compiled for the host: ONE launch over interleaved det-dynamics, speed-map and inactive
descriptors with different maps, start poses and goals equals, planner by planner, the batched rollout of its own mode
(rollout_batch_kernel<1> / <2>, itself held to single launches and the exact oracle elsewhere), bit for bit, and leaves
an inactive planner's costs untouched."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_batch
from tests.test_batch_emulated_cpu import p, ptrs, rollout_inputs

MIXED_HARNESS = r'''
// K planners of modes[i] (1 or 2) in ONE launch of the mode-dispatching kernel, gated by active (null: all run)
extern "C" void emu_rollout_mixed(int K, const int* modes, const int* active, const float* f, const int* g,
                                  const double* ratios, const int8_t** lin, const int8_t** ang, const int8_t** obs,
                                  const int8_t** unk, const int8_t** risk, const float** noise, const float** u_cur,
                                  float** costs) {
  std::vector<RolloutArgs> d(K);
  for (int i = 0; i < K; ++i) {
    RolloutArgs a{};
    emu::params(a.p, f + 23 * i, g + 9 * i, ratios + 2 * i, 1);
    a.mode = modes[i]; a.lin_grid = lin[i]; a.ang_grid = ang[i]; a.obstacle = obs[i]; a.unknown = unk[i];
    a.risk = risk[i]; a.noise = noise[i]; a.u_cur = u_cur[i]; a.costs = costs[i];
    d[i] = a;
  }
  const unsigned gx = (unsigned)((d[0].p.N + 127) / 128);
  emu::launch({gx, (unsigned)K, 1}, 128, [&] { rollout_batch_mixed_kernel(d.data(), active); });
}
'''

MODES = [1, 2, 2, 1, 2, 1]
ACTIVE = [1, 1, 0, 1, 1, 0]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return emu_batch.build_rollout(str(tmp_path_factory.mktemp("emu_mixed_rollout")), MIXED_HARNESS)


def args(ins, key):
    return ptrs([x[key] for x in ins])


def single_mode(lib, x, mode, N):
    """Costs of one planner through the batched rollout of its own mode (a batch of one)."""
    c = np.full(N, np.nan, np.float32)
    lib.emu_rollout(1, 1, mode, p(x["f"]), p(x["g"]), p(x["ratios"]), *[ptrs([x[k]]) for k in (
        "lin", "ang", "obs", "unk", "risk", "noise", "u")], ptrs([c]), ptrs([x["ob"]]), p(np.zeros(1, np.int32)))
    return c


@pytest.mark.parametrize("gated", [False, True])
def test_mixed_equals_per_mode(lib, gated):
    N, T = 150, 12
    ins = [rollout_inputs(m, s, N, T) for s, m in enumerate(MODES)]
    for s, x in enumerate(ins):                     # every planner gets a risk map: only mode 2 reads it
        if x["risk"] is None:
            x["risk"] = np.random.default_rng(50 + s).integers(0, 101, x["obs"].shape).astype(np.int8)
    K = len(MODES)
    costs = [np.full(N, np.nan, np.float32) for _ in range(K)]
    active = np.array(ACTIVE, np.int32) if gated else None
    lib.emu_rollout_mixed(K, p(np.array(MODES, np.int32)), p(active) if gated else None,
                          p(np.concatenate([x["f"] for x in ins])), p(np.concatenate([x["g"] for x in ins])),
                          p(np.concatenate([x["ratios"] for x in ins])),
                          *[args(ins, k) for k in ("lin", "ang", "obs", "unk", "risk", "noise", "u")], ptrs(costs))
    for i, (x, m) in enumerate(zip(ins, MODES)):
        if gated and not ACTIVE[i]:
            assert np.isnan(costs[i]).all(), "inactive planner %d was written" % i
            continue
        want = single_mode(lib, x, m, N)
        assert np.isfinite(want).all()
        assert costs[i].tobytes() == want.tobytes(), "planner %d (mode %d)" % (i, m)
    # the other mode gives other costs: the dispatch, not the inputs, decides
    assert single_mode(lib, ins[0], 2, N).tobytes() != costs[0].tobytes()
