"""A device loop's solve clock (csrc/reduce.cu, ``[emu:... loop_clock]``, run by the export launch that ends each loop
solve) emulated on the host, bit for bit: after the export that ends solve s, for s = 0 .. 7 and num_opt 1, 2 and 3,
over one-map, stochastic, mixed and shared-pair (fewer sampler sets than planners) layouts,
  - each kind's current sampler set is its staged set of parity (s + 1) & 1, byte for byte;
  - every stochastic planner's noise and box descriptor slot is the one its by-value iteration index
    (s + 1) * num_opt + k selects for every iteration k (slot ^ (k & 1) == staged slot ^ (iter & 1)), every other byte of
    those descriptors unchanged;
  - the clock reads s + 1.
A null clock leaves everything untouched, and at 2^31 - 1 solves the clock stops and raises its flag instead of
wrapping."""
import numpy as np
import pytest

from tests.emu_core import build as _build
from tests.emu_core import region

HARNESS = r'''
#include <cstddef>
using namespace b200;
// set_par: per kind, parity 0 then parity 1 (G[kind] sets each); nprep, box: K2 descriptors each
extern "C" void emu_clock(int* clock, void* cur0, void* cur1, const void* par00, const void* par01, const void* par10,
                          const void* par11, int G0, int G1, void* nprep, void* box, const int* slot0, int K2,
                          int num_opt) {
  LoopClock a{};
  a.clock = clock;
  a.set_cur[0] = reinterpret_cast<SampleGridsV2Args*>(cur0);
  a.set_cur[1] = reinterpret_cast<SampleGridsV2Args*>(cur1);
  a.set_par[0][0] = reinterpret_cast<const SampleGridsV2Args*>(par00);
  a.set_par[0][1] = reinterpret_cast<const SampleGridsV2Args*>(par01);
  a.set_par[1][0] = reinterpret_cast<const SampleGridsV2Args*>(par10);
  a.set_par[1][1] = reinterpret_cast<const SampleGridsV2Args*>(par11);
  a.G[0] = G0; a.G[1] = G1;
  a.nprep = reinterpret_cast<NoisePrepDesc*>(nprep);
  a.box = reinterpret_cast<SampleBoxDesc*>(box);
  a.slot0 = slot0;
  a.K2 = K2; a.num_opt = num_opt;
  emu::launch({1, 1, 1}, 128, [&] { loop_clock_body(a); });      // CTA 0 of the export launch
}
// 0: sizeof SampleGridsV2Args, 1: sizeof NoisePrepDesc, 2: its slot's offset, 3: sizeof SampleBoxDesc, 4: its slot's
extern "C" int emu_layout(int what) {
  const size_t v[] = {sizeof(SampleGridsV2Args), sizeof(NoisePrepDesc), offsetof(NoisePrepDesc, slot),
                      sizeof(SampleBoxDesc), offsetof(SampleBoxDesc, slot)};
  return (int)v[what];
}
'''


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return _build(str(tmp_path_factory.mktemp("loop_clock_emu")), "loop_clock_emu",
                  [region("kernels.h", "sampler_args"), region("kernels.h", "box_desc"),
                   region("kernels.h", "noise_prep_desc"), region("kernels.h", "loop_clock_args"),
                   region("reduce.cu", "loop_clock")], HARNESS)


class Layout(object):
    """A loop buffer's clock sections: G[kind] staged sets per parity and a current set per kind (random bytes, staged
    as trial_call_stage does: current = parity 0), K2 noise and box descriptors (random bytes, staged slots 0 / 1)."""

    def __init__(self, emu, G0, G1, K2, num_opt, seed):
        rng = np.random.default_rng(seed)
        self.emu = emu
        sz, self.np_sz, self.np_slot, self.bx_sz, self.bx_slot = (emu.emu_layout(i) for i in range(5))
        self.G, self.K2, self.num_opt = (G0, G1), K2, num_opt
        self.par = [[rng.integers(0, 256, max(G, 1) * sz, dtype=np.uint8) for _ in range(2)] for G in self.G]
        self.cur = [self.par[k][0].copy() for k in range(2)]
        self.slot0 = rng.integers(0, 2, 2 * K2).astype(np.int32)
        self.nprep = rng.integers(0, 256, max(K2, 1) * self.np_sz, dtype=np.uint8)
        self.box = rng.integers(0, 256, max(K2, 1) * self.bx_sz, dtype=np.uint8)
        for r in range(K2):
            self.slot(self.nprep, self.np_sz, self.np_slot)[r] = self.slot0[r]
            self.slot(self.box, self.bx_sz, self.bx_slot)[r] = self.slot0[K2 + r]
        self.clock = np.zeros(2, dtype=np.int32)

    def slot(self, buf, size, off):
        """The int32 slot field of each of the K2 descriptors in buf (a writable view)."""
        return np.ndarray((self.K2,), dtype=np.int32, buffer=buf, offset=off, strides=(size,))

    def export(self, clock=True):
        e = self.emu
        d = lambda a: a.ctypes.data                                                    # noqa: E731
        e.emu_clock(d(self.clock) if clock else None, d(self.cur[0]), d(self.cur[1]), d(self.par[0][0]),
                    d(self.par[0][1]), d(self.par[1][0]), d(self.par[1][1]), self.G[0], self.G[1], d(self.nprep),
                    d(self.box), d(self.slot0), self.K2, self.num_opt)

    def snapshot(self):
        return [a.copy() for a in (self.cur[0], self.cur[1], self.nprep, self.box, self.clock, self.par[0][0],
                                   self.par[0][1], self.par[1][0], self.par[1][1], self.slot0)]


LAYOUTS = {
    "onemap": (5, 0, 0),          # G0 one-map sets, G1 stochastic sets, K2 stochastic planners
    "stochastic": (0, 4, 4),
    "mixed": (3, 2, 2),
    "grouped": (2, 2, 5),         # shared pairs: five stochastic planners over two sets, one-map planners over two
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("num_opt", [1, 2, 3])
def test_clock_prepares_the_next_solve(emu, layout, num_opt):
    G0, G1, K2 = LAYOUTS[layout]
    L = Layout(emu, G0, G1, K2, num_opt, seed=num_opt * 10 + len(layout))
    nprep0, box0 = L.nprep.copy(), L.box.copy()
    sz = emu.emu_layout(0)
    for s in range(8):
        assert L.clock.tolist() == [s, 0]
        L.export()
        assert L.clock.tolist() == [s + 1, 0]
        for k in range(2):
            n = L.G[k] * sz
            assert L.cur[k][:n].tobytes() == L.par[k][(s + 1) & 1][:n].tobytes(), "kind %d after solve %d" % (k, s)
        for buf, ref, size, off, base in ((L.nprep, nprep0, L.np_sz, L.np_slot, 0),
                                          (L.box, box0, L.bx_sz, L.bx_slot, K2)):
            slots = L.slot(buf, size, off)
            for r in range(K2):
                for k in range(num_opt):
                    it = (s + 1) * num_opt + k                  # the by-value iteration index of solve s + 1
                    assert slots[r] ^ (k & 1) == L.slot0[base + r] ^ (it & 1), (s, r, k)
            got, want = buf.copy(), ref.copy()
            L.slot(got, size, off)[:] = 0
            L.slot(want, size, off)[:] = 0
            assert got.tobytes() == want.tobytes(), "a descriptor byte besides its slot changed"


def test_null_clock_leaves_everything(emu):
    L = Layout(emu, *LAYOUTS["mixed"], num_opt=1, seed=7)
    L.export()                                                  # the current sets now differ from parity 0's
    before = L.snapshot()
    L.export(clock=False)
    for a, b in zip(before, L.snapshot()):
        assert a.tobytes() == b.tobytes()


def test_clock_stops_at_the_solve_limit(emu):
    L = Layout(emu, *LAYOUTS["stochastic"], num_opt=1, seed=8)
    L.clock[0] = 2 ** 31 - 2
    L.export()
    assert L.clock.tolist() == [2 ** 31 - 1, 0]
    L.export()
    assert L.clock.tolist() == [2 ** 31 - 1, 1]
