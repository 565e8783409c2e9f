"""Host emulation of the control-update kernels (TEST INFRASTRUCTURE; tests/emu_core.py): the text of
update_partial_kernel / merge_partials / update_rank_kernel / update_apply_kernel (csrc/reduce.cu between the
``[emu:... update]`` markers) compiled with g++, one std::thread per CUDA thread.  Float arithmetic follows the
kernel's own order; ``exp`` is libm's instead of CUDA's (both within an ulp), so results are compared within the
bounds of tests/reduce_bounds.py."""
from tests.emu_core import build as _build
from tests.emu_core import region, shared_static

HARNESS = r'''
using namespace b200;
static UpdateArgs make(const float* costs, const float* noise, float* w_raw, float* cta_partials, float* rank_partial,
                       float* u_cur, float* weights, int N, int T, float lambda, const float* vr, const float* wr) {
  UpdateArgs a{};
  a.costs = costs; a.noise = noise; a.w_raw = w_raw; a.cta_partials = cta_partials; a.rank_partial = rank_partial;
  a.u_cur = u_cur; a.weights = weights; a.N = N; a.T = T; a.lambda = lambda;
  a.vrange[0] = vr[0]; a.vrange[1] = vr[1]; a.wrange[0] = wr[0]; a.wrange[1] = wr[1];
  emu::update_geometry(N, a.num_ctas, a.rows_per_cta);
  return a;
}
static const float kZero2[2] = {0, 0};

extern "C" int emu_update_num_ctas(int N) {
  return make(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, N, 1, 1.0f, kZero2, kZero2).num_ctas;
}

// launch_update_partial with UPD_TAIL_RANK: CTA partials + (last CTA) this rank's partial (2T+2 floats)
extern "C" void emu_update_partial(const float* costs, const float* noise, float* w_raw, float* cta_partials,
                                   float* rank_partial, int N, int T, float lambda) {
  const UpdateArgs a = make(costs, noise, w_raw, cta_partials, rank_partial, nullptr, nullptr, N, T, lambda, kZero2, kZero2);
  unsigned counter = 0;
  UpdateTail tl{};
  tl.counter = &counter; tl.mode = UPD_TAIL_RANK;
  emu::launch({(unsigned)a.num_ctas, 1, 1}, UPD_THREADS, [&] { update_partial_kernel(a, tl); });
}

// UPD_TAIL_APPLY: the whole one-rank update in ONE launch (partials, merge and apply by the last CTA)
extern "C" int emu_update_one_rank(const float* costs, const float* noise, float* w_raw, float* cta_partials,
                                   float* rank_partial, float* u_cur, float* weights, int N, int T, float lambda,
                                   const float* vr, const float* wr) {
  const UpdateArgs a = make(costs, noise, w_raw, cta_partials, rank_partial, u_cur, weights, N, T, lambda, vr, wr);
  unsigned counter = 0;
  UpdateTail tl{};
  tl.counter = &counter; tl.mode = UPD_TAIL_APPLY;
  emu::launch({(unsigned)a.num_ctas, 1, 1}, UPD_THREADS, [&] { update_partial_kernel(a, tl); });
  return counter == 0 ? 0 : 1;                    // the ticket counter is left at zero for the next launch
}

// UPD_TAIL_BCAST: the rank partial goes into slot `rank` of every peer's gather buffer (ws, 2T+2), flags raised
extern "C" int emu_update_bcast(const float* costs, const float* noise, float* w_raw, float* cta_partials,
                                float* rank_partial, int N, int T, float lambda, int ws, int rank, float* gather_all,
                                uint32_t* flags_all, uint32_t epoch) {
  const UpdateArgs a = make(costs, noise, w_raw, cta_partials, rank_partial, nullptr, nullptr, N, T, lambda, kZero2, kZero2);
  unsigned counter = 0;
  UpdateTail tl{};
  tl.counter = &counter; tl.mode = UPD_TAIL_BCAST; tl.ws = ws; tl.rank = rank; tl.epoch = epoch;
  for (int q = 0; q < ws; ++q) {
    tl.peer_gather[q] = gather_all + (size_t)q * ws * (2 * T + 2);
    tl.peer_flags[q] = flags_all + (size_t)q * ws;
  }
  emu::launch({(unsigned)a.num_ctas, 1, 1}, UPD_THREADS, [&] { update_partial_kernel(a, tl); });
  return counter == 0 ? 0 : 1;
}

// launch_update_finish: combine `count` gathered rank partials into u_cur and this rank's normalised weights
extern "C" void emu_update_finish(const float* gathered, int count, const float* w_raw, const float* cta_partials,
                                  float* u_cur, float* weights, int N, int T, float lambda, const float* vr,
                                  const float* wr) {
  const UpdateArgs a = make(nullptr, nullptr, const_cast<float*>(w_raw), const_cast<float*>(cta_partials), nullptr, u_cur,
                            weights, N, T, lambda, vr, wr);
  int ctas = a.num_ctas < 32 ? a.num_ctas : 32;
  if (ctas < 1) ctas = 1;
  emu::launch({(unsigned)ctas, 1, 1}, UPD_THREADS, [&] { update_apply_kernel(a, gathered, count, FlagWait{}); });
}
'''


def kernels(*more):
    """The update kernels' text (``update`` region, then the named regions of csrc/reduce.cu) with their argument
    structs and warp reductions."""
    return [region("kernels.h", "cost_dst"), region("kernels.h", "update_args"), region("kernels.h", "update_tail"),
            region("kernels.h", "update_desc"), region("common.cuh", "warp_min"), region("common.cuh", "warp_sum"),
            shared_static("".join(region("reduce.cu", r) for r in ("update",) + more), 10)]


def build(out_dir, extra=""):
    return _build(out_dir, "update_emu", kernels(), HARNESS + extra)
