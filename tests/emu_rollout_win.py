"""Host emulation of the windowed (TMA-staged) stochastic rollout kernel and its prepare kernel (TEST
INFRASTRUCTURE; tests/emu_core.py).  The kernels' text is lifted from csrc/rollout_win.cu between the
``[emu:... prepare]`` / ``[emu:... win_kernel]`` markers.  What stands in for the hardware (tests/emu_cuda.h): a
CUtensorMap is a plain descriptor (base, dims, pitch, box) and ``tma_load_2d/3d`` copy the box with zero fill outside
the tensor (what CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE does for integer types); mbarrier calls and fences are no-ops (the
copy is done when the call returns); shared-space addresses are offsets into one static buffer; ``__fadd_rd`` is a
round-down add derived from the rounded sum and its exact error (TwoSum); 1024 std::threads stand for the CTA.
Arithmetic helpers as in tests/emu_rollout.py (IEEE meaning; libm for the MUFU approximations)."""
from tests.emu_core import build as _build
from tests.emu_core import cell_index_rzi, drop_fences, extern_shared, region, shared_static

HARNESS = r'''
using namespace b200;
// stage_rollout of csrc/api.cu for MODE_TDM: prepare kernel, window origin, launch geometry of launch_rollout_win.
// shift_x / shift_y move the window away from the robot (cells) to force the global-memory path.
// The fused noise + controls kernel (launch_noise_prepare) next to the two kernels it replaces (sample_noise_kernel
// is restated here as its one-line body: generator g -> (std_v * normal, std_w * normal), tests/emu_noise.py runs the
// real one): states, noise, transposed controls, control costs and the reach statistic must agree bit for bit.
extern "C" int emu_noise_prepare(const uint64_t* states_in, const float* u_cur, int N, int T, float std_v, float std_w,
                                 float lambda, const float* vr, const float* wr, uint64_t* states_out, float* noise_out,
                                 double* noiseT_out, float* ctrl_out, float* reach_out) {
  const int npad = (N + 31) / 32 * 32;
  std::vector<uint64_t> st((size_t)N * T * 2);
  std::memcpy(st.data(), states_in, st.size() * 8);
  std::vector<float> noise((size_t)N * T * 2, 0.0f), ctrl(npad, 0.0f);
  std::vector<double2> noiseT((size_t)T * npad, double2{0, 0});
  float reach[2] = {0.0f, 123.0f};
  emu::launch({(unsigned)(npad / NP_NB), 1, 1}, 256, [&] {
    noise_prepare_kernel(st.data(), reinterpret_cast<float2*>(noise.data()), u_cur, noiseT.data(), ctrl.data(), reach, 0,
                         N, T, npad, std_v, std_w, lambda, std_v * std_v, std_w * std_w, vr[0], vr[1], wr[0], wr[1]);
  });
  if (reach[1] != 0.0f) return 1;                                  // the other slot is cleared for the next launch
  // the two separate kernels
  std::vector<uint64_t> st2((size_t)N * T * 2);
  std::memcpy(st2.data(), states_in, st2.size() * 8);
  std::vector<float> noise2((size_t)N * T * 2, 0.0f), ctrl2(npad, 0.0f);
  std::vector<double2> noiseT2((size_t)T * npad, double2{0, 0});
  for (size_t g = 0; g < (size_t)N * T; ++g) {
    Xoro s{st2[2 * g], st2[2 * g + 1]};
    noise2[2 * g] = fmul(std_v, xoro_normal(s));
    noise2[2 * g + 1] = fmul(std_w, xoro_normal(s));
    st2[2 * g] = s.s0; st2[2 * g + 1] = s.s1;
  }
  float reach2 = 0.0f;
  emu::launch({(unsigned)(npad / 32), 1, 1}, 256, [&] {
    prepare_rollout_kernel(reinterpret_cast<const float2*>(noise2.data()), u_cur, noiseT2.data(), ctrl2.data(), &reach2,
                           N, T, npad, lambda, std_v * std_v, std_w * std_w, vr[0], vr[1], wr[0], wr[1]);
  });
  if (std::memcmp(st.data(), st2.data(), st.size() * 8)) return 2;
  if (std::memcmp(noise.data(), noise2.data(), noise.size() * 4)) return 3;
  if (std::memcmp(noiseT.data(), noiseT2.data(), noiseT.size() * 16)) return 4;
  if (std::memcmp(ctrl.data(), ctrl2.data(), ctrl.size() * 4)) return 5;
  if (reach[0] != reach2) return 6;
  std::memcpy(states_out, st.data(), st.size() * 8);
  std::memcpy(noise_out, noise.data(), noise.size() * 4);
  std::memcpy(noiseT_out, noiseT.data(), noiseT.size() * 16);
  std::memcpy(ctrl_out, ctrl.data(), ctrl.size() * 4);
  *reach_out = reach[0];
  return 0;
}

// the prepare kernel alone on given noise (N, T, 2): its reach statistic max_n sum_t |clip(u_v + e_v)| (round-up adds)
extern "C" float emu_prepare_reach(const float* noise, const float* u_cur, int N, int T, const float* vr, const float* wr) {
  const int npad = (N + 31) / 32 * 32;
  std::vector<double2> noiseT((size_t)T * npad, double2{0, 0});
  std::vector<float> ctrl(npad, 0.0f);
  float reach = 0.0f;
  emu::launch({(unsigned)(npad / 32), 1, 1}, 256, [&] {
    prepare_rollout_kernel(reinterpret_cast<const float2*>(noise), u_cur, noiseT.data(), ctrl.data(), &reach, N, T, npad,
                           1.0f, 1.0f, 1.0f, vr[0], vr[1], wr[0], wr[1]);
  });
  return reach;
}

// cell_from_interval (the division-free decision of the rare path) against the reference's exact sequence:
// out_new[i] = the kernel's result for a[i] (magic-number floors of the interval's ends, then cell_from_interval),
// out_ref[i] = cell_index_exact(a[i], res); differ[i] = 1 when the floors differed (the decision ran)
extern "C" void emu_cell_between(const float* a, int n, float res, int* out_new, int* out_ref, int* differ) {
  const float inv_res = 1.0f / res;
  const float inv_lo = inv_res * (1.0f - 2.4e-7f), inv_hi = inv_res * (1.0f + 2.4e-7f);
  const float MAGIC = 12582912.0f;
  for (int i = 0; i < n; ++i) {
    const float k = __fadd_rd(fmaf(a[i], inv_lo, -1e-30f), MAGIC), k2 = __fadd_rd(fmaf(a[i], inv_hi, 1e-30f), MAGIC);
    differ[i] = __float_as_int(k) != __float_as_int(k2);
    out_new[i] = cell_from_interval(a[i], res, k, k2);
    out_ref[i] = cell_index_exact(a[i], res);
  }
}

// ctas: number of persistent CTAs (0: launch_rollout_win's own rule for a 132-SM device, an H100 SXM).
// dst_blocks: 1 = one map-major (M, N) destination; ws > 1 = the sharded layout, ws separate (ws*M, N/ws) "receive
// buffers" written at the rows of "rank" 1 (fill_cost_dst with direct = true) plus the epoch flags of CostSignal --
// checked here; costs_nm always comes back as the logical (N, M) array.
extern "C" int emu_rollout_win(const float* f, const int* g, const double* ratios, const int8_t* lin, const int8_t* ang,
                               const int8_t* obs, const int8_t* unk, const float* noise, const float* u_cur,
                               float* costs_nm, int shift_x, int shift_y, int* origin_out, float* reach_out, int ctas,
                               int dst_blocks, int unit_override, int sync_passes, int masks01) {
  RolloutWinArgs w{};
  emu::params(w.p, f, g, ratios, g[8]);
  const RolloutParams& p = w.p;
  const int npad = (p.N + 31) / 32 * 32;
  std::vector<double2> noiseT((size_t)(p.T + 1) * npad, double2{0, 0});      // + 1 row: the kernel prefetches unguarded
  std::vector<float> ctrl(npad, std::nanf(""));               // the padding beyond N: never written (cudaMalloc)
  float reach = 0.0f;
  emu::launch({(unsigned)(npad / 32), 1, 1}, 256, [&] {
    prepare_rollout_kernel(reinterpret_cast<const float2*>(noise), u_cur, noiseT.data(), ctrl.data(), &reach, p.N, p.T, npad,
                           p.lambda, p.u_std[0] * p.u_std[0], p.u_std[1] * p.u_std[1], p.vrange[0], p.vrange[1],
                           p.wrange[0], p.wrange[1]);
  });
  const int WW = WIN_WW, WH = (win_smem_layout(WIN_WW, 232, p.T).total <= 232448) ? 232 : 224;
  if (WH != 232) return 1;
  emu::win_place(w, WW, WH, shift_x, shift_y);
  w.npad = npad;
  w.lin_grid = lin; w.ang_grid = ang; w.obstacle = obs; w.unknown = unk;
  w.noiseT = reinterpret_cast<const float*>(noiseT.data()); w.ctrl = ctrl.data(); w.u_cur = u_cur;
  const int ws = dst_blocks < 1 ? 1 : dst_blocks;
  if (p.N % ws) return 4;
  const int n_per = p.N / ws, rank = ws > 1 ? 1 : 0;
  std::vector<std::vector<float>> recv(ws, std::vector<float>((size_t)ws * p.M * n_per, -1.0f));
  std::vector<std::vector<uint32_t>> flags(ws, std::vector<uint32_t>(ws, 0u));
  unsigned counter = 0;
  w.dst.n_per = n_per; w.dst.ld = n_per; w.dst.row0 = rank * p.M;
  for (int d = 0; d < ws; ++d) { w.dst.base[d] = recv[d].data(); w.sig.peer_flags[d] = flags[d].data(); }
  w.sig.ws = ws > 1 ? ws : 0; w.sig.rank = rank; w.sig.counter = &counter; w.sig.epoch = 7u;
  if (origin_out) { origin_out[0] = w.wx0; origin_out[1] = w.wy0; }
  if (reach_out) *reach_out = reach;
  const CUtensorMap t_lin{(const unsigned char*)lin, p.g.grid_cols, p.g.grid_rows, p.M, p.g.grid_pitch, WW, WH};
  const CUtensorMap t_ang{(const unsigned char*)ang, p.g.grid_cols, p.g.grid_rows, p.M, p.g.grid_pitch, WW, WH};
  const CUtensorMap t_obs{(const unsigned char*)obs, p.g.cols, p.g.rows, 1, p.g.mask_pitch, WW, WH};
  const CUtensorMap t_unk{(const unsigned char*)unk, p.g.cols, p.g.rows, 1, p.g.mask_pitch, WW, WH};
  if (ctas <= 0) {                                            // launch_rollout_win (rollout_win.cu)
    const long long total = (long long)p.M * (npad / 32);
    ctas = (int)std::min<long long>(std::max<long long>(total / 8, 1), 132);
  }
  w.unit = ((long long)p.M * (npad / 32) / (32LL * ctas) >= 1) ? 32 : 1;     // launch_rollout_win
  if (unit_override > 0) w.unit = unit_override;
  if (unit_override < 0) w.unit = 0;                         // shares by map (needs ctas >= M)
  w.sync_passes = sync_passes;
  w.masks01 = masks01;
  if (masks01) emu::launch({(unsigned)ctas, 1, 1}, 1024, [&] { rollout_win_kernel<1024, 232, true>(w, t_lin, t_ang, t_obs, t_unk); });
  else emu::launch({(unsigned)ctas, 1, 1}, 1024, [&] { rollout_win_kernel<1024, 232, false>(w, t_lin, t_ang, t_obs, t_unk); });
  for (int n = 0; n < p.N; ++n)
    for (int m = 0; m < p.M; ++m)
      costs_nm[(size_t)n * p.M + m] = recv[n / n_per][((size_t)rank * p.M + m) * n_per + n % n_per];
  if (ws > 1) {
    if (counter != 0) return 5;
    for (int d = 0; d < ws; ++d)
      for (int r = 0; r < ws; ++r)
        if (flags[d][r] != (r == rank ? 7u : 0u)) return 6;           // exactly this rank's flag, in every peer
    for (int d = 0; d < ws; ++d)                                      // rows of the other "ranks" untouched
      for (int r = 0; r < ws; ++r)
        if (r != rank)
          for (size_t i = 0; i < (size_t)p.M * n_per; ++i)
            if (recv[d][(size_t)r * p.M * n_per + i] != -1.0f) return 7;
  }
  return 0;
}

// window-first sampling (stage_rollout, api.cu): the detecting launch (mode 1, WIN_DETECT) or the redo of the flagged
// maps (mode 2, WIN_REDO) of the windowed kernel on the 232-row window, with launch_rollout_win's grid and share unit
// for a 132-SM device (unit 1 for the redo).  costs_mn: the map-major (M, N) costs, in / out (the redo rewrites the
// flagged maps only); esc[M]: the flags, in / out.  ctrl_pad: what ctrl holds beyond N (the planner's cudaMalloc leaves
// it as the allocation held it).  origin_out: wx0, wy0, ww, wh.
extern "C" int emu_rollout_win_esc(const float* f, const int* g, const double* ratios, const int8_t* lin, const int8_t* ang,
                                   const int8_t* obs, const int8_t* unk, const float* noise, const float* u_cur,
                                   float* costs_mn, unsigned char* esc, int mode, float ctrl_pad, int masks01,
                                   int* origin_out) {
  RolloutWinArgs w{};
  emu::params(w.p, f, g, ratios, g[8]);
  const RolloutParams& p = w.p;
  const int npad = (p.N + 31) / 32 * 32;
  std::vector<double2> noiseT((size_t)(p.T + 1) * npad, double2{0, 0});      // memset at create
  std::vector<float> ctrl(npad, ctrl_pad);
  emu::launch({(unsigned)(npad / 32), 1, 1}, 256, [&] {
    prepare_rollout_kernel(reinterpret_cast<const float2*>(noise), u_cur, noiseT.data(), ctrl.data(), nullptr, p.N, p.T,
                           npad, p.lambda, p.u_std[0] * p.u_std[0], p.u_std[1] * p.u_std[1], p.vrange[0], p.vrange[1],
                           p.wrange[0], p.wrange[1]);
  });
  const int WW = WIN_WW, WH = 232;
  if (win_smem_layout(WW, WH, p.T).total > 232448) return 1;
  emu::win_place(w, WW, WH);
  w.npad = npad;
  w.lin_grid = lin; w.ang_grid = ang; w.obstacle = obs; w.unknown = unk;
  w.noiseT = reinterpret_cast<const float*>(noiseT.data()); w.ctrl = ctrl.data(); w.u_cur = u_cur;
  w.dst.n_per = p.N; w.dst.ld = p.N; w.dst.row0 = 0; w.dst.base[0] = costs_mn;
  w.esc = esc; w.redo = mode == 2;
  w.masks01 = masks01;
  if (origin_out) { origin_out[0] = w.wx0; origin_out[1] = w.wy0; origin_out[2] = w.ww; origin_out[3] = w.wh; }
  const CUtensorMap t_lin{(const unsigned char*)lin, p.g.grid_cols, p.g.grid_rows, p.M, p.g.grid_pitch, WW, WH};
  const CUtensorMap t_ang{(const unsigned char*)ang, p.g.grid_cols, p.g.grid_rows, p.M, p.g.grid_pitch, WW, WH};
  const CUtensorMap t_obs{(const unsigned char*)obs, p.g.cols, p.g.rows, 1, p.g.mask_pitch, WW, WH};
  const CUtensorMap t_unk{(const unsigned char*)unk, p.g.cols, p.g.rows, 1, p.g.mask_pitch, WW, WH};
  const long long total = (long long)p.M * (npad / 32);        // launch_rollout_win
  const int ctas = (int)std::min<long long>(std::max<long long>(total / 8, 1), 132);
  w.unit = (total / (32LL * ctas) >= 4) ? 32 : (ctas >= p.M ? 0 : 1);
  if (w.redo) w.unit = 1;
  w.sync_passes = 0;
  auto run = [&](auto kern) { emu::launch({(unsigned)ctas, 1, 1}, 1024, [&] { kern(w, t_lin, t_ang, t_obs, t_unk); }); };
  if (mode == 1 && masks01) run(rollout_win_kernel<1024, 232, true, WIN_DETECT>);
  else if (mode == 1) run(rollout_win_kernel<1024, 232, false, WIN_DETECT>);
  else if (mode == 2 && masks01) run(rollout_win_kernel<1024, 232, true, WIN_REDO>);
  else if (mode == 2) run(rollout_win_kernel<1024, 232, false, WIN_REDO>);
  else return 2;
  return 0;
}
'''


def kernels(prep=(), win=()):
    """The prepare kernels (``prepare``, ``noise_prepare``, then the regions named in ``prep``) and the windowed kernel
    (``win_kernel``, then those named in ``win``) of csrc/rollout_win.cu, with the structs and helpers they use."""
    p = "".join(region("rollout_win.cu", r) for r in ("prepare", "noise_prepare") + tuple(prep))
    k = "".join(region("rollout_win.cu", r) for r in ("win_kernel",) + tuple(win))
    return [region("common.cuh", "params"), cell_index_rzi(region("common.cuh", "cell_index")),
            region("kernels.h", "cost_dst"), region("kernels.h", "win_args"), region("kernels.h", "noise_prep_desc"),
            region("common.cuh", "xoro"), region("common.cuh", "normal"), shared_static(p, 2),
            extern_shared(drop_fences(k, 3), 1)]


# the escape flag's store as it was before padding lanes were excluded: any NaN cost of the map's chunks flags it
FLAG_ANY_LANE = ("MODE == WIN_DETECT && live && cost != cost", "MODE == WIN_DETECT && cost != cost")


def build(out_dir, extra="", flag_any_lane=False):
    """``flag_any_lane``: compile the kernel with the flag store of FLAG_ANY_LANE[1] (padding lanes flag too)."""
    parts = kernels()
    if flag_any_lane:
        assert parts[-1].count(FLAG_ANY_LANE[0]) == 1
        parts[-1] = parts[-1].replace(*FLAG_ANY_LANE)
    return _build(out_dir, "rollout_win_emu" + ("_any_lane" if flag_any_lane else ""), parts, HARNESS + extra)
