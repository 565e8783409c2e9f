// sample.cu -- traction-map sampling from the PMF grid.
// Reference: TDM_Numba.sample_grids + sample_grids_numba (mppi_numba/terrain.py:610-694) and the
// generator set-up numba.cuda.random.create_xoroshiro128p_states (numba/cuda/random.py:226-264).
//
// Bit-exact contract: generator  tid_x*(ty*M) + m*ty + tid_y  walks its ceil(rows/tx) x ceil(cols/ty)
// tile row-major and draws ONE uniform per cell; q = int8(ceil(f64(u_f32)*100*alpha)); the first bin
// whose cumulative PMF reaches q is written as int8(100*(v_bin-lo)/(hi-lo)) (float64, truncated);
// if no bin reaches q the cell keeps its previous content.  The table of cumulative PMFs is built
// once per set_pmf (cell-major, so one cell's bins are contiguous) instead of re-summing B strided
// int8 loads per cell per map as the reference does.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>
#include "kernels.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------
// (B, rows, cols) PMF -> (rows, cols, bpad) running sums, clamped to int8 (comparisons against an
// int8 threshold are unaffected by the clamp); bins >= B repeat the last sum.
// [emu:begin build_cum]   (tests/emu_setter.py compiles the marked kernels for the host)
__global__ void build_cum_kernel(const int8_t* __restrict__ pmf, int8_t* __restrict__ cum, int B, int bpad,
                                 int rows, int cols) {
  const int cell = blockIdx.x * blockDim.x + threadIdx.x;
  if (cell >= rows * cols) return;
  int acc = 0;
  for (int b = 0; b < bpad; ++b) {
    if (b < B) acc += pmf[(size_t)b * rows * cols + cell];
    cum[(size_t)cell * bpad + b] = (int8_t)max(-128, min(127, acc));
  }
}

// [emu:end build_cum]
void launch_build_cum(const int8_t* pmf, int8_t* cum, int num_bins, int bpad, int rows, int cols,
                      cudaStream_t st) {
  const int cells = rows * cols;
  build_cum_kernel<<<(cells + 255) / 256, 256, 0, st>>>(pmf, cum, num_bins, bpad, rows, cols);
}

// ---------------------------------------------------------------------------------------------
// Device version of the PMF preprocessing of set_TDM_from_PMF_grid for the one-map planner modes
// (terrain.py:408-495) fused with cropping + zero-traction padding (terrain.py:511-543): one thread per
// PADDED cell.  The float64 arithmetic repeats numpy's operation order (0.01*cumsum, (0.01*p)*v, sequential
// cumsum, +1e-6 in the denominator) with explicitly rounded, uncontracted operations, so the chosen bin is
// the one the reference's host code chooses.
//   mode 1 (use_det_dynamics): all mass on the first bin whose value is >= the statistic
//   mode 2 (speed map)       : all mass on the last bin, risk = int8(100*(stat-lo)/range)
// [emu:begin collapse_pad]
__global__ void collapse_pad_kernel(const int8_t* __restrict__ raw, int8_t* __restrict__ out,
                                    int8_t* __restrict__ risk, int* __restrict__ bad_columns, const float* __restrict__ bin_values,
                                    int B, int H, int W, int keep_r, int keep_c, int pad, int risk_pitch, double alpha,
                                    float lo, float range, int mode) {
  const int Hp = keep_r + 2 * pad, Wp = keep_c + 2 * pad;
  const int cell = blockIdx.x * blockDim.x + threadIdx.x;
  if (cell >= Hp * Wp) return;
  const int r = cell / Wp, c = cell % Wp;
  const size_t plane = (size_t)Hp * Wp;
  const bool inner = r >= pad && r < pad + keep_r && c >= pad && c < pad + keep_c;
  if (!inner) {                                         // padding ring: zero traction, no risk information
    for (int b = 0; b < B; ++b) out[b * plane + cell] = (b == 0) ? 100 : 0;
    if (risk) risk[(size_t)r * risk_pitch + c] = 0;
    return;
  }
  const size_t src = (size_t)(r - pad) * W + (c - pad);
  const size_t splane = (size_t)H * W;
  int isum = 0;
  double wcum = 0.0, stat_m = 0.0, stat_w = 0.0;
  bool found = false;
  for (int b = 0; b < B; ++b) {
    const int pv = raw[b * splane + src];
    isum += pv;
    const double mass = __dmul_rn(0.01, (double)isum);
    wcum = __dadd_rn(wcum, __dmul_rn(__dmul_rn(0.01, (double)pv), (double)bin_values[b]));
    if (alpha != 1.0 && !found && mass >= alpha) { found = true; stat_m = mass; stat_w = wcum; }
    if (alpha != 1.0 && b == 0 && !found) { stat_m = mass; stat_w = wcum; }     // argmax of all-False is 0
  }
  if (isum != 100) atomicAdd(bad_columns, 1);
  const double stat = (alpha == 1.0) ? wcum : __ddiv_rn(stat_w, __dadd_rn(stat_m, 1e-6));
  if (mode == 1) {
    int chosen = 0;
    for (int b = 0; b < B; ++b)
      if (stat <= (double)bin_values[b]) { chosen = b; break; }
    for (int b = 0; b < B; ++b) out[b * plane + cell] = (b == chosen) ? 100 : 0;
  } else {
    for (int b = 0; b < B; ++b) out[b * plane + cell] = (b == B - 1) ? 100 : 0;
    const double v = __ddiv_rn(__dmul_rn(100.0, __dadd_rn(stat, -(double)lo)), (double)range);
    risk[(size_t)r * risk_pitch + c] = (int8_t)(long long)v;          // astype(int8): truncate, wrap
  }
}

// [emu:end collapse_pad]
void launch_collapse_pad(const int8_t* raw, int8_t* out, int8_t* risk, int* bad_columns, const float* bin_values, int B,
                         int H, int W, int keep_r, int keep_c, int pad, int risk_pitch, double alpha, float lo,
                         float range, int mode, cudaStream_t st) {
  const int cells = (keep_r + 2 * pad) * (keep_c + 2 * pad);
  collapse_pad_kernel<<<(cells + 255) / 256, 256, 0, st>>>(raw, out, risk, bad_columns, bin_values, B, H, W, keep_r,
                                                          keep_c, pad, risk_pitch, alpha, lo, range, mode);
}

// ---------------------------------------------------------------------------------------------
// v1 sampler: one thread per generator, direct global accesses.
__global__ void __launch_bounds__(128) sample_grids_kernel(const SampleGridsArgs a) {
  // thread order: ty fastest, then tx, then map -- a warp works on neighbouring tiles of one map
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int per_map = a.tx * a.ty;
  if (tid >= (int64_t)per_map * a.num_maps) return;
  const int m = (int)(tid / per_map);
  const int r = (int)(tid % per_map);
  const int tix = r / a.ty, tiy = r % a.ty;
  const int64_t gen = (int64_t)tix * ((int64_t)a.ty * a.num_maps) + (int64_t)m * a.ty + tiy;

  const int ncol = (a.cols + a.ty - 1) / a.ty;     // ceil(grid_cols / threads_y)
  const int nrow = (a.rows + a.tx - 1) / a.tx;
  const int r0 = min(tix * nrow, a.rows), r1 = min(r0 + nrow, a.rows);
  const int c0 = min(tiy * ncol, a.cols), c1 = min(c0 + ncol, a.cols);

  ulonglong2* sp = reinterpret_cast<ulonglong2*>(a.states) + gen;
  const ulonglong2 raw = *sp;
  Xoro s{raw.x, raw.y};
  int8_t* __restrict__ grid = a.grid + (size_t)m * a.grid_rows * a.pitch;

  for (int ri = r0; ri < r1; ++ri) {
    const int8_t* __restrict__ cum_row = a.cum + ((size_t)ri * a.cols + c0) * a.bpad;
    int8_t* __restrict__ out_row = grid + (size_t)ri * a.pitch;
    for (int ci = c0; ci < c1; ++ci, cum_row += a.bpad) {
      const float u = xoro_unit_f32(xoro_next(s));
      const double thr = ceil(((double)u * 100.0) * a.alpha_dyn);
      const int q = (int)(int8_t)(short)__double2int_rz(thr);     // cvt.rzi.s16.f64 ; low byte
      for (int b = 0; b < a.num_bins; ++b) {
        if (q <= (int)cum_row[b]) { out_row[ci] = a.qvals[b]; break; }
      }
    }
  }
  *sp = make_ulonglong2(s.s0, s.s1);
}

void launch_sample_grids(const SampleGridsArgs& a, cudaStream_t st) {
  const int64_t total = (int64_t)a.tx * a.ty * a.num_maps;
  const int threads = 128;
  sample_grids_kernel<<<(unsigned)((total + threads - 1) / threads), threads, 0, st>>>(a);
}

// ---------------------------------------------------------------------------------------------
// v2 sampler (the one solve() uses whenever the PMF is well-formed): same bit-exact streams, but
//   * a CTA owns one tile-row band of the map for GM consecutive maps: the band's cumulative-PMF rows
//     are staged ONCE in shared memory and reused by all GM maps x ty tile columns (the reference
//     re-reads B strided int8 per cell per map from global memory);
//   * the threshold q = int8(ceil(f64(f32(v*2^-53))*100*alpha)) is obtained WITHOUT the five float64 /
//     conversion (XU-pipe) instructions: q(v) is a monotone step function of the 53-bit draw v, so the
//     host tabulates its breakpoints T[k] = min{v : q(v) >= k} with the exact float arithmetic and folds
//     them into a 256-entry table over the top 8 bits of v: (q at the bucket start, the one breakpoint
//     inside the bucket, packed into one 64-bit word) -- one shared-memory load and one 64-bit compare per
//     draw (the host verifies that
//     no bucket holds two breakpoints, otherwise the generic kernel is used);
//   * the first bin whose cumulative mass reaches q is found with a SIMD-in-register byte compare and
//     one POPC instead of a loop;
//   * sampled bytes are staged per row in shared memory and written with coalesced 16-byte stores;
//   * NT = 2 samples the linear and angular maps together from ONE stream when both TDMs hold identical
//     generator states (same seed, same history -- the reference seeds both with cfg.seed, so their
//     streams are identical; SURVEY.md 9-Q8): the draw and the threshold are shared.
// [emu:begin sampler_v2]   (tests/emu_sampler.py compiles the text between these markers for the host)
// GF(2) jump-ahead: the xoroshiro128+ transition is linear, so advancing a state by K draws is a
// 128x128 bit-matrix product.  `mat` holds the 128 columns (2 x u64 each) of A^K.
__device__ __forceinline__ void xoro_jump(Xoro& s, const ulonglong2* __restrict__ mat) {
  uint64_t a0 = 0, a1 = 0;
#pragma unroll 4
  for (int j = 0; j < 64; ++j) {
    const ulonglong2 c = __ldg(mat + j);
    const uint64_t mk = 0ULL - ((s.s0 >> j) & 1ULL);
    a0 ^= c.x & mk; a1 ^= c.y & mk;
  }
#pragma unroll 4
  for (int j = 0; j < 64; ++j) {
    const ulonglong2 c = __ldg(mat + 64 + j);
    const uint64_t mk = 0ULL - ((s.s1 >> j) & 1ULL);
    a0 ^= c.x & mk; a1 ^= c.y & mk;
  }
  s.s0 = a0; s.s1 = a1;
}

// the same product with the matrix staged in shared memory (every thread of a CTA applies the same one or two
// matrices: 2 KB each, one cooperative copy instead of 128 dependent cache loads per thread)
__device__ __forceinline__ void xoro_jump_smem(Xoro& s, const ulonglong2* mat) {
  uint64_t a0 = 0, a1 = 0;
#pragma unroll 8
  for (int j = 0; j < 64; ++j) {
    const ulonglong2 c = mat[j];
    const uint64_t mk = 0ULL - ((s.s0 >> j) & 1ULL);
    a0 ^= c.x & mk; a1 ^= c.y & mk;
  }
#pragma unroll 8
  for (int j = 0; j < 64; ++j) {
    const ulonglong2 c = mat[64 + j];
    const uint64_t mk = 0ULL - ((s.s1 >> j) & 1ULL);
    a0 ^= c.x & mk; a1 ^= c.y & mk;
  }
  s.s0 = a0; s.s1 = a1;
}

// sampled value looked up from shared memory (false) or from a 16-byte register table with PRMT (true): the
// register variant costs four more ALU-pipe instructions per cell and map, the shared-memory one a byte load
constexpr bool SG_VALUES_IN_REGISTERS = false;
// count the bytes >= q with one POPC per word (true) or one POPC after shifting the words' flags apart (false)
#ifndef SG_POPC_VARIANT
#define SG_POPC_VARIANT 1
#endif
constexpr bool SG_POPC_PER_WORD = SG_POPC_VARIANT;

// BOUNDED: only maps [0, map_end) are sampled (else all a.num_maps); the generator of map m is the same either way
template <int NT, int NW, bool BOUNDED = false>
__device__ __forceinline__ void sample_grids_v2_body(const SampleGridsV2Args& a, int map_end = 0) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int nw = (NW > 0) ? NW : a.t[0].bpad / 4;
  const int bpad = nw * 4;
  const int ncol = (a.cols + a.ty - 1) / a.ty;
  const int nrow = (a.rows + a.tx - 1) / a.tx;
  const int tix = a.tix_lo + blockIdx.x / a.segs, seg = blockIdx.x % a.segs;
  const int t0 = min(tix * nrow, a.rows), t1 = min(t0 + nrow, a.rows);          // the generator's tile rows
  // this CTA's row segment of the tile.  A generator's stream is split into `segs` consecutive row
  // segments handled by different CTAs: segment `seg` starts from the state jumped ahead by
  // seg*seg_rows*(c1-c0) draws (GF(2) matrix), so the union of the segments is the reference's stream.
  const int r0 = min(t0 + seg * a.seg_rows, t1), r1 = min(r0 + a.seg_rows, t1);
  // rows of this segment inside the reach box (CTA-uniform)
  const int rs0 = max(r0, a.row_lo), rs1 = min(r1, a.row_hi);
  // active tile columns of THIS CTA: those of the launch, narrowed to the reach DISC when one is given -- the rows
  // [rs0, rs1) are at least dy cells away from the centre row, so only columns within sqrt(R^2 - dy^2) of the centre
  // column can be read.  Threads are re-mapped onto the narrower range, which parks whole warps instead of lanes.
  int tiy_lo = a.tiy_lo, nact = a.nact;
  if (a.disc_r > 0.0f && rs0 < rs1) {
    // row r holds the positions [r, r + 1) in cell coordinates: distance of [rs0, rs1) from the centre
    const float dy = (a.disc_cy < (float)rs0) ? (float)rs0 - a.disc_cy
                   : (a.disc_cy > (float)rs1) ? a.disc_cy - (float)rs1 : 0.0f;
    const float w2 = a.disc_r * a.disc_r - dy * dy;
    if (w2 <= 0.0f) {
      nact = 0;                                               // the whole segment lies outside the disc
    } else {
      const float w = sqrtf(w2) + 1.0f;
      const int lo = max(a.tiy_lo, (int)floorf((a.disc_cx - w) / (float)ncol));
      const int hi = min(a.tiy_lo + a.nact - 1, (int)floorf((a.disc_cx + w) / (float)ncol));
      tiy_lo = lo; nact = max(hi - lo + 1, 0);
    }
  }
  if (nact == 0) return;                                      // CTA-uniform: nothing to sample here
  // staged column window [cs0, cs1): the active tile columns, start rounded down to 16 cells (16-byte stores)
  const int cfirst = min(tiy_lo * ncol, a.cols);
  const int cs0 = cfirst & ~15;
  const int cs1 = min((tiy_lo + nact) * ncol, a.cols);
  const int wcols = cs1 - cs0;
  const int row_bytes = wcols * bpad;                        // the window's slice of one cumulative-table row
  const int row_bytes_al = (row_bytes + 15) & ~15;
  const int stage_pitch = (wcols + 15) & ~15;
  const int gm = a.gm;
  unsigned char* s_cum = smem;                               // [NT][row_bytes_al]
  unsigned char* s_stage = s_cum + NT * row_bytes_al;        // [NT][gm][stage_pitch]
  uint64_t* s_T = reinterpret_cast<uint64_t*>(s_stage + max(NT * gm * stage_pitch, 2 * 128 * 16));   // [256] thr | qbase
  unsigned char* s_q = reinterpret_cast<unsigned char*>(s_T + SAMPLE_TABLE_WORDS);   // [NT][128]
  // [2][128] segment-start jump matrices: they live in the (not yet used) output stage -- every thread has applied
  // them before the row loop's first barrier, after which the stage is written
  ulonglong2* s_J = reinterpret_cast<ulonglong2*>(s_stage);

  const int tid = threadIdx.x, nthreads = blockDim.x;
  const int tiy = tiy_lo + tid % nact, mloc = tid / nact;
  const int m = blockIdx.y * gm + mloc;
  const bool active = (mloc < gm) && (m < (BOUNDED ? map_end : a.num_maps));

  for (int i = tid; i < SAMPLE_TABLE_WORDS; i += nthreads) s_T[i] = a.thresholds[i];
  // value table indexed by ge = number of cumulative bytes >= q (the SIMD compare yields that count directly):
  // bin = 4*nw - ge, so the table is stored reversed and the lookup is one byte load at s_q[ge]
  for (int i = tid; i < 128; i += nthreads) {
    const int b = bpad - i;
    s_q[i] = (b >= 0) ? (unsigned char)a.t[0].qvals[b] : 0;
    if (NT == 2) s_q[128 + i] = (b >= 0) ? (unsigned char)a.t[1].qvals[b] : 0;
  }

  // alternative kept for A/B timing: value tables for <= 16 bins in registers (4 x 32-bit per TDM), PRMT lookup
  uint32_t qreg[NT][4];
  if (SG_VALUES_IN_REGISTERS) {
#pragma unroll
    for (int k = 0; k < NT; ++k) {
      const int8_t* qv = (NT == 2 && k == 1) ? a.t[1].qvals : a.t[0].qvals;
#pragma unroll
      for (int w = 0; w < 4; ++w) qreg[k][w] = __ldg(reinterpret_cast<const uint32_t*>(qv) + w);
    }
  }

  const int c0 = min(tiy * ncol, a.cols), c1 = min(c0 + ncol, a.cols);
  const int wc = c1 - c0;
  const int last_seg = (t1 > t0 && wc > 0) ? (t1 - t0 - 1) / a.seg_rows : 0;     // owner of the final state

  // one cumulative-table row of the window -> shared memory, with the guard bits of cell()
  auto stage_cum_row = [&](int ri) {
#pragma unroll
    for (int k = 0; k < NT; ++k) {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(a.t[k].cum + ((size_t)ri * a.cols + cs0) * bpad);
      uint32_t* dst = reinterpret_cast<uint32_t*>(s_cum + k * row_bytes_al);
#pragma unroll 8
      for (int i = tid; i < row_bytes / 4; i += nthreads) dst[i] = __ldg(src + i) | 0x80808080u;
    }
  };
  // the first row is staged before the jump-ahead below, whose arithmetic then hides the loads' latency (the jump
  // matrices overlay the output stage, not the cumulative rows)
  if (rs0 < rs1) stage_cum_row(rs0);

  const int64_t gen = (int64_t)tix * ((int64_t)a.ty * a.num_maps) + (int64_t)m * a.ty + tiy;
  if (seg > 0) {                                            // both width classes of this segment's jump (CTA-uniform)
    const ulonglong2* src = reinterpret_cast<const ulonglong2*>(a.jump) + (size_t)(seg - 1) * 2 * 128;
    for (int i = tid; i < 2 * 128; i += nthreads) s_J[i] = __ldg(src + i);
    __syncthreads();
  }
  Xoro s{0, 0};
  if (active) {
    const ulonglong2 raw = reinterpret_cast<const ulonglong2*>(a.t[0].states)[gen];
    s.s0 = raw.x; s.s1 = raw.y;
    if (seg > 0 && r1 > r0 && wc > 0) {
      const int cls = (wc == ncol) ? 0 : 1;                 // full-width tile column or the narrower last one
      xoro_jump_smem(s, s_J + cls * 128);
    }
  }
  // the draws of the segment's rows above the box are consumed without sampling (one xoroshiro step per cell), rows
  // below it are simply not walked
  if (active && rs0 < rs1)
    for (int64_t i = (int64_t)(rs0 - r0) * wc; i > 0; --i) xoro_next(s);

  // two barriers per row: row ri's cumulative slice is staged (and the previous row's output stage drained) before
  // the cells; after them, the write-back of row ri and the staging of row ri + 1 run together
  for (int ri = rs0; ri < rs1; ++ri) {
    __syncthreads();
    if (active) {
      // one cell: threshold from the 53-bit draw, then the first bin whose cumulative mass reaches it.
      // Returns the sampled value byte of each TDM; the caller stores them AFTER a group of cells so that
      // the shared-memory loads of the whole group are independent of the byte stores (ILP).
      auto cell = [&](int ci, uint64_t r, uint32_t (&outv)[NT]) {
        // bucket of the raw draw's top 8 bits: q at the bucket start and the single breakpoint inside it
        const uint32_t q = sample_threshold_q(r, s_T);
        const uint32_t qq = q * 0x01010101u;
#pragma unroll
        for (int k = 0; k < NT; ++k) {
          const uint32_t* cw = reinterpret_cast<const uint32_t*>(s_cum + k * row_bytes_al + (ci - cs0) * bpad);
          // staged bytes carry bit 7 (guard): (0x80 | cum) - q never borrows across bytes (cum, q <= 127) and
          // leaves bit 7 SET exactly for the bytes with cum >= q.
          int ge = 0;                                         // cum is monotone: first bin >= q  =  4*nw - ge
          if (SG_POPC_PER_WORD) {
            // one mask + one POPC per word (POPC issues on its own quarter-rate pipe, the shifts of the variant below
            // on the ALU pipe, which is the one this kernel saturates)
            if (NW > 0) {
#pragma unroll
              for (int w = 0; w < (NW > 0 ? NW : 1); ++w) ge += __popc((cw[w] - qq) & 0x80808080u);
            } else {
              for (int w = 0; w < nw; ++w) ge += __popc((cw[w] - qq) & 0x80808080u);
            }
          } else {
            // word w contributes its four flags at bit 7-w of each byte: shift, then one LOP3 does bits | (z & mask)
            uint32_t bits = 0;
            if (NW > 0) {
#pragma unroll
              for (int w = 0; w < (NW > 0 ? NW : 1); ++w) bits |= ((cw[w] - qq) >> (7 - w)) & (0x80808080u >> (7 - w));
            } else {
              for (int w = 0; w < nw; ++w) bits |= ((cw[w] - qq) >> (7 - w)) & (0x80808080u >> (7 - w));
            }
            ge = __popc(bits);
          }
          if (SG_VALUES_IN_REGISTERS && NW > 0 && NW <= 4) {
            const int bin = 4 * NW - ge;
            const uint32_t lo8 = __byte_perm(qreg[k][0], qreg[k][1], bin & 7);
            const uint32_t hi8 = __byte_perm(qreg[k][2], qreg[k][3], bin & 7);
            outv[k] = ((bin & 8) ? hi8 : lo8) & 0xffu;
          } else {
            outv[k] = s_q[k * 128 + ge];
          }
        }
      };
      unsigned char* st0 = s_stage + mloc * stage_pitch - cs0;          // indexed by the map column
      unsigned char* st1 = s_stage + (gm + mloc) * stage_pitch - cs0;
      int ci = c0;
      for (; ci + 4 <= c1; ci += 4) {          // 4 draws in stream order, then 4 independent cells (ILP)
        uint64_t r[4];
        uint32_t o[4][NT];
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = xoro_next(s);
#pragma unroll
        for (int j = 0; j < 4; ++j) cell(ci + j, r[j], o[j]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          st0[ci + j] = (unsigned char)o[j][0];
          if (NT == 2) st1[ci + j] = (unsigned char)o[j][NT - 1];
        }
      }
      for (; ci < c1; ++ci) {
        uint32_t o[NT];
        cell(ci, xoro_next(s), o);
        st0[ci] = (unsigned char)o[0];
        if (NT == 2) st1[ci] = (unsigned char)o[NT - 1];
      }
    }
    __syncthreads();                                          // every cell of row ri read s_cum and wrote the stage
    if (ri + 1 < rs1) stage_cum_row(ri + 1);
    // coalesced write-back of the gm x NT staged rows: 16-byte chunks, bytes at the ragged ends of the window
    const int chunks = (wcols + 15) / 16;
    const int maps_here = min(gm, (BOUNDED ? map_end : a.num_maps) - (int)blockIdx.y * gm);
    for (int idx = tid; idx < NT * maps_here * chunks; idx += nthreads) {
      const int ch = idx % chunks;
      const int km = idx / chunks;
      const int k = km / maps_here, ml = km % maps_here;
      const unsigned char* srow = s_stage + (k * gm + ml) * stage_pitch + ch * 16;
      int8_t* gbase = (NT == 2 && k == 1) ? a.t[1].grid : a.t[0].grid;
      int8_t* grow = gbase + ((size_t)(blockIdx.y * gm + ml) * a.grid_rows + ri) * a.pitch + cs0 + ch * 16;
      const int lo = max(cfirst - (cs0 + ch * 16), 0), hi = min(cs1 - (cs0 + ch * 16), 16);
      if (lo == 0 && hi == 16) {
        *reinterpret_cast<uint4*>(grow) = *reinterpret_cast<const uint4*>(srow);
      } else {
        for (int b = lo; b < hi; ++b) grow[b] = (int8_t)srow[b];
      }
    }
  }
  // states are double-buffered (another segment of the same generator may still have to read the old
  // state): exactly one segment per generator writes the new state
  if (a.write_states && active && seg == last_seg) {
    reinterpret_cast<ulonglong2*>(a.t[0].states_out)[gen] = make_ulonglong2(s.s0, s.s1);
    if (NT == 2) reinterpret_cast<ulonglong2*>(a.t[1].states_out)[gen] = make_ulonglong2(s.s0, s.s1);
  }
}

// four CTAs of 256 threads per SM: a budget of 64 registers, with which every single-planner variant but <2,8> runs
// without spills (left to itself ptxas picks 40-48 and spills in some of them)
template <int NT, int NW>
__global__ void __launch_bounds__(256, 4) sample_grids_v2_kernel(const SampleGridsV2Args a) {
  sample_grids_v2_body<NT, NW>(a);
}

// whole-tile advance of every generator (box mode: the sampler walks only part of each tile, so the states a
// whole-map walk would leave behind are produced by ONE GF(2) jump per generator).  Tile classes as sample_tile_draws.
__device__ __forceinline__ void advance_states_body(const ulonglong2* __restrict__ in, ulonglong2* __restrict__ out0,
                                                    ulonglong2* __restrict__ out1, const ulonglong2* __restrict__ mats,
                                                    int rows, int cols, int tx, int ty, int num_maps) {
  extern __shared__ __align__(16) unsigned char smem[];
  ulonglong2* s_M = reinterpret_cast<ulonglong2*>(smem);      // the four tile-class matrices, 8 KB
  for (int i = threadIdx.x; i < 4 * 128; i += blockDim.x) s_M[i] = __ldg(mats + i);
  __syncthreads();
  const int64_t gen = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gen >= (int64_t)tx * ty * num_maps) return;
  const int tix = (int)(gen / ((int64_t)ty * num_maps)), tiy = (int)(gen % ty);
  const int ncol = (cols + ty - 1) / ty, nrow = (rows + tx - 1) / tx;
  const int t0 = min(tix * nrow, rows), t1 = min(t0 + nrow, rows);
  const int c0 = min(tiy * ncol, cols), c1 = min(c0 + ncol, cols);
  const ulonglong2 raw = in[gen];
  Xoro s{raw.x, raw.y};
  if (t1 > t0 && c1 > c0) xoro_jump_smem(s, s_M + (((t1 - t0 == nrow) ? 0 : 2) + ((c1 - c0 == ncol) ? 0 : 1)) * 128);
  out0[gen] = make_ulonglong2(s.s0, s.s1);
  if (out1) out1[gen] = make_ulonglong2(s.s0, s.s1);
}
__global__ void __launch_bounds__(128) advance_states_kernel(const ulonglong2* __restrict__ in, ulonglong2* __restrict__ out0,
                                                             ulonglong2* __restrict__ out1, const ulonglong2* __restrict__ mats,
                                                             int rows, int cols, int tx, int ty, int num_maps) {
  advance_states_body(in, out0, out1, mats, rows, cols, tx, ty, num_maps);
}

// [emu:end sampler_v2]
// [emu:begin sampler_batch]
// batched one-map solves: one fused lin + ang whole-map launch for every pair of the batch, pair blockIdx.z (or
// pairs[blockIdx.z]: the pairs of one launch class of a trial batch).  The pairs share the kernel variant (bins) and the
// thread tile; the launch is sized for the largest pair, and each pair's CTAs do what its own launch does, from its
// descriptor (rows, cols, pitch, segments, TDM buffers, threshold table, jump matrices): the CTAs beyond its own
// launch return.  A pair with active[z] == 0 is left untouched (active null: every pair runs).
// The CTA lies inside its own pair's launch (CTA-uniform)
__device__ __forceinline__ bool v2_cta_in_launch(const SampleGridsV2Args& a) {
  return (int)blockIdx.x < sample_v2_grid_x(a) && (int)blockIdx.y * a.gm < a.num_maps;
}
template <int NT, int NW>
__global__ void __launch_bounds__(256) sample_grids_v2_batch_kernel(const SampleGridsV2Args* __restrict__ descs,
                                                                    const int* __restrict__ active = nullptr,
                                                                    const int* __restrict__ pairs = nullptr) {
  const int z = pairs ? pairs[blockIdx.z] : (int)blockIdx.z;
  if (active && !active[z]) return;
  const SampleGridsV2Args& a = descs[z];
  if (!v2_cta_in_launch(a)) return;
  sample_grids_v2_body<NT, NW>(a);
}
// Trials of planners sharing TDM pairs: blockIdx.z (or pairs[blockIdx.z]) is a group (its pair's descriptor), which
// samples at every step while any of its members runs (group_running, kernels.h).
template <int NT, int NW>
__global__ void __launch_bounds__(256) sample_grids_v2_group_batch_kernel(const SampleGridsV2Args* __restrict__ descs,
                                                                          const SampleGroupDesc* __restrict__ groups,
                                                                          const int* __restrict__ members,
                                                                          const int* __restrict__ active,
                                                                          const int* __restrict__ pairs = nullptr) {
  const int z = pairs ? pairs[blockIdx.z] : (int)blockIdx.z;
  if (!group_running(groups[z], members, active)) return;
  const SampleGridsV2Args& a = descs[z];
  if (!v2_cta_in_launch(a)) return;
  sample_grids_v2_body<NT, NW>(a);
}
// [emu:end sampler_batch]
// [emu:begin sampler_box_batch]
// closed-loop trials of a stochastic batch: the fused pair blockIdx.z (or pairs[blockIdx.z]: the pairs of one launch
// class) samples the reach box its planner's solve() would sample (reach_box_decide from the x0 the plant step wrote and
// this step's reach statistic), or whole maps.  The launch is sized for the largest box the static bound allows over
// the class: `mrows` tile rows times the largest pair's box row segments, `ncact` tile columns and the boxed launch's
// maps per CTA (a.gm, the class's); a pair's CTAs beyond its own mrows x a.segs and maps return.  A boxed step is one pass whose tile rows start at the box's
// first one; a CTA narrows to the box rows, columns and disc as the single boxed launch does, so it writes the same
// cells with the same draws.  A whole-map step (and any box larger than the launch) loops over groups of mrows tile rows
// and ncact tile columns.
// The passes of one CTA over tile rows [tix_lo, tix_hi) and tile columns [tiy_lo, tiy_hi) of maps [0, map_end).
template <int NW>
__device__ __forceinline__ void box_batch_passes(SampleGridsV2Args& a, int tix_lo, int tix_hi, int tiy_lo, int tiy_hi,
                                                 int mrows, int ncact, int map_end) {
  if ((int)blockIdx.x >= mrows * a.segs || (int)blockIdx.y * a.gm >= map_end) return;    // beyond this pair's launch
  const int nrow = (a.rows + a.tx - 1) / a.tx;
  const int tsub = (int)blockIdx.x / a.segs, seg = (int)blockIdx.x % a.segs;
  for (int tg = tix_lo; tg < tix_hi; tg += mrows) {
    const int tix = tg + tsub;
    if (tix >= tix_hi) continue;                                   // CTA-uniform
    const int t0 = min(tix * nrow, a.rows), t1 = min(t0 + nrow, a.rows);
    const int r0 = min(t0 + seg * a.seg_rows, t1), r1 = min(r0 + a.seg_rows, t1);
    if (max(r0, a.row_lo) >= min(r1, a.row_hi)) continue;          // no box rows in this segment
    for (int cg = tiy_lo; cg < tiy_hi; cg += ncact) {
      a.tix_lo = tg; a.tiy_lo = cg; a.nact = min(ncact, tiy_hi - cg);
      sample_grids_v2_body<2, NW, true>(a, map_end);
      __syncthreads();                                             // the next pass restages the shared memory
    }
  }
}

template <int NW>
__global__ void __launch_bounds__(256) sample_grids_v2_box_batch_kernel(const SampleGridsV2Args* __restrict__ descs,
                                                                        const SampleBoxDesc* __restrict__ boxes,
                                                                        const int* __restrict__ active, int iter,
                                                                        int mrows, int ncact,
                                                                        const int* __restrict__ pairs = nullptr) {
  const int z = pairs ? pairs[blockIdx.z] : (int)blockIdx.z;
  if (active && !active[z]) return;
  SampleGridsV2Args a = descs[z];
  const SampleBoxDesc& bd = boxes[z];
  const float reach = bd.reach[bd.slot ^ (iter & 1)];
  ReachBox b;
  const int how = reach_box_decide(bd.c, bd.x0[0], bd.x0[1], bd.c.mode == 2 ? &reach : nullptr, &b);
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
    bd.record[0] = how;
    bd.record[1] = how ? b.row_lo : 0; bd.record[2] = how ? b.row_hi : a.rows;
    bd.record[3] = how ? b.col_lo : 0; bd.record[4] = how ? b.col_hi : a.cols;
  }
  const int nrow = (a.rows + a.tx - 1) / a.tx;
  int tix_lo = 0, tix_hi = a.tx, tiy_lo = 0, tiy_hi = a.ty;          // tile rows / columns to cover, [lo, hi)
  if (how) {
    a.row_lo = b.row_lo; a.row_hi = b.row_hi;
    a.disc_cx = b.cx; a.disc_cy = b.cy; a.disc_r = b.r;
    tix_lo = b.row_lo / nrow; tix_hi = min(a.tx, (b.row_hi - 1) / nrow + 1);
    tiy_lo = b.tiy_lo; tiy_hi = b.tiy_lo + b.nact;
  }
  a.write_states = 0;
  box_batch_passes<NW>(a, tix_lo, tix_hi, tiy_lo, tiy_hi, mrows, ncact, a.num_maps);
}

// recording stochastic trials: the whole maps [0, map_end) of every pair whose step sampled a box (its record says so),
// re-walked from the step's pre-call states (descs[z].t[0].states) with the launch geometry of the box launch above and
// no state stores.  Inside the box that rewrites the values the boxed launch wrote; maps >= map_end keep their box.
template <int NW>
__global__ void __launch_bounds__(256) sample_grids_v2_complete_batch_kernel(const SampleGridsV2Args* __restrict__ descs,
                                                                             const SampleBoxDesc* __restrict__ boxes,
                                                                             const int* __restrict__ active, int map_end,
                                                                             int mrows, int ncact,
                                                                             const int* __restrict__ pairs = nullptr) {
  const int z = pairs ? pairs[blockIdx.z] : (int)blockIdx.z;
  if (active && !active[z]) return;
  if (boxes[z].record[0] == 0) return;                             // this step sampled whole maps already
  SampleGridsV2Args a = descs[z];
  a.write_states = 0;
  box_batch_passes<NW>(a, 0, a.tx, 0, a.ty, mrows, ncact, map_end);
}

// the state advance of those boxed samplings for every pair (pair blockIdx.y, or pairs[blockIdx.y]): lin's states into
// both TDMs' other buffers.  Each pair's rows, cols and thread tile come from its descriptor; the launch covers the
// tx x ty x num_maps generators its class shares.  The five int arguments (rows, cols, tx, ty, num_maps of a
// one-geometry launch) are not read.
__global__ void __launch_bounds__(128) advance_states_batch_kernel(const SampleGridsV2Args* __restrict__ descs,
                                                                   const SampleBoxDesc* __restrict__ boxes,
                                                                   const int* __restrict__ active, int, int, int, int, int,
                                                                   const int* __restrict__ pairs = nullptr) {
  const int z = pairs ? pairs[blockIdx.y] : (int)blockIdx.y;
  if (active && !active[z]) return;
  const SampleGridsV2Args& a = descs[z];
  advance_states_body(reinterpret_cast<const ulonglong2*>(a.t[0].states), reinterpret_cast<ulonglong2*>(a.t[0].states_out),
                      reinterpret_cast<ulonglong2*>(a.t[1].states_out),
                      reinterpret_cast<const ulonglong2*>(boxes[z].jump_tile), a.rows, a.cols, a.tx, a.ty, a.num_maps);
}

// The same three launches for groups of planners on one shared pair (group blockIdx.z / blockIdx.y or pairs[] of it,
// descs one per group, boxes one per planner).  A group's CTAs return while none of its members runs.  The box kernel decides every running
// member's box and samples their hull (reach_box_hull: one running member's box is exactly its own, disc included);
// CTA (0, 0) records the decision in the group's record and in every running member's.
template <int NW>
__global__ void __launch_bounds__(256) sample_grids_v2_group_box_batch_kernel(
    const SampleGridsV2Args* __restrict__ descs, const SampleBoxDesc* __restrict__ boxes,
    const SampleGroupDesc* __restrict__ groups, const int* __restrict__ members, const int* __restrict__ active, int iter,
    int mrows, int ncact, const int* __restrict__ pairs = nullptr) {
  const int z = pairs ? pairs[blockIdx.z] : (int)blockIdx.z;
  const SampleGroupDesc& gd = groups[z];
  ReachBox b;
  int n = 0;
  for (int j = gd.first; j < gd.first + gd.count; ++j) {
    const int k = members[j];
    if (!active[k]) continue;
    const SampleBoxDesc& bd = boxes[k];
    const float reach = bd.reach[bd.slot ^ (iter & 1)];
    ReachBox m;
    reach_box_decide(bd.c, bd.x0[0], bd.x0[1], bd.c.mode == 2 ? &reach : nullptr, &m);
    reach_box_hull_add(&b, n++, m);
  }
  if (n == 0) return;
  const int how = reach_box_hull_close(boxes[members[gd.first]].c, n, &b);
  SampleGridsV2Args a = descs[z];
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
    const int r[5] = {how, how ? b.row_lo : 0, how ? b.row_hi : a.rows, how ? b.col_lo : 0, how ? b.col_hi : a.cols};
    for (int c = 0; c < 5; ++c) gd.record[c] = r[c];
    for (int j = gd.first; j < gd.first + gd.count; ++j)
      if (active[members[j]])
        for (int c = 0; c < 5; ++c) boxes[members[j]].record[c] = r[c];
  }
  const int nrow = (a.rows + a.tx - 1) / a.tx;
  int tix_lo = 0, tix_hi = a.tx, tiy_lo = 0, tiy_hi = a.ty;          // tile rows / columns to cover, [lo, hi)
  if (how) {
    a.row_lo = b.row_lo; a.row_hi = b.row_hi;
    a.disc_cx = b.cx; a.disc_cy = b.cy; a.disc_r = b.r;
    tix_lo = b.row_lo / nrow; tix_hi = min(a.tx, (b.row_hi - 1) / nrow + 1);
    tiy_lo = b.tiy_lo; tiy_hi = b.tiy_lo + b.nact;
  }
  a.write_states = 0;
  box_batch_passes<NW>(a, tix_lo, tix_hi, tiy_lo, tiy_hi, mrows, ncact, a.num_maps);
}

template <int NW>
__global__ void __launch_bounds__(256) sample_grids_v2_group_complete_batch_kernel(
    const SampleGridsV2Args* __restrict__ descs, const SampleGroupDesc* __restrict__ groups,
    const int* __restrict__ members, const int* __restrict__ active, int map_end, int mrows, int ncact,
    const int* __restrict__ pairs = nullptr) {
  const int z = pairs ? pairs[blockIdx.z] : (int)blockIdx.z;
  const SampleGroupDesc& gd = groups[z];
  if (!group_running(gd, members, active)) return;
  if (gd.record[0] == 0) return;                                   // this step sampled whole maps already
  SampleGridsV2Args a = descs[z];
  a.write_states = 0;
  box_batch_passes<NW>(a, 0, a.tx, 0, a.ty, mrows, ncact, map_end);
}

__global__ void __launch_bounds__(128) advance_states_group_batch_kernel(const SampleGridsV2Args* __restrict__ descs,
                                                                         const SampleBoxDesc* __restrict__ boxes,
                                                                         const SampleGroupDesc* __restrict__ groups,
                                                                         const int* __restrict__ members,
                                                                         const int* __restrict__ active, int, int,
                                                                         int, int, int,
                                                                         const int* __restrict__ pairs = nullptr) {
  const int z = pairs ? pairs[blockIdx.y] : (int)blockIdx.y;
  const SampleGroupDesc& gd = groups[z];
  if (!group_running(gd, members, active)) return;
  const SampleGridsV2Args& a = descs[z];
  advance_states_body(reinterpret_cast<const ulonglong2*>(a.t[0].states), reinterpret_cast<ulonglong2*>(a.t[0].states_out),
                      reinterpret_cast<ulonglong2*>(a.t[1].states_out),
                      reinterpret_cast<const ulonglong2*>(boxes[members[gd.first]].jump_tile), a.rows, a.cols, a.tx,
                      a.ty, a.num_maps);
}
// [emu:end sampler_box_batch]

void launch_advance_states(const uint64_t* states, uint64_t* out0, uint64_t* out1, const uint64_t* mats, int rows,
                           int cols, int tx, int ty, int num_maps, cudaStream_t st) {
  const int64_t total = (int64_t)tx * ty * num_maps;
  advance_states_kernel<<<(unsigned)((total + 127) / 128), 128, 4 * 128 * 16, st>>>(
      reinterpret_cast<const ulonglong2*>(states), reinterpret_cast<ulonglong2*>(out0),
      reinterpret_cast<ulonglong2*>(out1), reinterpret_cast<const ulonglong2*>(mats), rows, cols, tx, ty, num_maps);
}

// draws of a whole-map walk per tile class: [0] full x full, [1] full height x last width, [2] last height x full
// width, [3] last x last ("last" = the one ragged, non-empty tile row / column; equal to "full" if none is ragged)
void sample_tile_draws(int rows, int cols, int tx, int ty, int64_t ks[4]) {
  const int nrow = (rows + tx - 1) / tx, ncol = (cols + ty - 1) / ty;
  int last_h = rows % nrow ? rows % nrow : nrow;
  int last_w = cols % ncol ? cols % ncol : ncol;
  ks[0] = (int64_t)nrow * ncol; ks[1] = (int64_t)nrow * last_w;
  ks[2] = (int64_t)last_h * ncol; ks[3] = (int64_t)last_h * last_w;
}

size_t sample_grids_v2_smem(const SampleGridsV2Args& a, int nt) {
  return sample_v2_smem_hd(a.tiy_lo, a.nact, a.ty, a.cols, a.t[0].bpad, a.gm, nt);
}

static int v2_threads(const SampleGridsV2Args& a) { return ((a.nact * a.gm + 31) / 32) * 32; }

template <int NT>
static void launch_v2_nt(const SampleGridsV2Args& a, cudaStream_t st) {
  const int nrow = (a.rows + a.tx - 1) / a.tx;
  const int tix_hi = std::min(a.tx - 1, (std::max(a.row_hi, a.row_lo + 1) - 1) / nrow);     // last tile row with box rows
  const dim3 grid((tix_hi - a.tix_lo + 1) * a.segs, (a.num_maps + a.gm - 1) / a.gm);
  const int threads = v2_threads(a);
  const size_t smem = sample_grids_v2_smem(a, NT);
  const int nw = a.t[0].bpad / 4;
  auto go = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, threads, smem, st>>>(a);
  };
  if (nw == 3) go(sample_grids_v2_kernel<NT, 3>);
  else if (nw == 8) go(sample_grids_v2_kernel<NT, 8>);
  else if (nw == 1) go(sample_grids_v2_kernel<NT, 1>);
  else go(sample_grids_v2_kernel<NT, 0>);
}

bool sample_grids_v2_fits(const SampleGridsV2Args& a, int nt) {
  return sample_v2_fits_hd(a.tiy_lo, a.nact, a.ty, a.cols, a.t[0].bpad, a.t[1].bpad, a.gm, nt);
}

void launch_sample_grids_v2(const SampleGridsV2Args& a, int nt, cudaStream_t st) {
  if (nt == 2) launch_v2_nt<2>(a, st); else launch_v2_nt<1>(a, st);
}

bool sample_grids_v2_same_launch(const SampleGridsV2Args& a, const SampleGridsV2Args& b) {
  return a.rows == b.rows && a.cols == b.cols && a.grid_rows == b.grid_rows && a.pitch == b.pitch && a.tx == b.tx &&
         a.ty == b.ty && a.num_maps == b.num_maps && a.segs == b.segs && a.seg_rows == b.seg_rows && a.gm == b.gm &&
         a.tix_lo == b.tix_lo && a.tiy_lo == b.tiy_lo && a.nact == b.nact && a.row_lo == b.row_lo &&
         a.row_hi == b.row_hi && a.t[0].bpad == b.t[0].bpad && a.t[1].bpad == b.t[1].bpad;
}

SampleClassLaunch sample_class_launch(const SampleGridsV2Args* const* members, int count) {
  SampleClassLaunch L{};
  L.nw = members[0]->t[0].bpad / 4;
  for (int i = 0; i < count; ++i) {
    const SampleGridsV2Args& a = *members[i];
    L.gx = std::max(L.gx, sample_v2_grid_x(a));
    L.gy = std::max(L.gy, (a.num_maps + a.gm - 1) / a.gm);
    L.gm = std::max(L.gm, a.gm);
    L.threads = std::max(L.threads, v2_threads(a));
    L.smem = std::max(L.smem, sample_grids_v2_smem(a, 2));
  }
  return L;
}

void launch_sample_grids_v2_batch(const SampleClassLaunch& L, const SampleGridsV2Args* descs, int count,
                                  const int* pairs, const int* active, cudaStream_t st, const SampleGroupDesc* groups,
                                  const int* members) {
  const dim3 grid(L.gx, L.gy, count);
  const int threads = L.threads;
  const size_t smem = L.smem;
  const int nw = L.nw;
  auto go = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, threads, smem, st>>>(descs, active, pairs);
  };
  auto go_groups = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, threads, smem, st>>>(descs, groups, members, active, pairs);
  };
  if (groups) {
    if (nw == 3) go_groups(sample_grids_v2_group_batch_kernel<2, 3>);
    else if (nw == 8) go_groups(sample_grids_v2_group_batch_kernel<2, 8>);
    else if (nw == 1) go_groups(sample_grids_v2_group_batch_kernel<2, 1>);
    else go_groups(sample_grids_v2_group_batch_kernel<2, 0>);
    return;
  }
  if (nw == 3) go(sample_grids_v2_batch_kernel<2, 3>);
  else if (nw == 8) go(sample_grids_v2_batch_kernel<2, 8>);
  else if (nw == 1) go(sample_grids_v2_batch_kernel<2, 1>);
  else go(sample_grids_v2_batch_kernel<2, 0>);
}

// shared memory of the box batch launch: the widest window of ncact tile columns anywhere in the map
// window-first sampling (solve(), api.cu), after the detecting rollout: CTA (0, 0) decides this solve's reach box from
// its reach statistic, as a reach-box solve would (record[0..4], as b200mppi_planner_sample_box reports it), counts the
// maps flagged in esc (record[5]) and clears `clear` (the other solve parity's flags); then every CTA whose maps include
// a flagged one re-walks its whole maps from the pre-call states (a: a whole-map plan on states_alt, no state stores)
// -- inside the sampled rectangle that rewrites the bytes already there.  No flag: every CTA returns after its check.
// [emu:begin window_complete]
template <int NW>
__global__ void __launch_bounds__(256) sample_window_complete_kernel(const SampleGridsV2Args a, const ReachBoxConst c,
                                                                     float x0x, float x0y, const float* __restrict__ reach,
                                                                     int* __restrict__ record,
                                                                     const unsigned char* __restrict__ esc,
                                                                     unsigned char* __restrict__ clear) {
  if (blockIdx.x == 0 && blockIdx.y == 0) {
    int flagged = 0;
    for (int i0 = 0; i0 < a.num_maps; i0 += blockDim.x)
      flagged += __syncthreads_count(i0 + (int)threadIdx.x < a.num_maps && esc[i0 + threadIdx.x]);
    for (int i = threadIdx.x; i < a.num_maps; i += blockDim.x) clear[i] = 0;
    if (threadIdx.x == 0) {
      const float r = *reach;
      ReachBox b;
      const int how = reach_box_decide(c, x0x, x0y, c.mode == 2 ? &r : nullptr, &b);
      record[0] = how;
      record[1] = how ? b.row_lo : 0; record[2] = how ? b.row_hi : a.rows;
      record[3] = how ? b.col_lo : 0; record[4] = how ? b.col_hi : a.cols;
      record[5] = flagged;
    }
  }
  bool any = false;
  for (int j = 0; j < a.gm; ++j) {
    const int m = (int)blockIdx.y * a.gm + j;
    any |= m < a.num_maps && esc[m] != 0;
  }
  if (!any) return;                                                  // CTA-uniform
  sample_grids_v2_body<2, NW>(a);
}
// [emu:end window_complete]

void launch_sample_window_complete(const SampleGridsV2Args& a, const ReachBoxConst& c, float x0x, float x0y,
                                   const float* reach, int* record, const unsigned char* esc, unsigned char* clear,
                                   cudaStream_t st) {
  const dim3 grid(a.tx * a.segs, (a.num_maps + a.gm - 1) / a.gm);
  const int threads = v2_threads(a);
  const size_t smem = sample_grids_v2_smem(a, 2);
  const int nw = a.t[0].bpad / 4;
  auto go = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, threads, smem, st>>>(a, c, x0x, x0y, reach, record, esc, clear);
  };
  if (nw == 3) go(sample_window_complete_kernel<3>);
  else if (nw == 8) go(sample_window_complete_kernel<8>);
  else if (nw == 1) go(sample_window_complete_kernel<1>);
  else go(sample_window_complete_kernel<0>);
}

// ---------------------------------------------------------------------------------------------
// Ground-truth realisations (b200mppi_tdm_draw_realisations): byte q of map 0 -> float64(((float)q * (hi - lo)) / 100
// + lo), the expression NumPy 2 evaluates for the reference notebook's sample_traction_grid (an int8 array with float32
// bounds stays float32), widened exactly.  Each operation is IEEE float32 rounded to nearest on its own -- no .ftz
// (the library is built with -ftz=true), no contraction -- so subnormal bounds convert as NumPy converts them.
// Plane blockIdx.y: p0 or p1; one thread per cell.
// [emu:begin realisation]
__device__ __forceinline__ float ieee_sub(float a, float b) {
#ifdef __CUDA_ARCH__
  float r; asm("sub.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
#else
  return a - b;
#endif
}
__device__ __forceinline__ float ieee_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  float r; asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
#else
  return a * b;
#endif
}
__device__ __forceinline__ float ieee_div(float a, float b) {
#ifdef __CUDA_ARCH__
  float r; asm("div.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
#else
  return a / b;
#endif
}
__device__ __forceinline__ float ieee_add(float a, float b) {
#ifdef __CUDA_ARCH__
  float r; asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
#else
  return a + b;
#endif
}
__device__ __forceinline__ double ieee_widen(float a) {
#ifdef __CUDA_ARCH__
  double r; asm("cvt.f64.f32 %0, %1;" : "=d"(r) : "f"(a)); return r;
#else
  return (double)a;
#endif
}
__global__ void __launch_bounds__(256) realisation_convert_kernel(const RealisationPlane p0, const RealisationPlane p1,
                                                                  int rows, int cols) {
  const bool second = blockIdx.y != 0;                              // field by field: no local copy of a plane
  const int8_t* grid = second ? p1.grid : p0.grid;
  const int pitch = second ? p1.pitch : p0.pitch;
  const float lo = second ? p1.lo : p0.lo, hi = second ? p1.hi : p0.hi;
  double* out = second ? p1.out : p0.out;
  const int64_t cell = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (cell >= (int64_t)rows * cols) return;
  const int r = (int)(cell / cols), c = (int)(cell % cols);
  const float q = (float)grid[(size_t)r * pitch + c];               // exact
  out[cell] = ieee_widen(ieee_add(ieee_div(ieee_mul(q, ieee_sub(hi, lo)), 100.0f), lo));
}
// [emu:end realisation]

void launch_realisation_convert(const RealisationPlane& p0, const RealisationPlane& p1, int planes, int rows, int cols,
                                cudaStream_t st) {
  const int64_t cells = (int64_t)rows * cols;
  realisation_convert_kernel<<<dim3((unsigned)((cells + 255) / 256), (unsigned)planes), 256, 0, st>>>(p0, p1, rows,
                                                                                                      cols);
}

static size_t box_batch_smem(const SampleGridsV2Args& geom, int ncact) {
  size_t smem = 0;
  for (int lo = 0; lo + ncact <= geom.ty; ++lo)
    smem = std::max(smem, sample_v2_smem_hd(lo, ncact, geom.ty, geom.cols, geom.t[0].bpad, geom.gm, 2));
  return smem;
}

bool sample_box_batch_fits(const SampleGridsV2Args& geom, int ncact) {
  return ncact >= 1 && ncact <= geom.ty && sample_v2_fits_hd(0, ncact, geom.ty, geom.cols, geom.t[0].bpad,
                                                             geom.t[1].bpad, geom.gm, 2) &&
         box_batch_smem(geom, ncact) <= 200 * 1024;
}

SampleClassLaunch sample_box_class_launch(const SampleGridsV2Args* const* members, int count, int mrows, int ncact) {
  SampleClassLaunch L{};
  L.nw = members[0]->t[0].bpad / 4;
  for (int i = 0; i < count; ++i) {
    const SampleGridsV2Args& a = *members[i];
    L.gx = std::max(L.gx, mrows * a.segs);
    L.gy = std::max(L.gy, (a.num_maps + a.gm - 1) / a.gm);
    L.gm = std::max(L.gm, a.gm);
    L.threads = std::max(L.threads, ((ncact * a.gm + 31) / 32) * 32);
    L.smem = std::max(L.smem, box_batch_smem(a, ncact));
  }
  return L;
}

void launch_sample_grids_v2_box_batch(const SampleClassLaunch& L, const SampleGridsV2Args* descs,
                                      const SampleBoxDesc* boxes, int count, const int* pairs, const int* active,
                                      int iter, int mrows, int ncact, cudaStream_t st, const SampleGroupDesc* groups,
                                      const int* members) {
  const dim3 grid(L.gx, L.gy, count);
  const int threads = L.threads;
  const size_t smem = L.smem;
  const int nw = L.nw;
  auto go = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, threads, smem, st>>>(descs, boxes, active, iter, mrows, ncact, pairs);
  };
  auto go_groups = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, threads, smem, st>>>(descs, boxes, groups, members, active, iter, mrows, ncact, pairs);
  };
  if (groups) {
    if (nw == 3) go_groups(sample_grids_v2_group_box_batch_kernel<3>);
    else if (nw == 8) go_groups(sample_grids_v2_group_box_batch_kernel<8>);
    else if (nw == 1) go_groups(sample_grids_v2_group_box_batch_kernel<1>);
    else go_groups(sample_grids_v2_group_box_batch_kernel<0>);
    return;
  }
  if (nw == 3) go(sample_grids_v2_box_batch_kernel<3>);
  else if (nw == 8) go(sample_grids_v2_box_batch_kernel<8>);
  else if (nw == 1) go(sample_grids_v2_box_batch_kernel<1>);
  else go(sample_grids_v2_box_batch_kernel<0>);
}

void launch_sample_grids_v2_complete_batch(const SampleClassLaunch& L, const SampleGridsV2Args* descs,
                                           const SampleBoxDesc* boxes, int count, const int* pairs, const int* active,
                                           int map_end, int mrows, int ncact, cudaStream_t st,
                                           const SampleGroupDesc* groups, const int* members) {
  const dim3 grid(L.gx, (map_end + L.gm - 1) / L.gm, count);
  const int threads = L.threads;
  const size_t smem = L.smem;
  const int nw = L.nw;
  auto go = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, threads, smem, st>>>(descs, boxes, active, map_end, mrows, ncact, pairs);
  };
  auto go_groups = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, threads, smem, st>>>(descs, groups, members, active, map_end, mrows, ncact, pairs);
  };
  if (groups) {
    if (nw == 3) go_groups(sample_grids_v2_group_complete_batch_kernel<3>);
    else if (nw == 8) go_groups(sample_grids_v2_group_complete_batch_kernel<8>);
    else if (nw == 1) go_groups(sample_grids_v2_group_complete_batch_kernel<1>);
    else go_groups(sample_grids_v2_group_complete_batch_kernel<0>);
    return;
  }
  if (nw == 3) go(sample_grids_v2_complete_batch_kernel<3>);
  else if (nw == 8) go(sample_grids_v2_complete_batch_kernel<8>);
  else if (nw == 1) go(sample_grids_v2_complete_batch_kernel<1>);
  else go(sample_grids_v2_complete_batch_kernel<0>);
}

void launch_advance_states_batch(const SampleGridsV2Args* descs, const SampleBoxDesc* boxes, int count, const int* pairs,
                                 int tx, int ty, int num_maps, const int* active, cudaStream_t st,
                                 const SampleGroupDesc* groups, const int* members) {
  const int64_t total = (int64_t)tx * ty * num_maps;
  const dim3 grid((unsigned)((total + 127) / 128), (unsigned)count);
  if (groups)
    advance_states_group_batch_kernel<<<grid, 128, 4 * 128 * 16, st>>>(descs, boxes, groups, members, active, 0, 0, tx,
                                                                        ty, num_maps, pairs);
  else
    advance_states_batch_kernel<<<grid, 128, 4 * 128 * 16, st>>>(descs, boxes, active, 0, 0, tx, ty, num_maps, pairs);
}

static inline void next_h(uint64_t& s0, uint64_t& s1);

// ---------------------------------------------------------------------------------------------
// Host: GF(2) transition matrices of xoroshiro128+ (columns as 2 x u64), A^K by square-and-multiply.
struct Gf2Mat { uint64_t c[128][2]; };

static void gf2_apply(const Gf2Mat& m, const uint64_t v[2], uint64_t out[2]) {
  uint64_t a0 = 0, a1 = 0;
  for (int w = 0; w < 2; ++w)
    for (int j = 0; j < 64; ++j)
      if ((v[w] >> j) & 1ULL) { a0 ^= m.c[64 * w + j][0]; a1 ^= m.c[64 * w + j][1]; }
  out[0] = a0; out[1] = a1;
}
static void gf2_mul(const Gf2Mat& a, const Gf2Mat& b, Gf2Mat& out) {      // out = a * b (apply b, then a)
  for (int j = 0; j < 128; ++j) gf2_apply(a, b.c[j], out.c[j]);
}
static void gf2_step_matrix(Gf2Mat& m) {
  for (int j = 0; j < 128; ++j) {
    uint64_t s0 = j < 64 ? (1ULL << j) : 0, s1 = j >= 64 ? (1ULL << (j - 64)) : 0;
    next_h(s0, s1);
    m.c[j][0] = s0; m.c[j][1] = s1;
  }
}
// out: [count][128][2] u64, matrix i advances a state by ks[i] draws
void build_jump_matrices(const int64_t* ks, int count, uint64_t* out) {
  Gf2Mat step;
  gf2_step_matrix(step);
  for (int i = 0; i < count; ++i) {
    Gf2Mat acc, base = step, tmp;
    for (int j = 0; j < 128; ++j) {                      // identity
      acc.c[j][0] = j < 64 ? (1ULL << j) : 0; acc.c[j][1] = j >= 64 ? (1ULL << (j - 64)) : 0;
    }
    for (uint64_t k = (uint64_t)ks[i]; k; k >>= 1) {
      if (k & 1ULL) { gf2_mul(base, acc, tmp); acc = tmp; }
      gf2_mul(base, base, tmp); base = tmp;
    }
    std::memcpy(out + (size_t)i * 256, acc.c, sizeof(acc.c));
  }
}

// out: [(segs-1)*2][128][2] u64, matrix (s-1)*2 + c advances a state by s*k[c] draws (c = 0, 1), s = 1 .. segs-1:
// the segment-start jumps of the sampler, built with one product per matrix (A^(s k) = A^k * A^((s-1) k)).
void build_jump_series(int64_t k0, int64_t k1, int segs, uint64_t* out) {
  if (segs < 2) return;
  const int64_t ks[2] = {k0, k1};
  std::vector<uint64_t> b(2 * 256);
  build_jump_matrices(ks, 2, b.data());
  Gf2Mat base[2], acc[2], tmp;
  for (int c = 0; c < 2; ++c) { std::memcpy(base[c].c, b.data() + (size_t)c * 256, sizeof(base[c].c)); acc[c] = base[c]; }
  for (int sgm = 1; sgm < segs; ++sgm)
    for (int c = 0; c < 2; ++c) {
      std::memcpy(out + ((size_t)(sgm - 1) * 2 + c) * 256, acc[c].c, sizeof(acc[c].c));
      gf2_mul(base[c], acc[c], tmp);
      acc[c] = tmp;
    }
}

// Host: breakpoints of q(v) = int8(ceil(f64(f32(v * 2^-53)) * 100.0 * alpha)) (terrain.py:682-683 as
// compiled: cvt.rn.f64.u64, mul.f64 2^-53, cvt.rn.f32.f64, cvt.f64.f32, mul.f64 100, mul.f64 alpha,
// cvt.rpi.f64, cvt.rzi.s16 -> low byte).  Returns false if q is not a monotone map into [0, q_cap]
// or if the integer estimate used by the kernel cannot be proven tight.
static inline int q_of_v(uint64_t v, double alpha) {
  const float u = (float)((double)v * (1.0 / 9007199254740992.0));
  volatile double t = (double)u * 100.0;
  volatile double t2 = t * alpha;
  const double c = std::ceil(t2);
  if (!(c > -32768.0 && c < 32767.0)) return 1 << 20;
  return (int)(int8_t)(int16_t)c;
}

bool build_sample_thresholds(double alpha, int q_cap, uint64_t* B /*[SAMPLE_TABLE_WORDS]*/) {
  if (!(alpha >= 0.0) || !(alpha * 100.0 <= 127.0)) return false;
  const uint64_t VMAX = (1ULL << 53) - 1;
  const int qmax = q_of_v(VMAX, alpha);
  if (qmax < 0 || qmax > q_cap || qmax > 127 || q_of_v(0, alpha) != 0) return false;
  std::vector<uint64_t> T((size_t)qmax + 2, ~0ULL);
  T[0] = 0;
  for (int k = 1; k <= qmax; ++k) {                   // smallest v with q(v) >= k (q monotone in v)
    uint64_t lo = 0, hi = VMAX;                       // q(lo) < k <= q(hi)
    while (hi - lo > 1) {
      const uint64_t mid = lo + (hi - lo) / 2;
      if (q_of_v(mid, alpha) >= k) hi = mid; else lo = mid;
    }
    T[k] = hi;
  }
  // bucket b covers the 53-bit draws v in [b << 45, (b+1) << 45), i.e. the RAW draws r = v << 11 | (11 low bits) in
  // [b << 56, (b+1) << 56): v >= T[k]  <=>  r >= T[k] << 11.  Valid iff at most one breakpoint lies strictly inside
  // each bucket and it raises q by exactly one.  No breakpoint inside: thr = 0 ("r >= thr" always true), qbase = q-1.
  // The entry is thr | qbase (sample_threshold_q): thr has its low 11 bits clear, qbase <= 127.
  for (int b = 0; b < 256; ++b) {
    const uint64_t start = (uint64_t)b << 45, end = start + (1ULL << 45);
    const int qb = q_of_v(start, alpha);
    uint64_t next = 0;
    int inside = 0;
    for (int k = 1; k <= qmax; ++k)
      if (T[k] > start && T[k] < end) { if (!inside) next = T[k]; ++inside; }
    if (inside > 1 || qb < 0 || qb > 127) return false;
    if (inside == 1) {
      if (q_of_v(next, alpha) != qb + 1) return false;
      B[b] = (next << 11) | (uint64_t)qb;
    } else if (qb > 0) {
      B[b] = (uint64_t)(qb - 1);
    } else {
      // q = 0 over a whole bucket: only v = 0 has q = 0 for alpha > 0 (bucket 0 then holds the breakpoint v = 1),
      // so this is alpha = 0; "never" needs thr > every r of the bucket (the next bucket's start), which bucket 255
      // cannot offer
      if (b == 255) return false;
      B[b] = (uint64_t)(b + 1) << 56;
    }
  }
  return true;
}

// ---------------------------------------------------------------------------------------------
// Host: numba-compatible generator states.  State 0 = splitmix64(seed) in both words; state i is
// state i-1 jumped 2^64 steps (random.py:47-69,103-126,226-241).
static inline uint64_t rotl_h(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
static inline void next_h(uint64_t& s0, uint64_t& s1) {
  uint64_t t = s1 ^ s0;
  s0 = rotl_h(s0, 55) ^ t ^ (t << 14);
  s1 = rotl_h(t, 36);
}
static inline void jump_h(uint64_t& s0, uint64_t& s1) {
  static const uint64_t JUMP[2] = {0xbeac0467eba5facbULL, 0xd86b048b86aa9922ULL};
  uint64_t a0 = 0, a1 = 0;
  for (int i = 0; i < 2; ++i)
    for (int b = 0; b < 64; ++b) {
      if (JUMP[i] & (1ULL << b)) { a0 ^= s0; a1 ^= s1; }
      next_h(s0, s1);
    }
  s0 = a0; s1 = a1;
}

void create_xoroshiro_states(uint64_t* out, int64_t first, int64_t count, uint64_t seed) {
  uint64_t z = seed + 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  z = z ^ (z >> 31);
  uint64_t s0 = z, s1 = z;
  for (int64_t i = 0; i < first; ++i) jump_h(s0, s1);
  for (int64_t i = 0; i < count; ++i) {
    out[2 * i] = s0; out[2 * i + 1] = s1;
    jump_h(s0, s1);
  }
}

}  // namespace b200
