// Which SM resource is shared between SMs?  One CTA (one SM busy) against one CTA per SM (all SMs busy) of the same
// per-thread loop of ONE instruction type: if the per-SM rate drops when the neighbours work, the unit is shared.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/pair_probe tools/pair_probe.cu && /tmp/pair_probe
#include <cstdio>
#include <cuda_runtime.h>

static int g_sms = 0;   // SMs of device 0 (main)

template <int OP>
__global__ void __launch_bounds__(1024) probe(float* out, int iters, float seed) {
  float a0 = seed + threadIdx.x * 1e-3f, a1 = a0 + 1.f, a2 = a0 + 2.f, a3 = a0 + 3.f;
  double d0 = a0, d1 = a1, d2 = a2, d3 = a3;
  for (int i = 0; i < iters; ++i) {
    if (OP == 0) {        // MUFU.SIN
      asm volatile("sin.approx.ftz.f32 %0, %0;" : "+f"(a0)); asm volatile("sin.approx.ftz.f32 %0, %0;" : "+f"(a1));
      asm volatile("sin.approx.ftz.f32 %0, %0;" : "+f"(a2)); asm volatile("sin.approx.ftz.f32 %0, %0;" : "+f"(a3));
    } else if (OP == 1) { // F2F.F64.F32 + F2F.F32.F64 round trip
      asm volatile("cvt.f64.f32 %0, %1;" : "=d"(d0) : "f"(a0)); asm volatile("cvt.rn.f32.f64 %0, %1;" : "=f"(a0) : "d"(d0));
      asm volatile("cvt.f64.f32 %0, %1;" : "=d"(d1) : "f"(a1)); asm volatile("cvt.rn.f32.f64 %0, %1;" : "=f"(a1) : "d"(d1));
    } else if (OP == 2) { // DFMA
      asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d0) : "d"(d1), "d"(d2)); asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d3) : "d"(d1), "d"(d2));
      asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d1) : "d"(d2), "d"(d3)); asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d2) : "d"(d3), "d"(d0));
    } else if (OP == 3) { // FFMA
      asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(a0) : "f"(a1), "f"(a2)); asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(a3) : "f"(a1), "f"(a2));
      asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(a1) : "f"(a2), "f"(a3)); asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(a2) : "f"(a3), "f"(a0));
    } else if (OP == 4) { // integer LOP3 / IADD mix
      unsigned u0 = __float_as_uint(a0), u1 = __float_as_uint(a1);
      asm volatile("add.u32 %0, %0, %1;" : "+r"(u0) : "r"(u1)); asm volatile("xor.b32 %0, %0, %1;" : "+r"(u1) : "r"(u0));
      asm volatile("add.u32 %0, %0, %1;" : "+r"(u0) : "r"(u1)); asm volatile("xor.b32 %0, %0, %1;" : "+r"(u1) : "r"(u0));
      a0 = __uint_as_float(u0); a1 = __uint_as_float(u1);
    } else if (OP == 5) { // MUFU.SQRT
      asm volatile("sqrt.approx.ftz.f32 %0, %0;" : "+f"(a0)); asm volatile("sqrt.approx.ftz.f32 %0, %0;" : "+f"(a1));
      asm volatile("sqrt.approx.ftz.f32 %0, %0;" : "+f"(a2)); asm volatile("sqrt.approx.ftz.f32 %0, %0;" : "+f"(a3));
    }
  }
  if (a0 + a1 + a2 + a3 + (float)(d0 + d1 + d2 + d3) == 12345.678f) out[0] = a0;
}

// L2-resident stream: every thread loads 16 B per iteration, coalesced (512 B per warp), from an 8 MB buffer, with
// `pad` FFMA per load in between (the rollout kernel's mix of streamed controls and arithmetic)
template <int PAD>
__global__ void __launch_bounds__(1024) stream(const double2* __restrict__ src, float* out, int iters, int words) {
  const int gt = blockIdx.x * 1024 + threadIdx.x;
  double acc = 0.0; float f = threadIdx.x;
  int idx = gt % words;
  for (int i = 0; i < iters; ++i) {
    const double2 v = __ldg(src + idx);
    idx += 8192; if (idx >= words) idx -= words;
    acc += v.x + v.y;
#pragma unroll
    for (int k = 0; k < PAD; ++k) asm volatile("fma.rn.f32 %0, %0, %0, %0;" : "+f"(f));
  }
  if (acc + f == 12345.678) out[0] = (float)acc;
}

// the same stream in the rollout kernel's setting: one 1024-thread CTA per SM holding 222 KB of shared memory (what is
// left of the 256 KB is the L1), 4 byte loads from shared memory per iteration; per-CTA durations by globaltimer
template <int PAD>
__global__ void __launch_bounds__(1024) stream_smem(const double2* __restrict__ src, float* out, int iters, int words, int bcast,
                                                    long long* dur) {
  extern __shared__ signed char win[];
  const int gt = blockIdx.x * 1024 + threadIdx.x;
  for (int i = threadIdx.x; i < 222 * 1024; i += 1024) win[i] = (signed char)i;
  __syncthreads();
  long long t0 = 0;
  if (threadIdx.x == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  double acc = 0.0; float f = threadIdx.x;
  int idx = (bcast ? (gt & ~31) : gt) % words;
  unsigned h = gt * 2654435761u;
  for (int i = 0; i < iters; ++i) {
    const double2 v = __ldg(src + idx);
    idx += 8192; if (idx >= words) idx -= words;
    h = h * 1664525u + 1013904223u;
    const int a0 = (h >> 8) % (55 * 1024);
    acc += v.x + v.y + win[a0] + win[a0 + 55 * 1024] + win[a0 + 110 * 1024] + win[a0 + 165 * 1024];
#pragma unroll
    for (int k = 0; k < PAD; ++k) asm volatile("fma.rn.f32 %0, %0, %0, %0;" : "+f"(f));
  }
  if (acc + f == 12345.678) out[0] = (float)acc;
  __syncthreads();
  if (threadIdx.x == 0) { long long t1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); dur[blockIdx.x] = t1 - t0; }
}

#include <algorithm>
#include <vector>
template <int PAD>
void run_stream_smem(const char* name, int iters, int bcast) {
  const int words = 1 << 20;                                        // 16 MB of double2
  double2* src; cudaMalloc(&src, (size_t)words * 16); cudaMemset(src, 0, (size_t)words * 16);
  float* out; cudaMalloc(&out, 4);
  long long* dur; cudaMalloc(&dur, g_sms * 8);
  cudaFuncSetAttribute(stream_smem<PAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, 222 * 1024);
  const int grids[2] = {1, g_sms};
  printf("%-34s", name);
  for (int k = 0; k < 2; ++k) {
    stream_smem<PAD><<<grids[k], 1024, 222 * 1024>>>(src, out, iters, words, bcast, dur);
    stream_smem<PAD><<<grids[k], 1024, 222 * 1024>>>(src, out, iters, words, bcast, dur);
    cudaDeviceSynchronize();
    std::vector<long long> d(grids[k]);
    cudaMemcpy(d.data(), dur, grids[k] * 8, cudaMemcpyDeviceToHost);
    std::sort(d.begin(), d.end());
    printf(" | %3d CTAs: per-CTA us min %.1f  p25 %.1f  median %.1f  p75 %.1f  max %.1f", grids[k], d[0] / 1e3, d[d.size() / 4] / 1e3,
           d[d.size() / 2] / 1e3, d[d.size() * 3 / 4] / 1e3, d.back() / 1e3);
  }
  printf("\n");
  cudaFree(src); cudaFree(out); cudaFree(dur);
}

template <int PAD>
void run_stream(const char* name, int iters) {
  const int words = 8 << 16;                                        // 8 MB of double2
  double2* src; cudaMalloc(&src, (size_t)words * 16); cudaMemset(src, 0, (size_t)words * 16);
  float* out; cudaMalloc(&out, 4);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float ms[3];
  const int grids[3] = {1, g_sms / 2, g_sms};
  for (int k = 0; k < 3; ++k) {
    stream<PAD><<<grids[k], 1024>>>(src, out, iters, words);
    cudaEventRecord(e0);
    stream<PAD><<<grids[k], 1024>>>(src, out, iters, words);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms[k], e0, e1);
  }
  const double gb = 1024.0 * 16 * iters / 1e6;                      // MB per CTA
  printf("%-28s 1 CTA %.3f ms (%.0f GB/s/SM) | %d CTAs %.3f ms (x%.2f) | %d CTAs %.3f ms (x%.2f, %.0f GB/s/SM, %.2f TB/s)\n", name, ms[0],
         gb / ms[0], grids[1], ms[1], ms[1] / ms[0], grids[2], ms[2], ms[2] / ms[0], gb / ms[2], gb * g_sms / ms[2] / 1e3);
  cudaFree(src); cudaFree(out);
}

template <int OP>
void run(const char* name, int iters) {
  float* out; cudaMalloc(&out, 4);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float ms[3];
  const int grids[3] = {1, g_sms / 2, g_sms};
  for (int k = 0; k < 3; ++k) {
    probe<OP><<<grids[k], 1024>>>(out, iters, 1.0f);            // warm-up
    cudaEventRecord(e0);
    probe<OP><<<grids[k], 1024>>>(out, iters, 1.0f);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms[k], e0, e1);
  }
  printf("%-28s 1 CTA %.3f ms | %d CTAs %.3f ms (x%.2f) | %d CTAs %.3f ms (x%.2f)\n", name, ms[0], grids[1], ms[1], ms[1] / ms[0], grids[2],
         ms[2], ms[2] / ms[0]);
  cudaFree(out);
}

int main() {
  cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0);
  const int it = 20000;
  run<3>("FFMA", it);
  run<4>("IADD/LOP3", it);
  run<0>("MUFU.SIN", it);
  run<5>("MUFU.SQRT", it);
  run<1>("F2F f32<->f64 round trip", it);
  run<2>("DFMA", it);
  run_stream<0>("L2 stream 16 B/thread", 4000);
  run_stream<16>("L2 stream + 16 FFMA", 4000);
  run_stream<32>("L2 stream + 32 FFMA", 4000);
  run_stream<64>("L2 stream + 64 FFMA", 4000);
  run_stream_smem<32>("222KB smem, stream + 32 FFMA", 2000, 0);
  run_stream_smem<64>("222KB smem, stream + 64 FFMA", 2000, 0);
  run_stream_smem<64>("222KB smem, bcast  + 64 FFMA", 2000, 1);
  return 0;
}
