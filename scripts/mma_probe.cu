// Issue-rate / latency probe for the legacy warp-level tensor instructions on sm_90a:
// HMMA.16816.F32 (fp16) vs IMMA.16832.U8.S8 (int8), plus the LOP3 rate, as a function of resident warps per SM
// and independent accumulator chains per warp.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o mma_probe mma_probe.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ void hmma(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void imma(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

template <int CH, int MODE>  // MODE 0 = HMMA, 1 = IMMA, 2 = HMMA + 5 ALU ops per mma (W4 fp16 unpack), 3 = IMMA + 4 LOP3 per mma
__global__ void probe(int iters, long long* cyc, float* sink, uint32_t seed) {
  float cf[CH][4];
  int ci[CH][4];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int i = 0; i < 4; ++i) cf[c][i] = 0.f, ci[c][i] = 0;
  uint32_t w0 = seed + threadIdx.x, w1 = seed * 3 + threadIdx.x, w2 = seed * 5, w3 = seed * 7, b0 = seed * 11, b1 = seed * 13;
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if (MODE == 0) hmma(cf[c], w0, w1, w2, w3, b0, b1);
      if (MODE == 1) imma(ci[c], w0, w1, w2, w3, b0, b1);
      if (MODE == 2) {
        const uint32_t s0 = w0 >> 8, s1 = w1 >> 8;  // 2 SHF + 4 LOP3 per HMMA is the current W4 cost (5 per HMMA on average)
        hmma(cf[c], w0 & 0x000f000fu, w1 & 0x000f000fu, s0 & 0x000f000fu, s1 & 0x000f000fu, b0, b1);
        w0 += 0x01010101u, w1 ^= s0;  // keep the unpack from being hoisted
      }
      if (MODE == 3) {
        imma(ci[c], w0 & 0x0f0f0f0fu, w1 & 0x0f0f0f0fu, w2 & 0x0f0f0f0fu, w3 & 0x0f0f0f0fu, b0, b1);
        w0 += 0x01010101u, w1 += 0x01010101u, w2 += 0x01010101u, w3 += 0x01010101u;
      }
    }
  }
  const long long t1 = clock64();
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int i = 0; i < 4; ++i) s += cf[c][i] + (float)ci[c][i];
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
  if (s == 123.456f) sink[0] = s;
}

template <int CH, int MODE>
static void run(const char* name, int warps, long long* d_cyc, float* d_sink) {
  const int iters = 4096;
  probe<CH, MODE><<<148, warps * 32>>>(iters, d_cyc, d_sink, 1);
  probe<CH, MODE><<<148, warps * 32>>>(iters, d_cyc, d_sink, 2);
  cudaDeviceSynchronize();
  long long h[148];
  cudaMemcpy(h, d_cyc, sizeof(h), cudaMemcpyDeviceToHost);
  double avg = 0;
  for (int i = 0; i < 148; ++i) avg += (double)h[i];
  avg /= 148;
  const double per_warp = avg / ((double)iters * CH);         // cycles between mma issues of one warp
  const double per_smsp = per_warp / ((warps + 3) / 4);         // cycles per mma per scheduler
  printf("%-28s warps/SM=%2d chains=%d  cycles/mma/warp=%7.2f  cycles/mma/SMSP=%6.2f\n", name, warps, CH, per_warp, per_smsp);
}

int main() {
  long long* d_cyc;
  float* d_sink;
  cudaMalloc(&d_cyc, 148 * sizeof(long long));
  cudaMalloc(&d_sink, 4);
  for (int warps : {1, 4, 8, 16}) {
    run<1, 0>("HMMA.16816.F32 dependent", warps, d_cyc, d_sink);
    run<4, 0>("HMMA.16816.F32 4 chains", warps, d_cyc, d_sink);
    run<1, 1>("IMMA.16832.U8.S8 dependent", warps, d_cyc, d_sink);
    run<4, 1>("IMMA.16832.U8.S8 4 chains", warps, d_cyc, d_sink);
    run<4, 2>("HMMA + W4 fp16 unpack", warps, d_cyc, d_sink);
    run<4, 3>("IMMA + W4 int8 unpack", warps, d_cyc, d_sink);
  }
  cudaError_t e = cudaGetLastError();
  printf("status: %s\n", cudaGetErrorString(e));
  return 0;
}
