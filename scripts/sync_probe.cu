// Dependency hand-off cost probe (sm_90a): how long does one "every CTA needs what every CTA just wrote" step take
//   (a) as a kernel boundary (plain stream order / programmatic dependent launch, inside a CUDA graph),
//   (b) as a software grid barrier inside one persistent kernel (148 CTAs), idle and while the SMs stream HBM.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o sync_probe sync_probe.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e_), __LINE__); return 1; } } while (0)

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// (a) one link of a kernel chain: every CTA reads the whole vector the previous link wrote (8 KB) and writes its slice
__global__ void link(const float* __restrict__ in, float* __restrict__ out, int n, int pdl) {
  if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += __ldcg(in + i);
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  __shared__ float ws[32];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += ws[w];
    const int per = n / gridDim.x;
    for (int i = 0; i < per; ++i) out[blockIdx.x * per + i] = t * 1e-3f + 1.f;
  }
}

// (b) persistent kernel: `rounds` times { every CTA writes its slice; grid barrier; every CTA reads the whole vector }
// mode 0: __threadfence + atomicAdd, poll ld.acquire     mode 1: red.release, poll ld.acquire
// mode 2: red.release, poll ld.relaxed then one fence.acquire
// load_warps > 0: that many extra warps per CTA stream `bg` (uint4 loads) until the barrier work is done
__global__ void persistent(float* buf0, float* buf1, int n, unsigned* ctr, int rounds, int mode, const uint4* bg,
                           size_t bg_vec, int load_warps, unsigned* stop, unsigned long long* t_out, unsigned* sink) {
  const int nbar = blockDim.x - load_warps * 32;  // threads doing the barrier work
  __shared__ float ws[32];
  if ((int)threadIdx.x >= nbar) {
    // background HBM stream
    const size_t stride = (size_t)gridDim.x * load_warps * 32;
    size_t i = (size_t)blockIdx.x * load_warps * 32 + (threadIdx.x - nbar);
    unsigned acc = 0;
    while (ld_relaxed(stop + 1) < gridDim.x) {
#pragma unroll 8
      for (int u = 0; u < 8; ++u) {
        const uint4 v = __ldcs(bg + i);
        acc ^= v.x ^ v.y ^ v.z ^ v.w;
        i += stride;
        if (i >= bg_vec) i -= bg_vec;
      }
    }
    if (acc == 0x12345678u) sink[0] = acc;
    return;
  }
  unsigned long long t0 = 0;
  if (threadIdx.x == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  float* in = buf0;
  float* out = buf1;
  const int per = n / gridDim.x;
  for (int r = 0; r < rounds; ++r) {
    // "compute": read the whole vector (written by all CTAs in the previous round)
    float s = 0.f;
    for (int i = threadIdx.x; i < n; i += nbar) s += __ldcg(in + i);
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
    asm volatile("bar.sync 1, %0;" ::"r"(nbar) : "memory");
    if (threadIdx.x < per) out[blockIdx.x * per + threadIdx.x] = ws[0] * 1e-3f + 1.f;
    asm volatile("bar.sync 1, %0;" ::"r"(nbar) : "memory");
    if (threadIdx.x == 0) {
      const unsigned target = (unsigned)(r + 1) * gridDim.x;
      if (mode == 0) {
        __threadfence();
        atomicAdd(ctr, 1u);
        while (ld_acquire(ctr) < target) {
        }
      } else if (mode == 1) {
        red_release(ctr, 1u);
        while (ld_acquire(ctr) < target) {
        }
      } else {
        red_release(ctr, 1u);
        while (ld_relaxed(ctr) < target) {
        }
        asm volatile("fence.acquire.gpu;" ::: "memory");
      }
    }
    asm volatile("bar.sync 1, %0;" ::"r"(nbar) : "memory");
    float* t = in;
    in = out;
    out = t;
  }
  if (threadIdx.x == 0) {
    unsigned long long t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    t_out[blockIdx.x] = t1 - t0;
    if (load_warps) atomicAdd(stop + 1, 1u);
  }
}

int main() {
  const int n = 4096 + 48;  // divisible by 148: 4144 = 148 * 28
  float *a, *b;
  CK(cudaMalloc(&a, n * 4));
  CK(cudaMalloc(&b, n * 4));
  CK(cudaMemset(a, 0, n * 4));
  CK(cudaMemset(b, 0, n * 4));
  cudaStream_t st;
  CK(cudaStreamCreate(&st));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  const int links = 400;
  for (int threads : {128, 512}) {
    for (int pdl = 0; pdl < 2; ++pdl) {
      cudaGraph_t g;
      cudaGraphExec_t ge;
      CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeGlobal));
      for (int i = 0; i < links; ++i) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(148);
        cfg.blockDim = dim3(threads);
        cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at;
        cfg.numAttrs = pdl;
        CK(cudaLaunchKernelEx(&cfg, link, (const float*)((i & 1) ? b : a), (i & 1) ? a : b, n, pdl));
      }
      CK(cudaStreamEndCapture(st, &g));
      CK(cudaGraphInstantiate(&ge, g, 0));
      for (int w = 0; w < 3; ++w) CK(cudaGraphLaunch(ge, st));
      CK(cudaEventRecord(e0, st));
      for (int w = 0; w < 5; ++w) CK(cudaGraphLaunch(ge, st));
      CK(cudaEventRecord(e1, st));
      CK(cudaStreamSynchronize(st));
      float ms;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("kernel chain  threads=%3d pdl=%d : %.3f us per dependent link (graph, 148 CTAs, 16 KB read each)\n", threads, pdl,
             ms * 1000.f / (5 * links));
    }
  }
  // persistent kernel
  unsigned* ctr;
  unsigned long long* t_out;
  unsigned* sink;
  CK(cudaMalloc(&ctr, 64));
  CK(cudaMalloc(&t_out, 148 * 8));
  CK(cudaMalloc(&sink, 4));
  const size_t bg_bytes = (size_t)4 << 30;
  uint4* bg;
  CK(cudaMalloc(&bg, bg_bytes));
  CK(cudaMemset(bg, 1, bg_bytes));
  const int rounds = 2000;
  for (int load_warps : {0, 8}) {
    for (int mode = 0; mode < 3; ++mode) {
      for (int nbar : {128, 512}) {
        CK(cudaMemset(ctr, 0, 64));
        const int threads = nbar + load_warps * 32;
        CK(cudaEventRecord(e0, st));
        persistent<<<148, threads, 0, st>>>(a, b, n, ctr, rounds, mode, bg, bg_bytes / 16, load_warps, ctr + 8, t_out, sink);
        CK(cudaEventRecord(e1, st));
        CK(cudaStreamSynchronize(st));
        std::vector<unsigned long long> h(148);
        CK(cudaMemcpy(h.data(), t_out, 148 * 8, cudaMemcpyDeviceToHost));
        unsigned long long mx = 0;
        for (auto v : h) mx = v > mx ? v : mx;
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        printf("grid barrier  mode=%d threads=%3d bg_load_warps=%d : %.3f us per round (write slice + barrier + read 16 KB)%s\n", mode,
               nbar, load_warps, (double)mx / 1000.0 / rounds, load_warps ? "  [under HBM streaming]" : "");
      }
    }
  }
  printf("status: %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
