// Standalone HBM streaming probe for sm_90a: how fast can one CTA per SM (or more) pull a big buffer
// through (a) a cp.async.bulk + mbarrier ring with a trivial consumer, (b) plain 128-bit LDG loops?
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o stream_probe scripts/stream_probe.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t par) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(b)), "r"(par) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void bulk(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// mode 0: ring. warp 0 = producers (np lanes, lane l handles slots l, l+np, ...), warps 1..nc = consumers:
// every consumer warp waits full, (optionally reads 16B per lane), arrives empty.
__global__ void ring_kernel(const uint8_t* __restrict__ src, size_t bytes_per_cta, int slot_bytes, int stages, int np,
                            int nc, int touch, unsigned long long* sink, int tile_slots) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* full = (uint64_t*)(smem + (size_t)stages * slot_bytes);
  uint64_t* empty = full + stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], nc); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint8_t* base = src + (size_t)blockIdx.x * bytes_per_cta;
  const int n_slots = (int)(bytes_per_cta / slot_bytes);
  // tile_slots > 0: GEMV-like interleaving -- this CTA's i-th slot belongs to tile (i / tile_slots) * gridDim.x + blockIdx.x
  auto slot_ptr = [&](int i) -> const uint8_t* {
    if (tile_slots <= 0) return base + (size_t)i * slot_bytes;
    const size_t tile = (size_t)(i / tile_slots) * gridDim.x + blockIdx.x;
    return src + (tile * tile_slots + (i % tile_slots)) * (size_t)slot_bytes;
  };
  if (warp == 0) {
    if (lane < np) {
      for (int i = lane; i < n_slots; i += np) {
        const int stage = i % stages;
        const uint32_t par = (i / stages) & 1;
        mbar_wait(&empty[stage], par ^ 1);
        mbar_expect(&full[stage], slot_bytes);
        bulk(smem + (size_t)stage * slot_bytes, slot_ptr(i), slot_bytes, &full[stage]);
      }
    }
  } else {
    unsigned long long acc = 0;
    for (int i = 0; i < n_slots; ++i) {
      const int stage = i % stages;
      const uint32_t par = (i / stages) & 1;
      mbar_wait(&full[stage], par);
      if (touch) {
        const uint4* p = (const uint4*)(smem + (size_t)stage * slot_bytes);
        for (int j = (warp - 1) * 32 + lane; j < slot_bytes / 16; j += nc * 32) { uint4 v = p[j]; acc += v.x ^ v.y ^ v.z ^ v.w; }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
    }
    if (acc == 0x123456789ull) *sink = acc;
  }
}

// mode 1: LDG.128 streaming, U loads in flight per thread
template <int U>
__global__ void ldg_kernel(const uint4* __restrict__ src, size_t vec_per_cta, unsigned long long* sink) {
  const uint4* base = src + (size_t)blockIdx.x * vec_per_cta;
  unsigned long long acc = 0;
  for (size_t i = threadIdx.x; i + (size_t)(U - 1) * blockDim.x < vec_per_cta; i += (size_t)U * blockDim.x) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v[u].x), "=r"(v[u].y), "=r"(v[u].z), "=r"(v[u].w) : "l"(base + i + (size_t)u * blockDim.x));
#pragma unroll
    for (int u = 0; u < U; ++u) acc += v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
  }
  if (acc == 0x123456789ull) *sink = acc;
}

static float time_it(void (*launch)(void*), void* ctx, int reps) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  launch(ctx); cudaDeviceSynchronize();
  cudaEventRecord(a);
  for (int i = 0; i < reps; ++i) launch(ctx);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  return ms / reps;
}

struct RingCfg { const uint8_t* src; size_t per_cta; int slot, stages, np, nc, touch, grid; unsigned long long* sink; int tile_slots; };
static void launch_ring(void* c) {
  RingCfg* r = (RingCfg*)c;
  size_t smem = (size_t)r->stages * r->slot + r->stages * 16;
  cudaFuncSetAttribute(ring_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  ring_kernel<<<r->grid, 32 * (1 + r->nc), smem>>>(r->src, r->per_cta, r->slot, r->stages, r->np, r->nc, r->touch, r->sink, r->tile_slots);
}
struct LdgCfg { const uint4* src; size_t vec_per_cta; int grid, threads, U; unsigned long long* sink; };
static void launch_ldg(void* c) {
  LdgCfg* r = (LdgCfg*)c;
  if (r->U == 4) ldg_kernel<4><<<r->grid, r->threads>>>(r->src, r->vec_per_cta, r->sink);
  else if (r->U == 8) ldg_kernel<8><<<r->grid, r->threads>>>(r->src, r->vec_per_cta, r->sink);
  else ldg_kernel<2><<<r->grid, r->threads>>>(r->src, r->vec_per_cta, r->sink);
}

int main() {
  setvbuf(stdout, NULL, _IONBF, 0);
  const size_t total = (size_t)148 * 2 * 1024 * 1024 * 4;  // 1184 MiB >> L2
  uint8_t* buf = nullptr;
  cudaError_t e0 = cudaMalloc(&buf, total);
  printf("malloc: %s\n", cudaGetErrorString(e0));
  cudaMemset(buf, 1, total);
  unsigned long long* sink; cudaMalloc(&sink, 8);
  int sms = 148;
  printf("mode      grid slotKB stages np nc touch   ms    GB/s\n");
  // contiguous vs GEMV-like tile-interleaved streams; short (25 MB) vs long (1.2 GB) kernels
  size_t sizes[] = {total, (size_t)25 << 20, (size_t)45 << 20, (size_t)8 << 20};
  for (int zi = 0; zi < 4; ++zi)
    for (int ts = 0; ts <= 2; ts += 2)
      for (int nc = 2; nc <= 16; nc *= 4) {
        int slot = 16384, stages = 8;
        RingCfg c{buf, sizes[zi] / sms / slot * slot, slot, stages, 1, nc, 0, sms, sink, ts};
        float ms = time_it(launch_ring, &c, 20);
        double gb = (double)c.per_cta * c.grid / ms / 1e6;
        printf("ring %s total=%4zuMB nc=%2d  %8.4f ms %7.0f GB/s\n", ts ? "tile-interleaved" : "contiguous      ", sizes[zi] >> 20, nc, ms, gb);
      }
  int threads[] = {256, 512, 1024};
  int Us[] = {2, 4, 8};
  for (int mult = 1; mult <= 1; mult *= 2)
    for (int ti = 2; ti < 3; ++ti)
      for (int ui = 1; ui < 2; ++ui) {
        LdgCfg c{(const uint4*)buf, total / 16 / (sms * mult), sms * mult, threads[ti], Us[ui], sink};
        float ms = time_it(launch_ldg, &c, 5);
        printf("ldg       %4d thr=%4d U=%d            %7.3f %7.0f\n", c.grid, c.threads, c.U, ms, (double)c.vec_per_cta * 16 * c.grid / ms / 1e6);
      }
  cudaError_t e = cudaDeviceSynchronize();
  printf("status: %s\n", cudaGetErrorString(e));
  return 0;
}
