// W4A16 prefill GEMM on the Hopper tensor cores (wgmma, fp32 accumulators in registers) and the elementwise kernels
// around it; replaces F.linear at M = prompt tokens (accessory/util/quant.py:18-46, llama.py:276-288) for prompts longer
// than one 32-token chunk of the decode GEMV.
//
// GEMM:   out[T, N] = x[T, K] . w_hat[N, K]^T
//   w_hat = fp16(fp16(q - z) * s16)  -- the reference's fake-quantised weight, reproduced bit for bit, so the prefill
//   logits follow F.linear(x, w_hat) with fp32 accumulation (accessory/util/quant.py:18-46 + SURVEY.md 8c).
//
// One CTA owns 128 output rows (eight 16-row tiles of the packed decode format, DESIGN.md section 3) and up to 256
// tokens.  D[rows x tokens] = A . B^T with A = dequantised weights (wgmma register operand), B = activations [T_pad x 64]
// fp16 per k-block in shared memory (K-major, 128-byte swizzle), D in registers (fp32).
//
// Warp roles (12 warps, three warpgroups; setmaxnreg moves registers from the third to the accumulators of the first two):
//   0..7   two consumer warpgroups; warp w owns the 16-row tile w.  Per k-block: ld.shared of its packed uint4, dequant
//          into four m64k16 A fragments, 4 x NC wgmma m64n32k16 (NC = T_pad / 32), wait; fp16 stores at the end
//   8      producer: packed W4 k-blocks HBM -> smem (8 bulk copies of 512 B per k-block, mbarrier expect_tx)
//   9..10  activation loaders: x[T][kb*64 .. +64] -> B stage, k permuted to the order of the packed fragments (below)
//   11     idle
//
// k order inside a 64-wide k-block.  Lane (g, t) of a packed tile holds rows g, g+8 at physical k 16t .. 16t+15 (four
// words: row g / g+8 x k 16t+0..7 / 16t+8..15), so the A fragment of k-step j is built from its own registers when
// logical k 16j + 8h + 2t + e (the fragment position, e = 0, 1) stands for physical k 16t + 8h + 2j + e.  The loaders
// store the activations in that logical order; the k-sum is the same sum.
//
// Pipelines: pk_full (bulk copies -> consumers), b_full (loaders -> consumers), empty (consumers, after the wgmma that read
// the stage completed -> producer and loaders).
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include <string>

#include "../../include/b200_decode.h"
#include "common.cuh"

namespace b200 {
namespace prefill {

constexpr int BM = 128, BK = 64, kStages = 4, kMaxT = 256, kNChunk = 32;
constexpr int kConsumerWarps = 8;
constexpr int kThreads = (kConsumerWarps + 4) * 32;
constexpr int kBBytes = kMaxT * BK * 2;     // 32 KB
constexpr int kPackedBytes = 8 * 512;       // 4 KB: one k-block of eight 16-row tiles
constexpr size_t kSmemBytes = (size_t)kStages * (kBBytes + kPackedBytes) + 3 * kStages * 8 + 1024;

struct Params {
  const uint8_t* qw;     // packed W4, tile-major (b200_pack_weight)
  const __half2* sz;     // per-channel (s, z) [N]
  const __half* x;       // [T][K]
  __half* out;           // [T][N]
  int N, K, KB, T, T_pad;  // T_pad = NC * 32 >= T, <= 256
};

// K-major, SWIZZLE_128B canonical layout of a [rows x 64] fp16 tile: 8-row groups of 1024 B, 16-byte chunk c of row r
// stored at chunk (c ^ (r & 7)).
__device__ __forceinline__ uint32_t sw128_offset(int row, int chunk) {
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4));
}

// wgmma shared-memory matrix descriptor (sm_90): start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), base offset [49,52),
// layout type [62,64) (1 = SWIZZLE_128B).  K-major, one swizzle atom wide: LBO unused (1), SBO = 1024 B between 8-row
// groups; the stage base is 1024-byte aligned, so the base offset is 0.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3ffff) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x 32] += A[64 x 16] (registers, fp16) . B[32 x 16]^T (shared memory, fp16, K-major), fp32 accumulate
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1)
      : "memory");
}

__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// (q - z) * s as the reference rounds it: q as 1024 + q (exact in fp16), minus (1024 + z) (exact), times s (one rounding)
__device__ __forceinline__ uint32_t deq2(uint32_t nib2, __half2 zoff, __half2 s2) {
  const uint32_t v = nib2 | 0x64006400u;
  const __half2 h = __hmul2(__hsub2(*reinterpret_cast<const __half2*>(&v), zoff), s2);
  return *reinterpret_cast<const uint32_t*>(&h);
}
// k pair 2j, 2j+1 of one packed u32 (8 consecutive k of one row, nibble order of pack.cpp kW4Nib: pairs at shifts
// 0, 8, 4, 12)
template <int J>
__device__ __forceinline__ uint32_t deq_pair(uint32_t w, __half2 zoff, __half2 s2) {
  constexpr int kShift = (J & 1) * 8 + (J >> 1) * 4;
  return deq2((w >> kShift) & 0x000f000fu, zoff, s2);
}

template <int NC>
__global__ void __launch_bounds__(kThreads, 1) prefill_gemm_w4_kernel(const __grid_constant__ Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);  // swizzle atoms need 1024-byte alignment
  uint8_t* b_st = smem;                                   // [kStages][32 KB]
  uint8_t* pk_st = b_st + kStages * kBBytes;              // [kStages][4 KB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(pk_st + kStages * kPackedBytes);
  uint64_t* pk_full = bars;                 // [kStages] producer -> consumers (tx bytes)
  uint64_t* b_full = pk_full + kStages;     // [kStages] loaders (64) -> consumers
  uint64_t* empty = b_full + kStages;       // [kStages] consumer warps (8) -> producer + loaders

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int row0 = blockIdx.x * BM;  // first output row of this CTA
  const int tile0 = row0 >> 4;

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&pk_full[s], 1);
      mbar_init(&b_full[s], 64);
      mbar_init(&empty[s], kConsumerWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < kConsumerWarps) {
    // ---------------- consumers: dequant -> wgmma, then the fp16 epilogue ----------------
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    const int g = lane >> 2, t4 = lane & 3;
    const __half2 sz_lo = p.sz[row0 + warp * 16 + g], sz_hi = p.sz[row0 + warp * 16 + g + 8];
    const __half2 s_lo = __half2half2(__low2half(sz_lo)), s_hi = __half2half2(__low2half(sz_hi));
    // 1024 + z: exact for |z| <= 1024
    const __half2 z_lo = __hadd2(__half2half2(__high2half(sz_lo)), __float2half2_rn(1024.f));
    const __half2 z_hi = __hadd2(__half2half2(__high2half(sz_hi)), __float2half2_rn(1024.f));
    float acc[NC][16];
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[c][i] = 0.f;
    for (int kb = 0; kb < p.KB; ++kb) {
      const int s = kb % kStages;
      const uint32_t par = (kb / kStages) & 1;
      mbar_wait(&pk_full[s], par);
      const uint4 w = lds_v4(pk_st + s * kPackedBytes + warp * 512 + lane * 16);
      // words: [0] row g, k 16t4 + 0..7; [1] row g+8, same k; [2] row g, k 16t4 + 8..15; [3] row g+8, same k
      uint32_t a[4][4];
#define B200_FRAG(J)                               \
  a[J][0] = deq_pair<J>(w.x, z_lo, s_lo);          \
  a[J][1] = deq_pair<J>(w.y, z_hi, s_hi);          \
  a[J][2] = deq_pair<J>(w.z, z_lo, s_lo);          \
  a[J][3] = deq_pair<J>(w.w, z_hi, s_hi);
      B200_FRAG(0) B200_FRAG(1) B200_FRAG(2) B200_FRAG(3)
#undef B200_FRAG
      mbar_wait(&b_full[s], par);
      const uint32_t b0 = smem_u32(b_st + s * kBBytes);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < BK / 16; ++j)  // +32 bytes per K = 16 step inside the 128-byte swizzle atom
#pragma unroll
        for (int c = 0; c < NC; ++c)     // +32 rows (4 swizzle atoms of 8 rows) per n-chunk
          wgmma_m64n32k16(acc[c], a[j], make_desc(b0 + c * 4096 + j * 32));
      wgmma_commit();
      wgmma_wait_all();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);  // this warp's reads of the packed and B stages are complete
    }
    // D fragment of warp w: acc[c][4i + 2h + e] = (row 16w + g + 8h, token 32c + 8i + 2t4 + e)
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int t = c * 32 + i * 8 + 2 * t4 + e, row = row0 + warp * 16 + g + 8 * h;
            if (t < p.T && row < p.N) p.out[(size_t)t * p.N + row] = __float2half_rn(acc[c][4 * i + 2 * h + e]);
          }
  } else {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
  }
  if (warp == kConsumerWarps) {
    // ---------------- producer: packed weights ----------------
    if (lane == 0) {
      for (int kb = 0; kb < p.KB; ++kb) {
        const int s = kb % kStages;
        const uint32_t par = (kb / kStages) & 1;
        mbar_wait(&empty[s], par ^ 1);
        mbar_arrive_expect_tx(&pk_full[s], kPackedBytes);
        for (int i = 0; i < 8; ++i)
          bulk_g2s(pk_st + s * kPackedBytes + i * 512, p.qw + ((size_t)(tile0 + i) * p.KB + kb) * 512, 512, &pk_full[s]);
      }
    }
  } else if (warp == kConsumerWarps + 1 || warp == kConsumerWarps + 2) {
    // ---------------- activation loaders: x block -> B stage in fragment k order ----------------
    // logical chunk c = 2j + h, word t  <-  physical word 4h + j + 8t  =  component j of input uint4 h + 2t
    const int lt = tid - (kConsumerWarps + 1) * 32;  // 0..63
    for (int kb = 0; kb < p.KB; ++kb) {
      const int s = kb % kStages;
      const uint32_t par = (kb / kStages) & 1;
      mbar_wait(&empty[s], par ^ 1);
      uint8_t* dst = b_st + s * kBBytes;
      for (int i = lt; i < p.T_pad * 2; i += 64) {
        const int t = i >> 1, h = i & 1;
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          v[u] = make_uint4(0, 0, 0, 0);
          if (t < p.T) v[u] = *reinterpret_cast<const uint4*>(p.x + (size_t)t * p.K + (size_t)kb * BK + (h + 2 * u) * 8);
        }
        *reinterpret_cast<uint4*>(dst + sw128_offset(t, 0 + h)) = make_uint4(v[0].x, v[1].x, v[2].x, v[3].x);
        *reinterpret_cast<uint4*>(dst + sw128_offset(t, 2 + h)) = make_uint4(v[0].y, v[1].y, v[2].y, v[3].y);
        *reinterpret_cast<uint4*>(dst + sw128_offset(t, 4 + h)) = make_uint4(v[0].z, v[1].z, v[2].z, v[3].z);
        *reinterpret_cast<uint4*>(dst + sw128_offset(t, 6 + h)) = make_uint4(v[0].w, v[1].w, v[2].w, v[3].w);
      }
      fence_async_smem();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
      mbar_arrive(&b_full[s]);
    }
  }
}

}  // namespace prefill
}  // namespace b200

// ---- elementwise kernels of the prefill chunk ----------------------------------------------------------------------------
namespace b200 {
void set_error(const std::string& s);
namespace prefill {

// h = resid (+ delta) -> h_out;  x = fp16(h * rsqrt(mean(h^2) + eps)) * gamma   (components.py:41-53, llama.py:286-287)
__global__ void rmsnorm_kernel(const __half* resid, const __half* delta, __half* h_out, const __half* gamma, float eps,
                               __half* x_out, int D) {
  const int t = blockIdx.x;
  extern __shared__ float red[];
  float ssq = 0.f;
  for (int i = threadIdx.x; i < D / 2; i += blockDim.x) {
    __half2 h = reinterpret_cast<const __half2*>(resid + (size_t)t * D)[i];
    if (delta) h = __hadd2(h, reinterpret_cast<const __half2*>(delta + (size_t)t * D)[i]);
    if (h_out) reinterpret_cast<__half2*>(h_out + (size_t)t * D)[i] = h;
    const float2 f = __half22float2(h);
    ssq = fmaf(f.x, f.x, ssq);
    ssq = fmaf(f.y, f.y, ssq);
  }
  ssq = warp_sum(ssq);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ssq;
  __syncthreads();
  float tot = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
  const float rstd = 1.0f / sqrtf(tot / (float)D + eps);
  for (int i = threadIdx.x; i < D / 2; i += blockDim.x) {
    __half2 h = reinterpret_cast<const __half2*>(resid + (size_t)t * D)[i];
    if (delta) h = __hadd2(h, reinterpret_cast<const __half2*>(delta + (size_t)t * D)[i]);
    const float2 f = __half22float2(h);
    reinterpret_cast<__half2*>(x_out + (size_t)t * D)[i] =
        __hmul2(__floats2half2_rn(f.x * rstd, f.y * rstd), reinterpret_cast<const __half2*>(gamma)[i]);
  }
}

// qkv [T][n_q + 2 n_kv] fp16 (GEMM output) -> RoPE on q, k (llama.py:59-77); q -> q_out [T][n_q]; k, v -> cache layouts
__global__ void rope_kv_kernel(const __half* qkv, __half* q_out, __half* kcache, __half* vtcache, const float2* rope,
                               const int* pos, int n_q, int n_kv, int tokens_per_seq, int cache_seq, int hkv) {
  const int t = blockIdx.x, N = n_q + 2 * n_kv;
  const int ps = pos[t], brow = t / tokens_per_seq;
  const __half* src = qkv + (size_t)t * N;
  for (int i = threadIdx.x; i < N / 2; i += blockDim.x) {
    const int row = 2 * i;
    const __half2 v = reinterpret_cast<const __half2*>(src)[i];
    const bool is_v = row >= n_q + n_kv;
    const int local = row < n_q ? row : (is_v ? row - n_q - n_kv : row - n_q);
    const int head = local >> 7, d = local & 127;
    __half o0 = __low2half(v), o1 = __high2half(v);
    if (!is_v) {
      const float2 cs = rope[(size_t)ps * 64 + (d >> 1)];
      const float xe = __half2float(o0), xo = __half2float(o1);
      o0 = __float2half_rn(__fsub_rn(__fmul_rn(xe, cs.x), __fmul_rn(xo, cs.y)));
      o1 = __float2half_rn(__fadd_rn(__fmul_rn(xe, cs.y), __fmul_rn(xo, cs.x)));
    }
    if (row < n_q) {
      reinterpret_cast<__half2*>(q_out + (size_t)t * n_q)[i] = __halves2half2(o0, o1);
    } else if (!is_v) {
      __half* dst = kcache + (((size_t)brow * hkv + head) * cache_seq + ps) * 128 + ((((d >> 3) ^ ((ps & 1) << 2)) << 3) | (d & 7));
      dst[0] = o0, dst[1] = o1;
    } else {
      __half* dst = vtcache + ((size_t)brow * hkv + head) * cache_seq * 128 + (size_t)(ps >> 5) * 4096 + d * 32 + (ps & 31);
      dst[0] = o0, dst[32] = o1;
    }
  }
}

// gu [T][2F] with w1 / w3 rows interleaved 8 + 8 per 16-row tile (EPI_SILU layout) -> act [T][F] = silu(w1 x) * (w3 x)
__global__ void silu_mul_kernel(const __half* gu, __half* act, int F) {
  const int t = blockIdx.x;
  for (int i = threadIdx.x; i < F; i += blockDim.x) {
    const int tile = i >> 3, r = i & 7;
    const __half a = gu[(size_t)t * 2 * F + tile * 16 + r], b = gu[(size_t)t * 2 * F + tile * 16 + 8 + r];
    const float af = __half2float(a);
    act[(size_t)t * F + i] = __hmul(__float2half_rn(af / (1.0f + expf(-af))), b);  // llama.py:252-256 rounding points
  }
}

}  // namespace prefill
}  // namespace b200

using namespace b200;

extern "C" int b200_prefill_gemm_w4(const b200_linear_t* lin, const void* x, void* out, int T, b200_stream_t stream) {
  using namespace b200::prefill;
  if (!lin || !x || !out || T < 1) return B200_E_INVAL;
  if (lin->bits != 4 || (lin->group_size > 0 && lin->group_size < lin->K) || (lin->N % BM) || (lin->K % BK) || !lin->qweight ||
      !lin->scales) {
    set_error("prefill_gemm_w4: per-channel W4 linear with N % 128 == 0 and K % 64 == 0 required");
    return B200_E_UNSUPPORTED;
  }
  static void (*const kernels[kMaxT / kNChunk])(Params) = {
      prefill_gemm_w4_kernel<1>, prefill_gemm_w4_kernel<2>, prefill_gemm_w4_kernel<3>, prefill_gemm_w4_kernel<4>,
      prefill_gemm_w4_kernel<5>, prefill_gemm_w4_kernel<6>, prefill_gemm_w4_kernel<7>, prefill_gemm_w4_kernel<8>};
  static bool configured[16] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  dev &= 15;
  if (!configured[dev]) {
    for (auto k : kernels) {
      cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
      if (e != cudaSuccess) {
        (void)cudaGetLastError();
        set_error(std::string("prefill_gemm_w4: cudaFuncSetAttribute: ") + cudaGetErrorString(e));
        return (int)e;
      }
    }
    configured[dev] = true;
  }
  for (int t0 = 0; t0 < T; t0 += kMaxT) {  // token blocks of <= 256: a CTA's accumulators are 128 rows x 256 fp32 registers
    Params p;
    p.qw = static_cast<const uint8_t*>(lin->qweight);
    p.sz = static_cast<const __half2*>(lin->scales);
    p.x = static_cast<const __half*>(x) + (size_t)t0 * lin->K;
    p.out = static_cast<__half*>(out) + (size_t)t0 * lin->N;
    p.N = lin->N, p.K = lin->K, p.KB = lin->K / BK, p.T = std::min(kMaxT, T - t0);
    const int nc = (p.T + kNChunk - 1) / kNChunk;
    p.T_pad = nc * kNChunk;
    kernels[nc - 1]<<<lin->N / BM, kThreads, kSmemBytes, static_cast<cudaStream_t>(stream)>>>(p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error(std::string("prefill_gemm_w4: launch: ") + cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

extern "C" int b200_prefill_rmsnorm(const void* resid, const void* delta, void* h_out, const void* gamma, float eps, void* x_out,
                                    int T, int D, b200_stream_t stream) {
  if (!resid || !gamma || !x_out || T < 1 || D < 2 || (D & 1)) return B200_E_INVAL;
  prefill::rmsnorm_kernel<<<T, 256, 8 * sizeof(float), static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(resid), static_cast<const __half*>(delta), static_cast<__half*>(h_out),
      static_cast<const __half*>(gamma), eps, static_cast<__half*>(x_out), D);
  return (int)cudaGetLastError();
}

extern "C" int b200_prefill_rope_kv(const void* qkv, void* q_out, void* kcache, void* vtcache, const float* rope,
                                    const int32_t* pos, int T, int n_q_rows, int n_kv_rows, int tokens_per_seq, int cache_seq,
                                    b200_stream_t stream) {
  if (!qkv || !q_out || !kcache || !vtcache || !rope || !pos || T < 1 || (n_q_rows & 127) || (n_kv_rows & 127) ||
      tokens_per_seq < 1)
    return B200_E_INVAL;
  prefill::rope_kv_kernel<<<T, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(qkv), static_cast<__half*>(q_out), static_cast<__half*>(kcache), static_cast<__half*>(vtcache),
      reinterpret_cast<const float2*>(rope), pos, n_q_rows, n_kv_rows, tokens_per_seq, cache_seq, n_kv_rows / 128);
  return (int)cudaGetLastError();
}

extern "C" int b200_prefill_silu_mul(const void* gu, void* act, int T, int F, b200_stream_t stream) {
  if (!gu || !act || T < 1 || F < 8 || (F & 7)) return B200_E_INVAL;
  prefill::silu_mul_kernel<<<T, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const __half*>(gu),
                                                                             static_cast<__half*>(act), F);
  return (int)cudaGetLastError();
}
