// Prompt GEMM on the Hopper tensor cores (wgmma, fp32 accumulators in registers) for per-channel W4 / W3 and fp16 linears,
// and the elementwise kernels around it; replaces F.linear at M = prompt tokens (accessory/util/quant.py:18-46,
// llama.py:276-288) for prompts longer than one 32-token chunk of the decode GEMV.
//
// GEMM:   out[T, N] = x[T, K] . w_hat[N, K]^T
//   w_hat = fp16(fp16(q - z) * s16)  -- the reference's fake-quantised weight, reproduced bit for bit, so the prefill
//   logits follow F.linear(x, w_hat) with fp32 accumulation (accessory/util/quant.py:18-46 + SURVEY.md 8c).  For fp16
//   linears w_hat is the weight itself.
//
// One CTA owns 128 output rows (eight 16-row tiles of the packed decode format, DESIGN.md section 3) and up to 256
// tokens.  D[rows x tokens] = A . B^T with A = dequantised weights (wgmma register operand), B = activations [T_pad x kK]
// fp16 per pipeline stage in shared memory (K-major), D in registers (fp32).
//
// Warp roles (12 warps, three warpgroups; setmaxnreg moves registers from the third to the accumulators of the first two):
//   0..7   two consumer warpgroups; warp w owns the 16-row tile w.  Per stage: ld.shared of its packed uint4(s), dequant
//          into kSteps m64k16 A fragments, kSteps x NC wgmma m64n32k16 (NC = T_pad / 32), wait; fp16 stores at the end
//   8      producer: packed weights HBM -> smem (8 bulk copies of one tile's stage bytes, mbarrier expect_tx)
//   9..10  activation loaders: x[T][stage k range] -> B stage, k permuted to the order of the packed fragments (below)
//   11     idle
//
// Per codec (pack.cpp), one stage holds:
//   W4   one 64-k block: lane (g, t) of a packed tile holds rows g, g+8 at physical k 16t .. 16t+15 (four words: row g /
//        g+8 x k 16t+0..7 / 16t+8..15).  The A fragment of k-step j is built from its own registers when logical k
//        16j + 8h + 2t + e (the fragment position, e = 0, 1) stands for physical k 16t + 8h + 2j + e.
//   W3   one 80-k block (5 k-steps): the lane holds k 20t .. 20t+19 (words: row g / g+8 x k 20t+0..9 / 20t+10..19);
//        logical k 16j + 8h + 2t + e stands for physical k 20t + 10h + 2j + e.  K need not be a multiple of 80: the
//        packer pads the last block with q = 0 (w_hat = -z s != 0), so the loaders write zero activations at k >= K.
//   fp16 four 16-k blocks: the lane's uint4 of block j is already the A fragment of k-step j when logical k
//        16j + 8h + 2t + e stands for physical k 16j + 4t + 2h + e.
// The loaders store the activations in that logical order; the k-sum is the same sum.
//
// Pipelines: pk_full (bulk copies -> consumers), b_full (loaders -> consumers), empty (consumers, after the wgmma that read
// the stage completed -> producer and loaders).
//
// Grouped MoE mode (b200_prefill_moe_gemm_w4, Mixtral prompts, W4 only): the same CTA with routed rows -- the producer
// streams the CTA's expert, the loaders gather the activation rows of the slots routed to it, the epilogue scatters to
// those slots (mixtral.py:266-294 runs the experts one at a time the same way: gather, expert, scatter).
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

enum class Codec { W4, W3, F16 };

// One pipeline stage of a codec: kK logical k (kSteps wgmma k-steps), kTileBytes packed bytes of one 16-row tile (contiguous
// in the tile-major layout), kBBytes of activations for 256 tokens.  Four stages fit the 227 KB of an H100 SM for all three:
// W4 4 x (32 + 4) KB, W3 4 x (40 + 4) KB, fp16 4 x (32 + 16) KB.
template <Codec C>
struct Stage {
  static constexpr int kK = C == Codec::W3 ? 80 : 64;
  static constexpr int kSteps = kK / 16;
  static constexpr int kTileBytes = C == Codec::F16 ? 4 * 512 : 512;
  static constexpr int kPackedBytes = 8 * kTileBytes;
  static constexpr int kBBytes = kMaxT * kK * 2;
  static constexpr size_t kSmemBytes = (size_t)kStages * (kBBytes + kPackedBytes) + 3 * kStages * 8 + 1024;
};

struct Params {
  const uint8_t* qw;     // packed weights, tile-major (b200_pack_weight / b200_pack_f16)
  const __half2* sz;     // per-channel (s, z) [N]; unused for fp16
  const __half* x;       // [T][K]
  __half* out;           // [T][N]
  int N, K, KB, T, T_pad;  // KB: pipeline stages over K; T_pad = NC * 32 >= T, <= 256
  const __half* bias;      // [N] fp16, read only by the kBias instances (b200_prefill_gemm_w4_bias)
  int bias_mode;           // B200_BIAS_ACC: fp16(acc + b); B200_BIAS_OUT: fp16(fp16(acc) + b)
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

// W3 stages are 80 k wide, which no 64-k swizzle atom tiles: K-major without swizzle (layout type 0), one column of
// 8 x 16-byte core matrices per 16-k step.  Core matrix (8-row group r8, k half h) of step j at
// j * 8192 + r8 * 256 + h * 128, its row r at + 16 r: LBO = 128 B between the two k halves, SBO = 256 B between 8-row groups.
constexpr int kW3StepBytes = kMaxT * 16 * 2;
__device__ __forceinline__ uint32_t w3_offset(int row, int step, int half) {
  return (uint32_t)(step * kW3StepBytes + (row >> 3) * 256 + half * 128 + (row & 7) * 16);
}
__device__ __forceinline__ uint64_t make_desc_w3(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3ffff) >> 4);
  d |= (uint64_t)(128 >> 4) << 16;
  d |= (uint64_t)(256 >> 4) << 32;
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
// k pair 2j, 2j+1 of one packed W3 u32 (10 consecutive k of one row, pack.cpp kW3Base: pair j's even element in the
// 3-bit field kW3Base[j] of the low half-word, its odd element in the same field of the high half-word)
template <int J>
__device__ __forceinline__ uint32_t deq_pair_w3(uint32_t w, __half2 zoff, __half2 s2) {
  constexpr int kBase[5] = {0, 3, 1, 4, 2};
  return deq2((w >> (3 * kBase[J])) & 0x00070007u, zoff, s2);
}

// One CTA of the GEMM: 128 output rows x p.T (<= NC * 32) tokens.  kRouted (the grouped MoE GEMM): token t of the CTA is
// slot rows[t] (shared memory); its activations are row rows[t] / src_div of p.x and its outputs row rows[t] of p.out.
template <Codec C, int NC, bool kRouted, bool kBias = false>
__device__ __forceinline__ void gemm_cta(const Params& p, uint8_t* smem_raw, const int* rows, int src_div) {
  using S = Stage<C>;
  constexpr int kBBytes = S::kBBytes, kPackedBytes = S::kPackedBytes;
  uint8_t* smem = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);  // swizzle atoms need 1024-byte alignment
  uint8_t* b_st = smem;                                   // [kStages][kBBytes]
  uint8_t* pk_st = b_st + kStages * kBBytes;              // [kStages][kPackedBytes]
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
    __half2 s_lo, s_hi, z_lo, z_hi;
    if constexpr (C != Codec::F16) {
      const __half2 sz_lo = p.sz[row0 + warp * 16 + g], sz_hi = p.sz[row0 + warp * 16 + g + 8];
      s_lo = __half2half2(__low2half(sz_lo)), s_hi = __half2half2(__low2half(sz_hi));
      // 1024 + z: exact for |z| <= 1024
      z_lo = __hadd2(__half2half2(__high2half(sz_lo)), __float2half2_rn(1024.f));
      z_hi = __hadd2(__half2half2(__high2half(sz_hi)), __float2half2_rn(1024.f));
    }
    float acc[NC][16];
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[c][i] = 0.f;
    for (int kb = 0; kb < p.KB; ++kb) {
      const int s = kb % kStages;
      const uint32_t par = (kb / kStages) & 1;
      mbar_wait(&pk_full[s], par);
      uint32_t a[S::kSteps][4];
      if constexpr (C == Codec::F16) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint4 w = lds_v4(pk_st + s * kPackedBytes + warp * S::kTileBytes + j * 512 + lane * 16);
          a[j][0] = w.x, a[j][1] = w.y, a[j][2] = w.z, a[j][3] = w.w;
        }
      } else {
        const uint4 w = lds_v4(pk_st + s * kPackedBytes + warp * 512 + lane * 16);
        // words: [0] row g, first half of the lane's k run; [1] row g+8, same k; [2] row g, second half; [3] row g+8
        if constexpr (C == Codec::W4) {
#define B200_FRAG(J)                               \
  a[J][0] = deq_pair<J>(w.x, z_lo, s_lo);          \
  a[J][1] = deq_pair<J>(w.y, z_hi, s_hi);          \
  a[J][2] = deq_pair<J>(w.z, z_lo, s_lo);          \
  a[J][3] = deq_pair<J>(w.w, z_hi, s_hi);
          B200_FRAG(0) B200_FRAG(1) B200_FRAG(2) B200_FRAG(3)
#undef B200_FRAG
        } else {
#define B200_FRAG(J)                               \
  a[J][0] = deq_pair_w3<J>(w.x, z_lo, s_lo);       \
  a[J][1] = deq_pair_w3<J>(w.y, z_hi, s_hi);       \
  a[J][2] = deq_pair_w3<J>(w.z, z_lo, s_lo);       \
  a[J][3] = deq_pair_w3<J>(w.w, z_hi, s_hi);
          B200_FRAG(0) B200_FRAG(1) B200_FRAG(2) B200_FRAG(3) B200_FRAG(4)
#undef B200_FRAG
        }
      }
      mbar_wait(&b_full[s], par);
      const uint32_t b0 = smem_u32(b_st + s * kBBytes);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < S::kSteps; ++j)
#pragma unroll
        for (int c = 0; c < NC; ++c) {   // +32 rows per n-chunk
          if constexpr (C == Codec::W3)
            wgmma_m64n32k16(acc[c], a[j], make_desc_w3(b0 + j * kW3StepBytes + c * 1024));
          else  // +32 bytes per K = 16 step inside the 128-byte swizzle atom, 4 swizzle atoms of 8 rows per n-chunk
            wgmma_m64n32k16(acc[c], a[j], make_desc(b0 + c * 4096 + j * 32));
        }
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
            if (t < p.T && row < p.N) {
              const float y = acc[c][4 * i + 2 * h + e];
              __half o;
              if constexpr (kBias) {
                const __half b = p.bias[row];
                o = p.bias_mode == B200_BIAS_ACC ? __float2half_rn(__fadd_rn(y, __half2float(b))) : __hadd(__float2half_rn(y), b);
              } else {
                o = __float2half_rn(y);
              }
              p.out[(size_t)(kRouted ? rows[t] : t) * p.N + row] = o;
            }
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
          bulk_g2s(pk_st + s * kPackedBytes + i * S::kTileBytes, p.qw + ((size_t)(tile0 + i) * p.KB + kb) * S::kTileBytes,
                   S::kTileBytes, &pk_full[s]);
      }
    }
  } else if (warp == kConsumerWarps + 1 || warp == kConsumerWarps + 2) {
    // ---------------- activation loaders: x block -> B stage in fragment k order ----------------
    const int lt = tid - (kConsumerWarps + 1) * 32;  // 0..63
    for (int kb = 0; kb < p.KB; ++kb) {
      const int s = kb % kStages;
      const uint32_t par = (kb / kStages) & 1;
      mbar_wait(&empty[s], par ^ 1);
      uint8_t* dst = b_st + s * kBBytes;
      // thread (t, h): token t, half h of the stage's k range
      for (int i = lt; i < p.T_pad * 2; i += 64) {
        const int t = i >> 1, h = i & 1;
        if constexpr (C == Codec::W4) {
          // logical chunk c = 2j + h, word t  <-  physical word 4h + j + 8t  =  component j of input uint4 h + 2t
          uint4 v[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            v[u] = make_uint4(0, 0, 0, 0);
            if (t < p.T) {
              const int src = kRouted ? rows[t] / src_div : t;
              v[u] = *reinterpret_cast<const uint4*>(p.x + (size_t)src * p.K + (size_t)kb * BK + (h + 2 * u) * 8);
            }
          }
          *reinterpret_cast<uint4*>(dst + sw128_offset(t, 0 + h)) = make_uint4(v[0].x, v[1].x, v[2].x, v[3].x);
          *reinterpret_cast<uint4*>(dst + sw128_offset(t, 2 + h)) = make_uint4(v[0].y, v[1].y, v[2].y, v[3].y);
          *reinterpret_cast<uint4*>(dst + sw128_offset(t, 4 + h)) = make_uint4(v[0].z, v[1].z, v[2].z, v[3].z);
          *reinterpret_cast<uint4*>(dst + sw128_offset(t, 6 + h)) = make_uint4(v[0].w, v[1].w, v[2].w, v[3].w);
        } else if constexpr (C == Codec::F16) {
          // 16-k blocks 2h, 2h+1; logical chunk (j, hh) of block j, word t  <-  physical word 2t + hh of the block
          const __half* src = p.x + (size_t)t * p.K + (size_t)kb * S::kK;
#pragma unroll
          for (int jj = 0; jj < 2; ++jj) {
            const int j = 2 * h + jj;
            uint4 lo = make_uint4(0, 0, 0, 0), hi = lo;
            if (t < p.T) {
              lo = *reinterpret_cast<const uint4*>(src + j * 16);
              hi = *reinterpret_cast<const uint4*>(src + j * 16 + 8);
            }
            *reinterpret_cast<uint4*>(dst + sw128_offset(t, 2 * j)) = make_uint4(lo.x, lo.z, hi.x, hi.z);
            *reinterpret_cast<uint4*>(dst + sw128_offset(t, 2 * j + 1)) = make_uint4(lo.y, lo.w, hi.y, hi.w);
          }
        } else {
          // physical words 20h .. 20h+19 of the 40 (lane groups t' = 2h, 2h+1): word 10t' + 5hh + j of the block is word t'
          // of logical chunk (j, hh), so this thread fills bytes 8h .. 8h+7 of every chunk.  Zero at k >= K (K % 16 == 0:
          // a uint4 of 8 k lies wholly on one side of K), so nothing past column K of the row is read.
          const __half* src = p.x + (size_t)t * p.K + (size_t)kb * S::kK;
          uint4 v[5];
#pragma unroll
          for (int u = 0; u < 5; ++u) {
            v[u] = make_uint4(0, 0, 0, 0);
            if (t < p.T && kb * S::kK + 40 * h + 8 * u < p.K) v[u] = *reinterpret_cast<const uint4*>(src + 40 * h + 8 * u);
          }
          const uint32_t* w = reinterpret_cast<const uint32_t*>(v);
#pragma unroll
          for (int j = 0; j < 5; ++j)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
              *reinterpret_cast<uint2*>(dst + w3_offset(t, j, hh) + 8 * h) = make_uint2(w[5 * hh + j], w[10 + 5 * hh + j]);
        }
      }
      fence_async_smem();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
      mbar_arrive(&b_full[s]);
    }
  }
}

template <int NC>
__global__ void __launch_bounds__(kThreads, 1) prefill_gemm_w4_kernel(const __grid_constant__ Params p) {
  extern __shared__ uint8_t smem_raw[];
  gemm_cta<Codec::W4, NC, false>(p, smem_raw, nullptr, 1);
}
template <int NC>
__global__ void __launch_bounds__(kThreads, 1) prefill_gemm_w3_kernel(const __grid_constant__ Params p) {
  extern __shared__ uint8_t smem_raw[];
  gemm_cta<Codec::W3, NC, false>(p, smem_raw, nullptr, 1);
}
template <int NC>
__global__ void __launch_bounds__(kThreads, 1) prefill_gemm_f16_kernel(const __grid_constant__ Params p) {
  extern __shared__ uint8_t smem_raw[];
  gemm_cta<Codec::F16, NC, false>(p, smem_raw, nullptr, 1);
}
// b200_prefill_gemm_w4_bias: the same CTA with the bias added at the store (separate instances; the ones above are untouched)
template <Codec C, int NC>
__global__ void __launch_bounds__(kThreads, 1) prefill_gemm_bias_kernel(const __grid_constant__ Params p) {
  extern __shared__ uint8_t smem_raw[];
  gemm_cta<C, NC, false, true>(p, smem_raw, nullptr, 1);
}

// ---- grouped MoE GEMM: the same CTA over the slots routed to one expert -------------------------------------------------
constexpr int kMaxMoeExperts = 64;  // the router's limit (moe.cu kMaxExperts)

struct MoeParams {
  const int32_t* slot_expert;  // [n_slots] global expert id of every slot
  const __half* x;             // [n_slots / src_div rows][K]
  __half* out;                 // [n_slots][N]
  int N, K, n_slots, src_div, e_first;
  const uint8_t* qw[kMaxMoeExperts];
  const __half2* sz[kMaxMoeExperts];
};

// grid (N / 128, e_count, ceil(n_slots / 256)): CTA (x, i, b) owns output rows [128 x, 128 x + 128) of expert e_first + i for
// entries [256 b, 256 b + 256) of that expert's slot list (its slots in increasing order).  Every CTA scans slot_expert
// itself (n_slots int32, L2-resident), so the launch needs no workspace, atomics or index-building pass; a CTA with no
// entries exits before it issues any copy.
__global__ void __launch_bounds__(kThreads, 1) prefill_moe_gemm_w4_kernel(const __grid_constant__ MoeParams mp) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ int rows[kMaxT];
  __shared__ int warp_hits[kThreads / 32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int expert = mp.e_first + blockIdx.y, lo = blockIdx.z * kMaxT;
  int found = 0;  // list entries in the slots scanned so far (CTA-uniform)
  for (int s0 = 0; s0 < mp.n_slots && found < lo + kMaxT; s0 += kThreads) {
    const int s = s0 + tid;
    const bool hit = s < mp.n_slots && mp.slot_expert[s] == expert;
    const uint32_t m = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) warp_hits[warp] = __popc(m);
    __syncthreads();
    int idx = found + __popc(m & ((1u << lane) - 1u));
    for (int w = 0; w < kThreads / 32; ++w) {
      const int c = warp_hits[w];
      idx += w < warp ? c : 0;
      found += c;
    }
    if (hit && idx >= lo && idx < lo + kMaxT) rows[idx - lo] = s;
    __syncthreads();  // warp_hits is rewritten by the next round; rows is complete after the last one
  }
  const int n = min(found - lo, kMaxT);
  if (n <= 0) return;
  Params p;
  p.qw = mp.qw[blockIdx.y];
  p.sz = mp.sz[blockIdx.y];
  p.x = mp.x;
  p.out = mp.out;
  p.N = mp.N, p.K = mp.K, p.KB = mp.K / BK, p.T = n;
  switch ((n + kNChunk - 1) / kNChunk) {  // the accumulator count is a compile-time NC, as in the dense launches
#define B200_NC(NC)                                          \
  case NC:                                                   \
    p.T_pad = NC * kNChunk;                                  \
    gemm_cta<Codec::W4, NC, true>(p, smem_raw, rows, mp.src_div); \
    break;
    B200_NC(1) B200_NC(2) B200_NC(3) B200_NC(4) B200_NC(5) B200_NC(6) B200_NC(7) B200_NC(8)
#undef B200_NC
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

namespace b200 {
namespace prefill {

using GemmKernel = void (*)(Params);
template <Codec C, int NC, bool kBias>
constexpr GemmKernel gemm_kernel() {
  if constexpr (kBias) return prefill_gemm_bias_kernel<C, NC>;
  else if constexpr (C == Codec::W4) return prefill_gemm_w4_kernel<NC>;
  else if constexpr (C == Codec::W3) return prefill_gemm_w3_kernel<NC>;
  else return prefill_gemm_f16_kernel<NC>;
}

template <Codec C, bool kBias = false>
int launch_gemm(const b200_linear_t* lin, const void* x, void* out, int T, cudaStream_t stream, const void* bias = nullptr,
                int bias_mode = 0) {
  using S = Stage<C>;
  static const GemmKernel kernels[kMaxT / kNChunk] = {
      gemm_kernel<C, 1, kBias>(), gemm_kernel<C, 2, kBias>(), gemm_kernel<C, 3, kBias>(), gemm_kernel<C, 4, kBias>(),
      gemm_kernel<C, 5, kBias>(), gemm_kernel<C, 6, kBias>(), gemm_kernel<C, 7, kBias>(), gemm_kernel<C, 8, kBias>()};
  static bool configured[16] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  dev &= 15;
  if (!configured[dev]) {
    for (auto k : kernels) {
      cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S::kSmemBytes);
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
    p.N = lin->N, p.K = lin->K, p.KB = (lin->K + S::kK - 1) / S::kK, p.T = std::min(kMaxT, T - t0);
    p.bias = static_cast<const __half*>(bias);
    p.bias_mode = bias_mode;
    const int nc = (p.T + kNChunk - 1) / kNChunk;
    p.T_pad = nc * kNChunk;
    kernels[nc - 1]<<<lin->N / BM, kThreads, S::kSmemBytes, stream>>>(p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error(std::string("prefill_gemm_w4: launch: ") + cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

}  // namespace prefill
}  // namespace b200

static int check_prefill_linear(const b200_linear_t* lin, const void* x, void* out, int T) {
  using namespace b200::prefill;
  if (!lin || !x || !out || T < 1) return B200_E_INVAL;
  const int bits = lin->bits;
  const int k_quantum = bits == 3 ? 16 : BK;  // W3: the loaders zero the activations of the padded tail of the last 80-k block
  if ((bits != 4 && bits != 3 && bits != 16) || (lin->group_size > 0 && lin->group_size < lin->K) || (lin->N % BM) ||
      (lin->K % k_quantum) || !lin->qweight || (bits != 16 && !lin->scales)) {
    set_error("prefill_gemm_w4: per-channel W4 / W3 or fp16 linear with N % 128 == 0 and K % 64 == 0 (W3: K % 16 == 0) "
              "required");
    return B200_E_UNSUPPORTED;
  }
  return 0;
}

extern "C" int b200_prefill_gemm_w4(const b200_linear_t* lin, const void* x, void* out, int T, b200_stream_t stream) {
  using namespace b200::prefill;
  const int rc = check_prefill_linear(lin, x, out, T);
  if (rc) return rc;
  const int bits = lin->bits;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (bits == 4) return launch_gemm<Codec::W4>(lin, x, out, T, st);
  if (bits == 3) return launch_gemm<Codec::W3>(lin, x, out, T, st);
  return launch_gemm<Codec::F16>(lin, x, out, T, st);
}

extern "C" int b200_prefill_gemm_w4_bias(const b200_linear_t* lin, const void* x, const void* bias, int bias_mode, void* out,
                                         int T, b200_stream_t stream) {
  using namespace b200::prefill;
  if (!bias || (bias_mode != B200_BIAS_ACC && bias_mode != B200_BIAS_OUT)) {
    set_error("prefill_gemm_w4_bias: needs a bias and bias_mode 1 (B200_BIAS_ACC) or 2 (B200_BIAS_OUT)");
    return B200_E_INVAL;
  }
  const int rc = check_prefill_linear(lin, x, out, T);
  if (rc) return rc;
  const int bits = lin->bits;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (bits == 4) return launch_gemm<Codec::W4, true>(lin, x, out, T, st, bias, bias_mode);
  if (bits == 3) return launch_gemm<Codec::W3, true>(lin, x, out, T, st, bias, bias_mode);
  return launch_gemm<Codec::F16, true>(lin, x, out, T, st, bias, bias_mode);
}

extern "C" int b200_prefill_moe_gemm_w4(const b200_linear_t* experts, int e_first, int e_count, const int32_t* slot_expert,
                                        int n_slots, int src_div, const void* x, void* out, b200_stream_t stream) {
  using namespace b200::prefill;
  if (!experts || !slot_expert || !x || !out) {
    set_error("prefill_moe_gemm_w4: null pointer");
    return B200_E_INVAL;
  }
  if (e_count < 1 || n_slots < 1 || src_div < 1) {
    set_error("prefill_moe_gemm_w4: e_count, n_slots and src_div must be >= 1");
    return B200_E_INVAL;
  }
  if (e_count > kMaxMoeExperts) {
    set_error("prefill_moe_gemm_w4: more than 64 experts in one launch");
    return B200_E_UNSUPPORTED;
  }
  MoeParams mp = {};
  mp.N = experts[0].N, mp.K = experts[0].K;
  for (int i = 0; i < e_count; ++i) {
    const b200_linear_t& l = experts[i];
    if (l.bits != 4 || (l.group_size > 0 && l.group_size < l.K) || l.N != mp.N || l.K != mp.K || (l.N % BM) || (l.K % BK) ||
        l.N < BM || l.K < BK || !l.qweight || !l.scales) {
      set_error("prefill_moe_gemm_w4: per-channel W4 experts of equal N % 128 == 0 and K % 64 == 0 required");
      return B200_E_UNSUPPORTED;
    }
    mp.qw[i] = static_cast<const uint8_t*>(l.qweight);
    mp.sz[i] = static_cast<const __half2*>(l.scales);
  }
  mp.slot_expert = slot_expert;
  mp.x = static_cast<const __half*>(x);
  mp.out = static_cast<__half*>(out);
  mp.n_slots = n_slots, mp.src_div = src_div, mp.e_first = e_first;
  static bool configured[16] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  dev &= 15;
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(prefill_moe_gemm_w4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)Stage<Codec::W4>::kSmemBytes);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      set_error(std::string("prefill_moe_gemm_w4: cudaFuncSetAttribute: ") + cudaGetErrorString(e));
      return (int)e;
    }
    configured[dev] = true;
  }
  const dim3 grid(mp.N / BM, e_count, (n_slots + kMaxT - 1) / kMaxT);
  prefill_moe_gemm_w4_kernel<<<grid, kThreads, Stage<Codec::W4>::kSmemBytes, static_cast<cudaStream_t>(stream)>>>(mp);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error(std::string("prefill_moe_gemm_w4: launch: ") + cudaGetErrorString(e));
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
