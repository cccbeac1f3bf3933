// One persistent kernel = one whole bs = 1 decode step of a dense LLaMA (TP = 1, W4 per-channel + fp16 lm_head):
//
//   L x [ RMSNorm + QKV + RoPE + KV-append | split-KV attention | merge + wo | residual + RMSNorm + gate/up + SiLU*mul | down ]
//   -> residual + RMSNorm + lm_head -> fp32 logits                                      (llama.py:394-427, 276-288)
//
// Why: as separate kernels every one of the 5L+1 dependent phases costs a drain, a dependency release, an x-staging
// round trip and a cold ring during which HBM idles; together that is comparable to the time the step's
// 4.6 GB take at full bandwidth.  Here one CTA per SM stays resident for the whole step:
//   * the producer warp streams weights / K-V tiles of phase after phase through ONE shared-memory ring and never
//     waits for a dependency (weights are constants); while the MMA warps sit at a grid barrier and re-stage the
//     activation vector, the ring (~150 KB per SM = 3.4 us of HBM time) keeps filling, so HBM does not idle;
//   * the MMA / epilogue roles are the bs = 1 integer-tensor-path GEMV phases of gemv1_core.cuh (exact IMMA dot
//     products) and, for the fp16 lm_head, the HMMA phase of gemv_core.cuh;
//   * attention runs on the same 16 MMA warps: a CTA takes one (kv head, split) item, every warp one 32-position tile
//     at a time out of the ring (online softmax as in attn.cu), partials (m, l, O) are merged inside the CTA through
//     shared memory and across splits by the wo phase's prologue (no extra barrier);
//   * phases are separated by a grid barrier: epilogue warps release-arrive on a per-phase counter after their stores,
//     one MMA thread acquire-polls it; the last CTA out resets the counters (CUDA-graph replay safe).
// Per-layer pointers travel as kernel parameters (constant bank): phase descriptors are built in registers.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>

#include "gemv1_core.cuh"

namespace b200 {

constexpr int kMegaMaxLayers = 96;
constexpr int kTileKV = 32;  // kv positions per attention tile: K tile 8 KB + V tile 8 KB = one ring slot

struct MegaLayer {
  const uint8_t *wqkv, *wo, *w13, *w2;
  const __half2 *sqkv, *so, *s13, *s2;
  const __half *attn_norm, *ffn_norm;
};

struct MegaParams {
  int n_layers, D, Hq, Hkv, F, V, cache_seq, stages, n_split, xq_bytes;
  int flags;  // experiment knobs (B200_STEP1_FLAGS): 1 = no __threadfence before the release-arrive
  float eps, scale_log2;
  const long long* token;
  const __half* tok_emb;
  const int* pos;
  const float2* rope;
  __half* kcache;
  __half* vtcache;
  long long kv_layer_stride;  // halfs between the caches of consecutive layers
  __half *h0, *h1, *q, *act;
  float* attn_ws;  // O fp32 [Hq][n_split][128], then (m, l) float2 [Hq][n_split]
  const uint8_t* lm_head;
  const __half* final_norm;
  // communication block (one per rank, identical layout, peer-mapped for tp_world > 1; see b200_step1_comm_bytes):
  //   u32 bar[5L+1] phase arrival counters (monotonic) | u32 exit counter | u32 epoch (launches completed) | pad to 256 B
  //   fp16 parts[2][tp_world][D]   row-parallel partial sums of wo (0) and w2 (1), slot r written by rank r
  //   fp32 logits[V * tp_world]    gathered logits
  int tp_world, tp_rank;
  uint8_t* comm[8];        // comm[r] = rank r's block; comm[tp_rank] is local
  int parts_off, logits_off;  // byte offsets inside a block
  unsigned long long* tl;  // optional [5L+1][8] timestamps of CTA 0 (ns): gate passed, x staged, loop done, epilogue arrived,
                           // first weight slot seen, producer issued the phase's last slot, epilogue staged its scales
  MegaLayer layer[kMegaMaxLayers];
};

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_sys_add(unsigned* p, unsigned v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// Phase barriers.  Counters are monotonic (never reset): launch number `epoch` waits for (epoch + 1) * arrivals-per-launch,
// compared wrap-safe.  Phases whose output other RANKS consume (wo, w2, lm_head) collect n_cta arrivals from every rank.
struct Bars {
  unsigned* local;    // this rank's counters
  unsigned epoch1;    // epoch + 1
  int n_cta, world;
};
__device__ __forceinline__ bool phase_is_cross(int ph, int n_ph) { return ph == n_ph - 1 || (ph % 5) == 2 || (ph % 5) == 4; }
__device__ __forceinline__ void bar_wait(const Bars& b, int ph, int n_ph) {
  const bool cross = b.world > 1 && phase_is_cross(ph, n_ph);
  const unsigned target = b.epoch1 * (unsigned)(b.n_cta * (cross ? b.world : 1));
  if (cross) {
    while ((int)(ld_acquire_sys_u32(b.local + ph) - target) < 0) {
    }
  } else {
    while ((int)(ld_acquire_u32(b.local + ph) - target) < 0) {
    }
  }
}
__device__ __forceinline__ void bar_arrive(const MegaParams& mp, int ph, int n_ph) {
  const bool cross = mp.tp_world > 1 && phase_is_cross(ph, n_ph);
  if (cross) {
    __threadfence_system();  // this CTA's stores into the peers' blocks are visible before the arrivals
    for (int r = 0; r < mp.tp_world; ++r) red_release_sys_add(reinterpret_cast<unsigned*>(mp.comm[r]) + ph, 1u);
  } else {
    if (!(mp.flags & 1)) __threadfence();
    red_release_add(reinterpret_cast<unsigned*>(mp.comm[mp.tp_rank]) + ph, 1u);
  }
}
__device__ __forceinline__ void mtl(const MegaParams& mp, int ph, int k) {
  if (mp.tl && blockIdx.x == 0) mp.tl[ph * 8 + k] = gtime_ns();
}

// ---- phase descriptors ---------------------------------------------------------------------------------------
enum { PH_QKV = 0, PH_ATTN = 1, PH_WO = 2, PH_W13 = 3, PH_W2 = 4 };

__device__ __forceinline__ void gemv_common(GemvParams& p, const MegaParams& mp, const uint8_t* qw, const __half2* sz, int N,
                                            int K, int bits) {
  p.bits = bits;
  p.qw = qw;
  p.sz = sz;
  p.N = N;
  p.K = K;
  const int kblk = bits == 4 ? 64 : 16;
  p.KB = K / kblk;
  p.Kpad = K;
  p.n_tiles = N / 16;
  p.G = 1;
  p.gb_mask = 0x7fffffff;
  p.T = 1;
  p.eps = mp.eps;
  p.stages = mp.stages;
  p.tokens_per_seq = 1;
  p.src_div = 1;
  p.x_stride = K + kXPad;
  p.n_chunk64 = K / 64;
}

__device__ __forceinline__ GemvParams make_phase(const MegaParams& mp, int layer, int kind) {
  GemvParams p = {};
  const MegaLayer& L = mp.layer[layer];
  p.tl = (mp.tl && blockIdx.x == 0) ? mp.tl + (size_t)(5 * layer + kind) * 8 : nullptr;
  if (kind == PH_QKV) {
    gemv_common(p, mp, L.wqkv, L.sqkv, (mp.Hq + 2 * mp.Hkv) * 128, mp.D, 4);
    p.pro = B200_PRO_RMSNORM;
    p.epi = B200_EPI_QKV;
    if (layer == 0) {
      p.resid = nullptr;  // token embedding row: resolved after the dependency wait (make_embed_resid)
      p.h_out = mp.h0;
    } else {
      p.resid = mp.h1, p.h_out = mp.h0;
      p.delta = reinterpret_cast<const __half*>(mp.comm[mp.tp_rank] + mp.parts_off) + (size_t)mp.tp_world * mp.D;  // w2 partials
      p.n_delta = mp.tp_world;
    }
    p.gamma = L.attn_norm;
    p.out = mp.q;
    p.n_q_rows = mp.Hq * 128, p.n_kv_rows = mp.Hkv * 128;
    p.rope = mp.rope, p.pos = mp.pos;
    p.kcache = mp.kcache + (size_t)layer * mp.kv_layer_stride;
    p.vtcache = mp.vtcache + (size_t)layer * mp.kv_layer_stride;
    p.cache_seq = mp.cache_seq, p.hkv = mp.Hkv;
  } else if (kind == PH_WO) {
    gemv_common(p, mp, L.wo, L.so, mp.D, mp.Hq * 128, 4);
    p.pro = kProAttnMerge;
    p.epi = B200_EPI_F16;
    p.xin = reinterpret_cast<const __half*>(mp.attn_ws);
    p.resid = reinterpret_cast<const __half*>(mp.attn_ws + (size_t)mp.Hq * mp.n_split * 128);
    p.n_slots = mp.n_split;
    p.n_bcast = mp.tp_world;
    for (int r = 0; r < mp.tp_world; ++r)
      p.bcast[r] = reinterpret_cast<__half*>(mp.comm[r] + mp.parts_off) + (size_t)mp.tp_rank * mp.D;
    p.out = p.bcast[mp.tp_rank];
  } else if (kind == PH_W13) {
    gemv_common(p, mp, L.w13, L.s13, 2 * mp.F, mp.D, 4);
    p.pro = B200_PRO_RMSNORM;
    p.epi = B200_EPI_SILU;
    p.resid = mp.h0, p.h_out = mp.h1;
    p.delta = reinterpret_cast<const __half*>(mp.comm[mp.tp_rank] + mp.parts_off);  // wo partials of all ranks
    p.n_delta = mp.tp_world;
    p.gamma = L.ffn_norm;
    p.out = mp.act;
  } else {  // PH_W2
    gemv_common(p, mp, L.w2, L.s2, mp.D, mp.F, 4);
    p.pro = B200_PRO_NONE;
    p.epi = B200_EPI_F16;
    p.xin = mp.act;
    p.n_bcast = mp.tp_world;
    for (int r = 0; r < mp.tp_world; ++r)
      p.bcast[r] = reinterpret_cast<__half*>(mp.comm[r] + mp.parts_off) + (size_t)(mp.tp_world + mp.tp_rank) * mp.D;
    p.out = p.bcast[mp.tp_rank];
  }
  return p;
}

__device__ __forceinline__ GemvParams make_head(const MegaParams& mp) {
  GemvParams p = {};
  gemv_common(p, mp, mp.lm_head, nullptr, mp.V, mp.D, 16);
  p.pro = B200_PRO_RMSNORM;
  p.epi = B200_EPI_F32;
  p.resid = mp.h1;
  p.delta = reinterpret_cast<const __half*>(mp.comm[mp.tp_rank] + mp.parts_off) + (size_t)mp.tp_world * mp.D;
  p.n_delta = mp.tp_world;
  p.gamma = mp.final_norm;
  p.n_bcast = mp.tp_world;
  for (int r = 0; r < mp.tp_world; ++r) p.bcast[r] = mp.comm[r] + mp.logits_off;
  p.bcast_off = mp.tp_rank * mp.V;  // this rank's slice of the vocabulary (ColumnParallelLinear output, gather_output=True)
  p.out = p.bcast[mp.tp_rank];
  return p;
}

// ---- attention phase -------------------------------------------------------------------------------------------
struct AttnItem {
  int kvh, split, s_begin, s_end, n_tiles;
};
__device__ __forceinline__ AttnItem attn_item(const MegaParams& mp, int item, int kv_len) {
  AttnItem it;
  it.kvh = item / mp.n_split;
  it.split = item % mp.n_split;
  const int chunk = ((kv_len + mp.n_split - 1) / mp.n_split + kTileKV - 1) / kTileKV * kTileKV;
  it.s_begin = it.split * chunk;
  it.s_end = min(kv_len, it.s_begin + chunk);
  it.n_tiles = it.s_end > it.s_begin ? (it.s_end - it.s_begin + kTileKV - 1) / kTileKV : 0;
  return it;
}

__device__ __forceinline__ int k_swz1(int row) { return (row & 1) << 2; }

// MMA warps: split-KV attention of this CTA's items for the single query token (rows = the n_rep <= 8 query heads of a
// kv head ride the M dimension; rows 8..15 of the HMMAs are zero padding).  Same math as attn.cu.
__device__ __forceinline__ void attn_mma_phase(const MegaParams& mp, const G1Smem& sm, int layer, int warp, int lane, int cta,
                                               int n_cta, G1State& st) {
  const int g = lane >> 2, t4 = lane & 3;
  const int kv_len = mp.pos[0] + 1;
  const int n_rep = mp.Hq / mp.Hkv;
  const int n_items = mp.Hkv * mp.n_split;
  float* mo = reinterpret_cast<float*>(sm.red);  // merge area [16 warps][4 rows][128] + [16][4][2]: red + scratch + xq
  float* mml = mo + kConsumerWarps * 4 * 128;
  int stage = st.stage;
  uint32_t par = st.par;
  for (int item = cta; item < n_items; item += n_cta) {
    const AttnItem it = attn_item(mp, item, kv_len);
    // ---- Q fragments: row g = query head kvh*n_rep + g (zero beyond n_rep), 4 chunks of 32 d ----
    uint32_t qf[4][4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      uint4 v = make_uint4(0, 0, 0, 0);
      if (g < n_rep) v = __ldcg(reinterpret_cast<const uint4*>(mp.q + ((size_t)it.kvh * n_rep + g) * 128 + c * 32 + t4 * 8));
      qf[c][0] = v.x, qf[c][1] = v.y, qf[c][2] = v.z, qf[c][3] = v.w;
    }
    float oacc[16][2];
    float m_run = -INFINITY, l_run = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) oacc[j][0] = oacc[j][1] = 0.f;

    for (int i = 0; i < it.n_tiles; ++i) {
      mbar_wait(&sm.full[stage], par);
      if ((i & (kConsumerWarps - 1)) == warp) {
        const uint8_t* ks = sm.ring + (size_t)stage * kSlotBytes;
        const uint8_t* vs = ks + kTileKV * 256;
        const int s0 = it.s_begin + i * kTileKV;
        float sacc[4][2];
#pragma unroll
        for (int X = 0; X < 4; ++X) {
          float c4[4] = {0.f, 0.f, 0.f, 0.f};
          const int row = 8 * (g >> 1) + (g & 1) + 2 * X;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const uint4 kb = lds_v4(ks + row * 256 + (((4 * c + t4) ^ k_swz1(row)) << 4));
            mma16816(c4, qf[c][0], 0u, qf[c][1], 0u, kb.x, kb.y);
            mma16816(c4, qf[c][2], 0u, qf[c][3], 0u, kb.z, kb.w);
          }
          sacc[X][0] = c4[0], sacc[X][1] = c4[1];
        }
        float tmax = -INFINITY;
#pragma unroll
        for (int X = 0; X < 4; ++X)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int s = s0 + 8 * t4 + 2 * X + e;
            sacc[X][e] = (s < it.s_end) ? sacc[X][e] * mp.scale_log2 : -INFINITY;
            tmax = fmaxf(tmax, sacc[X][e]);
          }
        tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
        tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
        const float m_new = fmaxf(m_run, tmax);  // finite: every tile has >= 1 valid position
        const float corr = exp2f(m_run - m_new);
        m_run = m_new;
        l_run *= corr;
        uint32_t pa[2][2];
#pragma unroll
        for (int X = 0; X < 4; ++X) {
          const __half2 h01 = __floats2half2_rn(exp2f(sacc[X][0] - m_run), exp2f(sacc[X][1] - m_run));
          const float2 f01 = __half22float2(h01);  // row sums from the fp16-rounded P (what the second GEMM multiplies)
          l_run += f01.x + f01.y;
          pa[X >> 1][X & 1] = *reinterpret_cast<const uint32_t*>(&h01);
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          float c4[4] = {oacc[j][0] * corr, oacc[j][1] * corr, 0.f, 0.f};
          const uint4 vb = lds_v4(vs + (8 * j + g) * 64 + (t4 << 4));
          mma16816(c4, pa[0][0], 0u, pa[0][1], 0u, vb.x, vb.y);
          mma16816(c4, pa[1][0], 0u, pa[1][1], 0u, vb.z, vb.w);
          oacc[j][0] = c4[0], oacc[j][1] = c4[1];
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.empty[stage]);
      if (++stage == mp.stages) stage = 0, par ^= 1;
    }
    l_run += __shfl_xor_sync(0xffffffffu, l_run, 1);
    l_run += __shfl_xor_sync(0xffffffffu, l_run, 2);
    // ---- merge the 16 warp partials of this item through shared memory, 4 query rows per pass, fixed warp order ----
    for (int r0 = 0; r0 < n_rep; r0 += 4) {
      if (g >= r0 && g < r0 + 4) {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          *reinterpret_cast<float2*>(mo + ((size_t)warp * 4 + (g - r0)) * 128 + 8 * j + 2 * t4) = make_float2(oacc[j][0], oacc[j][1]);
        if (t4 == 0) mml[(warp * 4 + (g - r0)) * 2 + 0] = m_run, mml[(warp * 4 + (g - r0)) * 2 + 1] = l_run;
      }
      named_bar_sync(1, kConsumerThreads);
      const int row = threadIdx.x >> 7, d = threadIdx.x & 127;  // 512 threads = 4 rows x 128 dims
      if (r0 + row < n_rep) {
        float M = -INFINITY;
#pragma unroll
        for (int w = 0; w < kConsumerWarps; ++w) M = fmaxf(M, mml[(w * 4 + row) * 2]);
        float Lsum = 0.f, o = 0.f;
#pragma unroll
        for (int w = 0; w < kConsumerWarps; ++w) {
          const float mw = mml[(w * 4 + row) * 2];
          const float f = (mw == -INFINITY) ? 0.f : exp2f(mw - M);
          Lsum += mml[(w * 4 + row) * 2 + 1] * f;
          o += mo[((size_t)w * 4 + row) * 128 + d] * f;
        }
        const int hq = it.kvh * n_rep + r0 + row;
        float* ws_o = mp.attn_ws;
        float2* ws_ml = reinterpret_cast<float2*>(mp.attn_ws + (size_t)mp.Hq * mp.n_split * 128);
        ws_o[((size_t)hq * mp.n_split + it.split) * 128 + d] = o;
        if (d == 0) ws_ml[hq * mp.n_split + it.split] = make_float2(M, Lsum);
      }
      named_bar_sync(1, kConsumerThreads);
    }
  }
  st.stage = stage, st.par = par;
}

// producer side of the attention phase: (K tile, V tile) pairs of this CTA's items; only the tile holding the row that
// the QKV phase of this step appends waits for that phase's grid barrier
__device__ __forceinline__ void attn_producer_phase(const MegaParams& mp, const G1Smem& sm, const Bars& bars, int layer, int ph,
                                                    int cta, int n_cta, G1State& st) {
  const int kv_len = mp.pos[0] + 1;
  const int n_items = mp.Hkv * mp.n_split;
  const __half* kc = mp.kcache + (size_t)layer * mp.kv_layer_stride;
  const __half* vt = mp.vtcache + (size_t)layer * mp.kv_layer_stride;
  int stage = st.stage;
  uint32_t par = st.par;
  bool waited = false;
  for (int item = cta; item < n_items; item += n_cta) {
    const AttnItem it = attn_item(mp, item, kv_len);
    const size_t kv_base = (size_t)it.kvh * mp.cache_seq * 128;
    for (int i = 0; i < it.n_tiles; ++i) {
      mbar_wait(&sm.empty[stage], par ^ 1);
      const int s0 = it.s_begin + i * kTileKV;
      if (!waited && s0 + kTileKV >= kv_len) {
        bar_wait(bars, ph - 1, 5 * mp.n_layers + 1);  // the row appended by this step's QKV phase is in global memory
        asm volatile("fence.proxy.async;" ::: "memory");
        waited = true;
      }
      uint8_t* dst = sm.ring + (size_t)stage * kSlotBytes;
      mbar_arrive_expect_tx(&sm.full[stage], 2 * kTileKV * 256);
      bulk_g2s(dst, kc + kv_base + (size_t)s0 * 128, kTileKV * 256, &sm.full[stage]);
      bulk_g2s(dst + kTileKV * 256, vt + kv_base + (size_t)s0 * 128, kTileKV * 256, &sm.full[stage]);
      if (++stage == mp.stages) stage = 0, par ^= 1;
    }
  }
  st.stage = stage, st.par = par;
}

// ---- the kernel --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 1) decode_step1_kernel(const __grid_constant__ MegaParams mp) {
  extern __shared__ __align__(128) uint8_t smem[];
  G1Smem sm;
  sm.ring = smem;
  sm.full = reinterpret_cast<uint64_t*>(smem + (size_t)mp.stages * kSlotBytes);
  sm.empty = sm.full + mp.stages;
  sm.red_full = sm.empty + mp.stages;
  sm.red_empty = sm.red_full + 2;
  uint64_t* x_ready = sm.red_empty + 2;  // fp16 lm_head phase only (+1 pad)
  sm.red = reinterpret_cast<int*>(x_ready + 2);
  sm.scratch = reinterpret_cast<float*>(sm.red + 2 * kConsumerWarps * 128);
  sm.xq = reinterpret_cast<uint8_t*>(sm.scratch + 32);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cta = blockIdx.x, n_cta = gridDim.x;
  if (tid == 0) {
    for (int s = 0; s < mp.stages; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], kConsumerWarps);
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(&sm.red_full[b], kConsumerWarps);
      mbar_init(&sm.red_empty[b], kEpiWarps);
    }
    mbar_init(x_ready, kConsumerWarps);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  const int L = mp.n_layers, n_ph = 5 * L + 1;
  unsigned* const lbar = reinterpret_cast<unsigned*>(mp.comm[mp.tp_rank]);  // [0, n_ph) counters, [n_ph] exit, [n_ph+1] epoch

  if (warp == kConsumerWarps) {
    // ================= producer: every phase's HBM stream, back to back =================
    if (lane == 0) {
      G1State st;
      bool dep = false;
      for (int l = 0; l < L; ++l) {
        {
          const GemvParams p = make_phase(mp, l, PH_QKV);
          g1_producer_phase(p, sm, cta, n_cta, st);
          mtl(mp, 5 * l + PH_QKV, 5);
        }
        if (!dep) {
          pdl_wait();  // pos[] and the epoch (and everything else of the previous step) are final
          dep = true;
        }
        const Bars bars = {lbar, lbar[n_ph + 1] + 1u, n_cta, mp.tp_world};
        attn_producer_phase(mp, sm, bars, l, 5 * l + PH_ATTN, cta, n_cta, st);
        mtl(mp, 5 * l + PH_ATTN, 5);
        {
          const GemvParams p = make_phase(mp, l, PH_WO);
          g1_producer_phase(p, sm, cta, n_cta, st);
          mtl(mp, 5 * l + PH_WO, 5);
        }
        {
          const GemvParams p = make_phase(mp, l, PH_W13);
          g1_producer_phase(p, sm, cta, n_cta, st);
          mtl(mp, 5 * l + PH_W13, 5);
        }
        {
          const GemvParams p = make_phase(mp, l, PH_W2);
          g1_producer_phase(p, sm, cta, n_cta, st);
          mtl(mp, 5 * l + PH_W2, 5);
        }
      }
      const GemvParams p = make_head(mp);
      g1_producer_phase(p, sm, cta, n_cta, st);
    }
    return;
  }

  if (warp > kConsumerWarps) {
    // ================= epilogue warps: reduce + store every GEMV phase, then arrive on its grid barrier =================
    const int etid = tid - (kConsumerWarps + 1) * 32;
    pdl_wait();
    int lt = 0;
    const unsigned epoch1 = lbar[n_ph + 1] + 1u;
    auto arrive = [&](int ph) {
      asm volatile("bar.sync 2, %0;" ::"n"(kEpiWarps * 32) : "memory");
      if (etid == 0) {
        bar_arrive(mp, ph, n_ph);
        mtl(mp, ph, 3);
      }
    };
    for (int l = 0; l < L; ++l) {
      {
        const GemvParams p = make_phase(mp, l, PH_QKV);
        g1_epilogue_phase<B200_EPI_QKV>(p, sm, etid, lane, cta, n_cta, lt);
        arrive(5 * l + PH_QKV);
      }
      {
        const GemvParams p = make_phase(mp, l, PH_WO);
        g1_epilogue_phase<B200_EPI_F16>(p, sm, etid, lane, cta, n_cta, lt);
        arrive(5 * l + PH_WO);
      }
      {
        const GemvParams p = make_phase(mp, l, PH_W13);
        g1_epilogue_phase<B200_EPI_SILU>(p, sm, etid, lane, cta, n_cta, lt);
        arrive(5 * l + PH_W13);
      }
      {
        const GemvParams p = make_phase(mp, l, PH_W2);
        g1_epilogue_phase<B200_EPI_F16>(p, sm, etid, lane, cta, n_cta, lt);
        arrive(5 * l + PH_W2);
      }
    }
    {
      const GemvParams p = make_head(mp);
      float* xsum = reinterpret_cast<float*>(sm.xq) + 32 * kConsumerWarps;
      epilogue_role<16, 1>(p, 1, nullptr, 1, false, etid, lane, reinterpret_cast<const float*>(sm.red), sm.red_full,
                           sm.red_empty, x_ready, xsum, lt, 0);
    }
    arrive(n_ph - 1);
    if (etid == 0) {
      // the logits slices of every rank have landed here before this kernel completes (the all-gather of the head)
      const Bars bars = {lbar, epoch1, n_cta, mp.tp_world};
      if (mp.tp_world > 1) bar_wait(bars, n_ph - 1, n_ph);
      // the CTA that leaves last advances the epoch for the next launch / graph replay (counters are never reset)
      const unsigned old = atomicAdd(lbar + n_ph, 1u);
      if (old + 1u == epoch1 * (unsigned)n_cta) {
        lbar[n_ph + 1] = epoch1;
        __threadfence();
      }
    }
    return;
  }

  // ================= MMA warps =================
  G1State st;
  pdl_wait();  // token / pos / caches / epoch of the previous step are final
  const Bars bars = {lbar, lbar[n_ph + 1] + 1u, n_cta, mp.tp_world};
  auto phase_gate = [&](int ph) {
    // grid barrier: phase ph reads what every CTA (of every rank, after a row-parallel phase) wrote in phase ph - 1
    if (ph > 0) {
      if (tid == 0) bar_wait(bars, ph - 1, n_ph);
      named_bar_sync(1, kConsumerThreads);
    }
    if (tid == 0) mtl(mp, ph, 0);
  };
  for (int l = 0; l < L; ++l) {
    {
      GemvParams p = make_phase(mp, l, PH_QKV);
      if (l == 0) p.resid = mp.tok_emb + (size_t)mp.token[0] * mp.D;  // ParallelEmbedding row (llama.py:399)
      phase_gate(5 * l + PH_QKV);
      g1_mma_phase<B200_PRO_RMSNORM>(p, sm, warp, lane, cta, n_cta, st);
      if (tid == 0) mtl(mp, 5 * l + PH_QKV, 2);
    }
    {
      phase_gate(5 * l + PH_ATTN);
      attn_mma_phase(mp, sm, l, warp, lane, cta, n_cta, st);
      // every store of the partials is ordered before the arrival: barrier among the MMA warps, then one release
      named_bar_sync(1, kConsumerThreads);
      if (tid == 0) {
        bar_arrive(mp, 5 * l + PH_ATTN, n_ph);
        mtl(mp, 5 * l + PH_ATTN, 2);
      }
    }
    {
      const GemvParams p = make_phase(mp, l, PH_WO);
      phase_gate(5 * l + PH_WO);
      g1_mma_phase<kProAttnMerge>(p, sm, warp, lane, cta, n_cta, st);
      if (tid == 0) mtl(mp, 5 * l + PH_WO, 2);
    }
    {
      const GemvParams p = make_phase(mp, l, PH_W13);
      phase_gate(5 * l + PH_W13);
      g1_mma_phase<B200_PRO_RMSNORM>(p, sm, warp, lane, cta, n_cta, st);
      if (tid == 0) mtl(mp, 5 * l + PH_W13, 2);
    }
    {
      const GemvParams p = make_phase(mp, l, PH_W2);
      phase_gate(5 * l + PH_W2);
      g1_mma_phase<B200_PRO_NONE>(p, sm, warp, lane, cta, n_cta, st);
      if (tid == 0) mtl(mp, 5 * l + PH_W2, 2);
    }
  }
  {
    // fp16 lm_head on the HMMA path (gemv_core.cuh); its staging buffers alias the digit-plane area
    const GemvParams p = make_head(mp);
    phase_gate(n_ph - 1);
    float* scratch = reinterpret_cast<float*>(sm.xq);         // [32][16]
    float* xsum = scratch + 32 * kConsumerWarps;               // [32]
    float* csum = xsum + 32;                                   // [n_chunk64]
    __half* xs = reinterpret_cast<__half*>(csum + ((p.n_chunk64 + 3) & ~3));
    stage_x(p, 1, nullptr, xs, csum, xsum, scratch, tid);
    if (lane == 0) mbar_arrive(x_ready);
    long long c0 = 0, c1 = 0;
    mma_phase<16, 1, 0>(p, 1, 1, false, sm.ring, sm.full, sm.empty, reinterpret_cast<float*>(sm.red), sm.red_full,
                        sm.red_empty, xs, csum, st.stage, st.par, st.lt, warp, lane, c0, c1, false);
    if (tid == 0) mtl(mp, n_ph - 1, 2);
  }
}

}  // namespace b200

using namespace b200;

extern "C" size_t b200_step1_attn_ws_bytes(int Hq, int n_split) { return (size_t)Hq * n_split * (128 * 4 + 8); }
static size_t comm_bar_bytes(int n_layers) { return ((size_t)(5 * n_layers + 3) * 4 + 255) / 256 * 256; }
extern "C" size_t b200_step1_comm_logits_offset(int n_layers, int dim, int tp_world) {
  return comm_bar_bytes(n_layers) + ((size_t)2 * tp_world * dim * 2 + 255) / 256 * 256;
}
extern "C" size_t b200_step1_comm_bytes(int n_layers, int dim, int vocab_local, int tp_world) {
  return b200_step1_comm_logits_offset(n_layers, dim, tp_world) + (size_t)vocab_local * tp_world * 4;
}

extern "C" int b200_step1_choose_split(int Hkv) {
  // one (kv head, split) item per CTA: the KV stream of a layer is spread over as many SMs as the head count allows
  static const int force = getenv("B200_STEP1_SPLIT") ? atoi(getenv("B200_STEP1_SPLIT")) : 0;
  if (force > 0) return std::min(force, 8);
  return std::max(1, std::min(8, sm_count() / std::max(Hkv, 1)));
}

extern "C" int b200_decode_step1(const b200_step1_args_t* a, b200_stream_t stream) {
  if (!a || a->n_layers < 1 || a->n_layers > kMegaMaxLayers) {
    set_error("step1: n_layers must be in 1..96");
    return B200_E_INVAL;
  }
  if (a->dim <= 0 || (a->dim & 127) || a->ffn <= 0 || (a->ffn & 127) || a->dim > 8192 || a->ffn > 16384 || a->n_heads < 1 ||
      a->n_kv_heads < 1 || a->n_heads % a->n_kv_heads || a->n_heads / a->n_kv_heads > 8 || a->n_heads * 128 > 16384 ||
      (a->vocab & 15) || (a->cache_seq % kTileKV) || a->cache_seq < kTileKV) {
    set_error("step1: unsupported shape (dim/ffn multiples of 128, head_dim 128, n_rep <= 8, vocab % 16 == 0, cache_seq % 32 == 0)");
    return B200_E_UNSUPPORTED;
  }
  if (!a->token || !a->tok_emb || !a->pos || !a->rope || !a->kcache || !a->vtcache || !a->h0 || !a->h1 || !a->q ||
      !a->act || !a->attn_ws || !a->comm || !a->wqkv || !a->wo || !a->w13 || !a->w2 ||
      !a->attn_norm || !a->ffn_norm || !a->final_norm) {
    set_error("step1: null pointer");
    return B200_E_INVAL;
  }
  if (a->tp_world < 1 || a->tp_world > 8 || a->tp_rank < 0 || a->tp_rank >= a->tp_world) {
    set_error("step1: tp_world must be 1..8 and 0 <= tp_rank < tp_world");
    return B200_E_INVAL;
  }
  for (int r = 0; r < a->tp_world; ++r)
    if (!a->comm[r]) {
      set_error("step1: null communication block");
      return B200_E_INVAL;
    }
  static MegaParams mp;  // ~8 KB: keep it off the stack of the (single) host thread per device
  memset(&mp, 0, sizeof(mp));
  mp.n_layers = a->n_layers, mp.D = a->dim, mp.Hq = a->n_heads, mp.Hkv = a->n_kv_heads, mp.F = a->ffn, mp.V = a->vocab;
  mp.cache_seq = a->cache_seq;
  mp.eps = a->eps;
  mp.scale_log2 = (1.0f / sqrtf(128.0f)) * 1.4426950408889634f;
  mp.token = reinterpret_cast<const long long*>(a->token);
  mp.tok_emb = static_cast<const __half*>(a->tok_emb);
  mp.pos = a->pos;
  mp.rope = reinterpret_cast<const float2*>(a->rope);
  mp.kcache = static_cast<__half*>(a->kcache), mp.vtcache = static_cast<__half*>(a->vtcache);
  mp.kv_layer_stride = a->kv_layer_stride;
  mp.h0 = static_cast<__half*>(a->h0), mp.h1 = static_cast<__half*>(a->h1), mp.q = static_cast<__half*>(a->q);
  mp.act = static_cast<__half*>(a->act);
  mp.tp_world = a->tp_world, mp.tp_rank = a->tp_rank;
  for (int r = 0; r < a->tp_world; ++r) mp.comm[r] = static_cast<uint8_t*>(a->comm[r]);
  mp.parts_off = (int)comm_bar_bytes(a->n_layers);
  mp.logits_off = (int)b200_step1_comm_logits_offset(a->n_layers, a->dim, a->tp_world);
  mp.attn_ws = static_cast<float*>(a->attn_ws);
  mp.final_norm = static_cast<const __half*>(a->final_norm);
  mp.tl = static_cast<unsigned long long*>(a->timeline);
  const int Nqkv = (a->n_heads + 2 * a->n_kv_heads) * 128;
  auto chk = [&](const b200_linear_t& l, int N, int K, int bits, const char* what) {
    if (l.bits != bits || l.N != N || l.K != K || !l.qweight || (bits != 16 && (!l.scales || (l.group_size > 0 && l.group_size < K)))) {
      set_error(std::string("step1: ") + what + " must be a per-channel W4 (lm_head: fp16) linear of the model's shape");
      return false;
    }
    return true;
  };
  for (int i = 0; i < a->n_layers; ++i) {
    if (!chk(a->wqkv[i], Nqkv, a->dim, 4, "wqkv") || !chk(a->wo[i], a->dim, a->n_heads * 128, 4, "wo") ||
        !chk(a->w13[i], 2 * a->ffn, a->dim, 4, "w13") || !chk(a->w2[i], a->dim, a->ffn, 4, "w2"))
      return B200_E_UNSUPPORTED;
    MegaLayer& L = mp.layer[i];
    L.wqkv = static_cast<const uint8_t*>(a->wqkv[i].qweight), L.sqkv = static_cast<const __half2*>(a->wqkv[i].scales);
    L.wo = static_cast<const uint8_t*>(a->wo[i].qweight), L.so = static_cast<const __half2*>(a->wo[i].scales);
    L.w13 = static_cast<const uint8_t*>(a->w13[i].qweight), L.s13 = static_cast<const __half2*>(a->w13[i].scales);
    L.w2 = static_cast<const uint8_t*>(a->w2[i].qweight), L.s2 = static_cast<const __half2*>(a->w2[i].scales);
    L.attn_norm = static_cast<const __half*>(a->attn_norm[i]), L.ffn_norm = static_cast<const __half*>(a->ffn_norm[i]);
  }
  if (!chk(a->lm_head, a->vocab, a->dim, 16, "lm_head")) return B200_E_UNSUPPORTED;
  mp.lm_head = static_cast<const uint8_t*>(a->lm_head.qweight);
  static const int flags = getenv("B200_STEP1_FLAGS") ? atoi(getenv("B200_STEP1_FLAGS")) : 0;
  mp.flags = flags;
  mp.n_split = a->n_split > 0 ? a->n_split : b200_step1_choose_split(a->n_kv_heads);
  if (mp.n_split > 8) mp.n_split = 8;

  // shared memory: ring | barriers | red (16 KB) | scratch | digit planes of the widest K (also: lm_head staging, attention merge)
  const int Kmax = std::max(std::max(a->dim, a->ffn), a->n_heads * 128);
  size_t xq = (size_t)kPlanes * ((((size_t)Kmax + 127) / 128) * 128 + 64);
  xq = std::max(xq, (size_t)(32 * kConsumerWarps + 32 + a->dim / 64 + 4) * 4 + (size_t)(a->dim + kXPad) * 2);  // lm_head staging
  xq = std::max(xq, (size_t)kConsumerWarps * 4 * 130 * 4);  // attention merge (starts in red; conservative)
  const size_t cap = std::min<size_t>(smem_optin(), 227 * 1024) - 6144;  // static: sz_s / rope_s of three epilogue instances
  auto total = [&](int stages) {
    return (size_t)stages * kSlotBytes + (size_t)stages * 16 + 6 * 8 + (size_t)2 * kConsumerWarps * 128 * 4 + 32 * 4 + xq;
  };
  static const int ring_kb = getenv("B200_STEP1_RING_KB") ? atoi(getenv("B200_STEP1_RING_KB")) : 192;
  int stages = std::max(2, std::min(ring_kb * 1024 / kSlotBytes, 12));
  while (stages > 2 && total(stages) > cap) --stages;
  if (total(stages) > cap) {
    set_error("step1: shared memory budget exceeded");
    return B200_E_UNSUPPORTED;
  }
  mp.stages = stages;
  mp.xq_bytes = (int)xq;
  const size_t smem = total(stages);
  static size_t configured[16] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  dev &= 15;
  if (smem > configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(decode_step1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      set_error(std::string("step1: cudaFuncSetAttribute: ") + cudaGetErrorString(e));
      return (int)e;
    }
    configured[dev] = smem;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(sm_count());  // one CTA per SM: every CTA is resident, as the grid barriers require
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[2];
  int na = 0;
  static const int coop = getenv("B200_STEP1_COOP") ? atoi(getenv("B200_STEP1_COOP")) : 1;
  if (coop) {
    attr[na].id = cudaLaunchAttributeCooperative;  // fail the launch instead of deadlocking if the grid cannot be co-resident
    attr[na].val.cooperative = 1;
    ++na;
  }
  if (a->use_pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  cudaError_t e = cudaLaunchKernelEx(&cfg, decode_step1_kernel, mp);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    set_error(std::string("step1: launch: ") + cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}
