// Persistent whole-step kernel, DATAFLOW version: one bs = 1 decode step of a dense LLaMA per launch and tensor-parallel
// rank, WITHOUT grid barriers.  (mega1.cu is the grid-barrier version of the same step.)
//
// What the timeline of mega1 showed: every phase boundary cost
// three dependent global round trips under streaming load -- stores + fence + arrive, poll the counter, load x -- five
// phases per layer.  Here every vector that crosses CTAs travels in the "flag-in-data" format of
// low-latency collectives (NCCL's LL protocol): 8-byte units {payload, sequence number}, written with one 8-byte store
// (single-copy atomic) and polled by the consumer until the sequence number of the producing phase appears.  A consumer
// therefore sees its input ONE round trip after the producer's store lands; there is no fence, no counter, no barrier:
//   * GEMV epilogues store {half2(y[2i], y[2i+1]), seq}; attention stores {float, seq};
//   * every MMA warp polls exactly the slice of the next activation vector it multiplies itself;
//   * the residual stream h never goes to global memory: every CTA keeps its own copy in shared memory and adds the
//     (rank-summed) wo / w2 outputs to it while staging -- all CTAs compute identical values (fixed order);
//   * the K/V row of the current position is patched into the last KV tile in shared memory from an LL copy, so the
//     producer warp never waits for anything but a free ring slot;
//   * tensor parallelism: row-parallel partial sums are LL-stored into EVERY rank's buffer over NVLink and added in rank
//     order (fp32, one rounding) by the consumer -- the all-reduce of reduce_from_model_parallel_region (quant.py:41)
//     costs one NVLink store latency and no kernel.  Only the vocabulary-sharded logits need one barrier at the end.
// Reuse across layers / launches is safe without barriers: a CTA can only enter phase p+1 after EVERY CTA (of every rank,
// for row-parallel outputs) has written its phase-p output, i.e. has finished reading its phase-p inputs; buffers are
// rewritten five phases later.  Sequence numbers (launch epoch * phases + phase + 1) never repeat.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>

#include "gemv1_core.cuh"

namespace b200 {
namespace ll {

constexpr int kMaxLayers = 96;
constexpr int kTileKV = 32;
constexpr int kMaxSplit = 8;

struct Layer {
  const uint8_t *wqkv, *wo, *w13, *w2;
  const __half2 *sqkv, *so, *s13, *s2;
  const __half *attn_norm, *ffn_norm;
};

// Communication block of a rank (same layout on every rank; peer-mapped when tp_world > 1).  Offsets in bytes.
struct CommLayout {
  int ctl;      // u32 exit counter, u32 epoch, u32 error, u32 final-barrier counter, then u32 hint[5L+1] (see hint_wait)
  int yq;       // LL half pairs  [Hq*128/2]
  int ykv;      // LL half pairs  [Hkv][2][64]
  int att;      // LL floats      [Hq][n_split][130]   (O[128], m, l)
  int po;       // LL half pairs  [tp][D/2]             wo partial sums, slot r written by rank r
  int act;      // LL half pairs  [F/2]
  int pf;       // LL half pairs  [tp][D/2]             w2 partial sums
  int logits;   // fp32           [V * tp]
  int total;
};

struct Params {
  int n_layers, D, Hq, Hkv, F, V, cache_seq, stages, n_split;
  int tp_world, tp_rank;
  int flags;  // B200_STEP1_FLAGS: 2 = no hint gate (every thread polls the data from the start), 4 = scales staged in-phase
  float eps, scale_log2;
  const long long* token;
  const __half* tok_emb;
  const int* pos;
  const float2* rope;
  __half* kcache;
  __half* vtcache;
  long long kv_layer_stride;
  const uint8_t* lm_head;
  const __half* final_norm;
  uint8_t* comm[8];
  CommLayout lay;
  unsigned long long* tl;  // optional [5L+1][8] ns stamps of CTA 0: 0 inputs valid, 1 x staged, 2 tiles done, 3 epilogue stored
  Layer layer[kMaxLayers];
};

// "The producers of phase ph are probably done" hint: one relaxed counter per phase, bumped (no fence) by every CTA after
// its LL stores and watched by ONE thread per consumer CTA.  It only gates WHEN the consumers start polling the data (75 000
// threads spinning on not-yet-written units took about half of the L2's request rate); correctness still rests on the sequence numbers inside the data.
__device__ __forceinline__ unsigned* hint_ptr(const Params& mp, int rank, int ph) {
  return reinterpret_cast<unsigned*>(mp.comm[rank] + mp.lay.ctl + 64) + ph;
}
__device__ __forceinline__ bool phase_is_cross(int ph, int n_ph) { return ph != n_ph - 1 && ((ph % 5) == 2 || (ph % 5) == 4); }
__device__ __forceinline__ void hint_bump(const Params& mp, int ph, int n_ph) {
  if (mp.tp_world > 1 && phase_is_cross(ph, n_ph)) {
    for (int r = 0; r < mp.tp_world; ++r)
      asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(hint_ptr(mp, r, ph)), "r"(1u) : "memory");
  } else {
    asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(hint_ptr(mp, mp.tp_rank, ph)), "r"(1u) : "memory");
  }
}
__device__ __forceinline__ void hint_wait(const Params& mp, int ph, int n_ph, unsigned epoch1, int n_cta) {
  const bool cross = mp.tp_world > 1 && phase_is_cross(ph, n_ph);
  const unsigned target = epoch1 * (unsigned)(n_cta * (cross ? mp.tp_world : 1));
  const unsigned* p = hint_ptr(mp, mp.tp_rank, ph);
  unsigned v, spins = 0;
  do {
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  } while ((int)(v - target) < 0 && ++spins < kSpinCap);  // on a time-out the data polls below report the error
}

__device__ __forceinline__ void mtl(const Params& mp, int ph, int k) {
  if (mp.tl && blockIdx.x == 0) mp.tl[ph * 8 + k] = gtime_ns();
}

enum { PH_QKV = 0, PH_ATTN = 1, PH_WO = 2, PH_W13 = 3, PH_W2 = 4 };

__device__ __forceinline__ void gemv_common(GemvParams& p, const Params& mp, const uint8_t* qw, const __half2* sz, int N, int K,
                                            int bits) {
  p.bits = bits;
  p.qw = qw;
  p.sz = sz;
  p.N = N;
  p.K = K;
  p.KB = K / (bits == 4 ? 64 : 16);
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
// weights / shapes of a GEMV phase (the data pointers of the activations are handled by the LL staging / epilogue code)
__device__ __forceinline__ GemvParams make_phase(const Params& mp, int layer, int kind) {
  GemvParams p = {};
  const Layer& L = mp.layer[layer];
  if (kind == PH_QKV) {
    gemv_common(p, mp, L.wqkv, L.sqkv, (mp.Hq + 2 * mp.Hkv) * 128, mp.D, 4);
    p.gamma = L.attn_norm;
    p.n_q_rows = mp.Hq * 128, p.n_kv_rows = mp.Hkv * 128;
    p.kcache = mp.kcache + (size_t)layer * mp.kv_layer_stride;
    p.vtcache = mp.vtcache + (size_t)layer * mp.kv_layer_stride;
    p.cache_seq = mp.cache_seq, p.hkv = mp.Hkv;
  } else if (kind == PH_WO) {
    gemv_common(p, mp, L.wo, L.so, mp.D, mp.Hq * 128, 4);
  } else if (kind == PH_W13) {
    gemv_common(p, mp, L.w13, L.s13, 2 * mp.F, mp.D, 4);
    p.gamma = L.ffn_norm;
  } else {
    gemv_common(p, mp, L.w2, L.s2, mp.D, mp.F, 4);
  }
  return p;
}
__device__ __forceinline__ GemvParams make_head(const Params& mp) {
  GemvParams p = {};
  gemv_common(p, mp, mp.lm_head, nullptr, mp.V, mp.D, 16);
  p.pro = B200_PRO_RMSNORM;
  p.epi = B200_EPI_F32;
  p.gamma = mp.final_norm;
  if (mp.tp_world > 1) {
    p.n_bcast = mp.tp_world;
    for (int r = 0; r < mp.tp_world; ++r) p.bcast[r] = mp.comm[r] + mp.lay.logits;
    p.bcast_off = mp.tp_rank * mp.V;
  }
  p.out = mp.comm[mp.tp_rank] + mp.lay.logits;
  return p;
}

// ---- MMA-warp staging: every warp produces the digit planes of the slice of x it multiplies itself ---------------------
// lane -> 8-element piece `it` of the warp's slice: element offset, or -1
__device__ __forceinline__ int piece_e0(int it, int warp, int lane, int KB, int slots_per_tile) {
  const int half = lane >> 4, sub = lane & 15;
  const int s = 2 * it + half;
  const int blk = s * kSlotBlocks + warp * kChunk + (sub >> 3);
  return (s < slots_per_tile && blk < KB) ? blk * 64 + (sub & 7) * 8 : -1;
}

// RMSNorm phases (QKV, W13, head): h (shared-memory copy of the residual stream) += sum of rank partials; x = norm(h) * gamma.
// Returns the warp's sum of x; when xs_out != nullptr the fp16 x is written there instead of digit planes (head phase).
__device__ __forceinline__ float stage_norm(const Params& mp, const GemvParams& p, const G1Smem& sm, __half* hs,
                                            const uint8_t* parts, uint32_t seq, bool has_delta, const __half* emb_row,
                                            __half* xs_out, int warp, int lane, unsigned* err) {
  const int slots_per_tile = (mp.D / 64 + kSlotBlocks - 1) / kSlotBlocks;  // slices are defined by the W4 k-blocks of K = D
  const int KB = mp.D / 64;
  const int xq_stride = (((mp.D + 127) >> 7) << 7) + 64;
  uint4 hv[2], gv[2];
  int e0s[2];
  float ssq = 0.f;
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    e0s[it] = piece_e0(it, warp, lane, KB, slots_per_tile);
    hv[it] = gv[it] = make_uint4(0, 0, 0, 0);
    if (e0s[it] >= 0) {
      gv[it] = *reinterpret_cast<const uint4*>(p.gamma + e0s[it]);
      uint4 a = emb_row ? *reinterpret_cast<const uint4*>(emb_row + e0s[it]) : *reinterpret_cast<const uint4*>(hs + e0s[it]);
      if (has_delta) {
        const uint4 b = ll_rank_sum8(parts, mp.D, mp.tp_world, e0s[it], seq, err);
        __half2* ha = reinterpret_cast<__half2*>(&a);
        const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
        for (int j = 0; j < 4; ++j) ha[j] = __hadd2(ha[j], hb[j]);  // the reference's fp16 residual add (llama.py:286-287)
      }
      *reinterpret_cast<uint4*>(hs + e0s[it]) = a;  // own slice of the CTA's residual-stream copy
      hv[it] = a;
      const __half2* h = reinterpret_cast<const __half2*>(&a);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        ssq = fmaf(f.x, f.x, ssq);
        ssq = fmaf(f.y, f.y, ssq);
      }
    }
  }
  ssq = warp_sum(ssq);
  if (lane == 0) sm.scratch[warp] = ssq;
  named_bar_sync(1, kConsumerThreads);
  float tot = 0.f;
#pragma unroll
  for (int wi = 0; wi < kConsumerWarps; ++wi) tot += sm.scratch[wi];
  const float rstd = 1.0f / sqrtf(tot / (float)mp.D + mp.eps);
  float xs = 0.f;
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    if (e0s[it] >= 0) {
      uint4 xo;
      const __half2* h = reinterpret_cast<const __half2*>(&hv[it]);
      const __half2* gh = reinterpret_cast<const __half2*>(&gv[it]);
      __half2* o = reinterpret_cast<__half2*>(&xo);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        o[j] = __hmul2(__floats2half2_rn(f.x * rstd, f.y * rstd), gh[j]);  // components.py:52-53 rounding points
      }
      if (xs_out) {
        *reinterpret_cast<uint4*>(xs_out + e0s[it]) = xo;
        xs += hsum8(xo);
      } else {
        xs += stage_piece(xo, sm.xq, xq_stride, e0s[it]);
      }
    }
  }
  named_bar_sync(1, kConsumerThreads);  // scratch may be reused; (head phase) every warp reads all of xs_out
  return warp_sum(xs);
}

// W2 phase: x = act (LL half vector, K = F)
__device__ __forceinline__ float stage_plain(const Params& mp, const GemvParams& p, const G1Smem& sm, const uint8_t* vec,
                                             uint32_t seq, int warp, int lane, unsigned* err) {
  const int slots_per_tile = (p.KB + kSlotBlocks - 1) / kSlotBlocks;
  const int xq_stride = (((p.K + 127) >> 7) << 7) + 64;
  float xs = 0.f;
  const uint8_t* ptr[4];
  bool on[4];
  int e0s[4];
  uint4 pay[4];
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    e0s[it] = piece_e0(it, warp, lane, p.KB, slots_per_tile);
    on[it] = e0s[it] >= 0;
    ptr[it] = vec + (size_t)max(e0s[it], 0) * 4;
  }
  ll_poll32<4>(ptr, on, seq, pay, err);
#pragma unroll
  for (int it = 0; it < 4; ++it)
    if (on[it]) xs += stage_piece(pay[it], sm.xq, xq_stride, e0s[it]);
  return warp_sum(xs);
}

// WO phase: x = attention output = merge of the split-KV partials (LL floats [Hq][n_split][130]) of the lane's head
__device__ __forceinline__ float stage_attn_merge(const Params& mp, const GemvParams& p, const G1Smem& sm, const uint8_t* att,
                                                  uint32_t seq, int warp, int lane, unsigned* err) {
  const int slots_per_tile = (p.KB + kSlotBlocks - 1) / kSlotBlocks;
  const int xq_stride = (((p.K + 127) >> 7) << 7) + 64;
  const int ns = mp.n_split;
  float xs = 0.f;
  for (int it = 0; it < 4; ++it) {
    const int e0 = piece_e0(it, warp, lane, p.KB, slots_per_tile);
    if (e0 < 0) continue;
    const int hq = e0 >> 7, d0 = e0 & 127;
    const uint8_t* base = att + (size_t)hq * ns * 130 * 8;
    // (m, l) of every split: one batch
    const uint8_t* mp_ptr[kMaxSplit];
    bool on[kMaxSplit];
    uint2 ml[kMaxSplit];
#pragma unroll
    for (int sp = 0; sp < kMaxSplit; ++sp) on[sp] = sp < ns, mp_ptr[sp] = base + ((size_t)min(sp, ns - 1) * 130 + 128) * 8;
    ll_poll16<kMaxSplit>(mp_ptr, on, seq, ml, err);
    float M = -INFINITY;
#pragma unroll
    for (int sp = 0; sp < kMaxSplit; ++sp)
      if (sp < ns) M = fmaxf(M, __uint_as_float(ml[sp].x));
    float Lsum = 0.f, acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    // O[d0 .. d0+7] of the splits, two splits (4 blocks of 32 bytes) per batch, accumulated in split order
    for (int sp0 = 0; sp0 < ns; sp0 += 2) {
      const uint8_t* optr[4];
      bool oon[4];
      uint4 ov[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int sp = sp0 + (u >> 1);
        oon[u] = sp < ns;
        optr[u] = base + ((size_t)min(sp, ns - 1) * 130 + d0 + (u & 1) * 4) * 8;
      }
      ll_poll32<4>(optr, oon, seq, ov, err);
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const int sp = sp0 + h2;
        if (sp < ns) {
          float mv = 0.f, lv = 0.f;
#pragma unroll
          for (int q = 0; q < kMaxSplit; ++q)
            if (q == sp) mv = __uint_as_float(ml[q].x), lv = __uint_as_float(ml[q].y);
          const float f = (mv == -INFINITY) ? 0.f : exp2f(mv - M);
          Lsum += lv * f;
          const uint4 lo = ov[2 * h2], hi = ov[2 * h2 + 1];
          acc[0] += __uint_as_float(lo.x) * f, acc[1] += __uint_as_float(lo.y) * f;
          acc[2] += __uint_as_float(lo.z) * f, acc[3] += __uint_as_float(lo.w) * f;
          acc[4] += __uint_as_float(hi.x) * f, acc[5] += __uint_as_float(hi.y) * f;
          acc[6] += __uint_as_float(hi.z) * f, acc[7] += __uint_as_float(hi.w) * f;
        }
      }
    }
    uint4 xo;
    __half2* xh = reinterpret_cast<__half2*>(&xo);
#pragma unroll
    for (int j = 0; j < 4; ++j) xh[j] = __floats2half2_rn(acc[2 * j] / Lsum, acc[2 * j + 1] / Lsum);  // fp16 like SDPA's output
    xs += stage_piece(xo, sm.xq, xq_stride, e0);
  }
  return warp_sum(xs);
}

// ---- epilogue warps: reduce the integer partials of a tile, scale, fused epilogue, LL stores ---------------------------
// kind: PH_QKV (RoPE + cache append + LL q / fresh k, v), PH_WO / PH_W2 (LL partial sums to every rank), PH_W13 (SiLU * mul)
constexpr int kMaxLocal = 16;
struct EpiStage {
  __half2 (*sz)[kMaxLocal * 16];  // [2][256] double buffer of (s, z): phase number & 1
  float2* rope;                   // [256] RoPE factors (QKV phases only; single buffer: one QKV phase per 5)
};
// issue the asynchronous copies of a phase's scales (and RoPE factors) into the buffer the NEXT epilogue_ll call reads
__device__ __forceinline__ void epi_prefetch(const Params& mp, const GemvParams& p, const EpiStage& es, int buf, bool qkv,
                                             int etid, int cta, int n_cta) {
  const int tile_begin = (int)(((long long)p.n_tiles * cta) / n_cta);
  const int tile_end = (int)(((long long)p.n_tiles * (cta + 1)) / n_cta);
  const int n_local = tile_end - tile_begin;
  for (int i = etid; i < n_local * 16 && n_local <= kMaxLocal; i += kEpiWarps * 32) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(&es.sz[buf][i])), "l"(p.sz + (size_t)tile_begin * 16 + i) : "memory");
    if (qkv) {
      const int row = tile_begin * 16 + i;
      const bool rot = row < p.n_q_rows + p.n_kv_rows;
      const int d = (row < p.n_q_rows ? row : row - p.n_q_rows) & 127;
      if (rot)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(&es.rope[i])), "l"(mp.rope + (size_t)mp.pos[0] * 64 + (d >> 1)) : "memory");
      else
        es.rope[i] = make_float2(1.f, 0.f);
    }
  }
  cp_async_commit();
}

template <int KIND>
__device__ __forceinline__ void epilogue_ll(const Params& mp, const GemvParams& p, const G1Smem& sm, const EpiStage& es, int buf,
                                            uint32_t seq, int etid, int lane, int cta, int n_cta, int& lt_io) {
  const int tile_begin = (int)(((long long)p.n_tiles * cta) / n_cta);
  const int tile_end = (int)(((long long)p.n_tiles * (cta + 1)) / n_cta);
  // scales (and RoPE factors) of this CTA's tiles were prefetched into shared memory during the PREVIOUS phase
  // (epi_prefetch below): a dependent global load at the start of a 1-2 tile phase would sit on its critical path
  const int n_local = tile_end - tile_begin;
  const bool staged = n_local <= kMaxLocal;
  int ps = 0;
  if (KIND == PH_QKV) ps = mp.pos[0];
  const __half2* sz_s = es.sz[buf];
  const float2* rope_s = es.rope;
  cp_async_wait<1>();  // everything but the prefetch of the NEXT phase (the most recent group) has landed
  asm volatile("bar.sync 2, %0;" ::"n"(kEpiWarps * 32) : "memory");  // every thread's prefetch for this phase has landed
  const int c = etid & 7, r0 = etid >> 3;
  const float pw = c < kPlanes ? __int_as_float((127 + 7 * c - 28) << 23) : 0.f;
  uint8_t* const comm = mp.comm[mp.tp_rank];
  int lt = lt_io;
  for (int tile = tile_begin, li = 0; tile < tile_end; ++tile, ++lt, ++li) {
    const int buf = lt & 1;
    __half2 sza, szb;
    if (staged) {
      sza = sz_s[li * 16 + r0], szb = sz_s[li * 16 + r0 + 8];
    } else {
      sza = p.sz[(size_t)tile * 16 + r0], szb = p.sz[(size_t)tile * 16 + r0 + 8];
    }
    float2 cs[2];
    if (KIND == PH_QKV) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = tile * 16 + r0 + 8 * hh;
        const bool rot = row < p.n_q_rows + p.n_kv_rows;
        const int d = (row < p.n_q_rows ? row : row - p.n_q_rows) & 127;
        cs[hh] = staged ? rope_s[li * 16 + r0 + 8 * hh] : (rot ? mp.rope[(size_t)ps * 64 + (d >> 1)] : make_float2(1.f, 0.f));
      }
    }
    mbar_wait(&sm.red_full[buf], (lt >> 1) & 1);
    const int* rbase = sm.red + (size_t)buf * kConsumerWarps * 128;
    float y[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = r0 + 8 * hh;
      int isum = 0;
      float fsum = 0.f;
#pragma unroll
      for (int wi = 0; wi < kConsumerWarps; ++wi) {
        const int vv = rbase[wi * 128 + r * 8 + c];
        isum += vv;
        fsum += __int_as_float(vv);
      }
      float f = c < kPlanes ? (float)isum * pw : 0.f;
      f += __shfl_xor_sync(0xffffffffu, f, 1);
      f += __shfl_xor_sync(0xffffffffu, f, 2);
      f += __shfl_xor_sync(0xffffffffu, f, 4);
      const float xsum = __shfl_sync(0xffffffffu, fsum, (lane & 24) | 6);
      const __half2 szv = hh ? szb : sza;
      y[hh] = __low2float(szv) * (f - __high2float(szv) * xsum);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.red_empty[buf]);
    // lanes r0 and r0 ^ 1 (lane ^ 8) hold an adjacent row pair: the even one stores the 8-byte LL unit
    const bool storer = (c == 0) && ((r0 & 1) == 0);
    if (KIND == PH_W13) {
      const __half a = __float2half_rn(y[0]), b = __float2half_rn(y[1]);
      const float af = __half2float(a);
      const __half sl = __float2half_rn(af / (1.0f + expf(-af)));  // F.silu in fp32, rounded to fp16 (llama.py:252-256)
      const __half mine = __hmul(sl, b);                            // output element tile*8 + r0
      const unsigned other = __shfl_xor_sync(0xffffffffu, (unsigned)__half_as_ushort(mine), 8);
      if (storer) ll_store(comm + mp.lay.act + (size_t)(tile * 8 + r0) * 4, (unsigned)__half_as_ushort(mine) | (other << 16), seq);
    } else {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = r0 + 8 * hh, row = tile * 16 + r;
        const __half y16 = __float2half_rn(y[hh]);
        if (KIND == PH_WO || KIND == PH_W2) {
          const unsigned other = __shfl_xor_sync(0xffffffffu, (unsigned)__half_as_ushort(y16), 8);
          if (storer) {
            const unsigned pay = (unsigned)__half_as_ushort(y16) | (other << 16);
            const size_t off = (size_t)(KIND == PH_WO ? mp.lay.po : mp.lay.pf) + ((size_t)mp.tp_rank * mp.D + row) * 4;
            for (int rr = 0; rr < mp.tp_world; ++rr) ll_store(mp.comm[rr] + off, pay, seq);  // the all-reduce's data movement
          }
        } else {  // PH_QKV
          const float mine = __half2float(y16);
          const float oth = __shfl_xor_sync(0xffffffffu, mine, 8);  // row r ^ 1
          const bool is_v = row >= p.n_q_rows + p.n_kv_rows;
          const int local = row < p.n_q_rows ? row : (is_v ? row - p.n_q_rows - p.n_kv_rows : row - p.n_q_rows);
          const int head = local >> 7, d = local & 127;
          float val = mine;
          if (!is_v) {  // interleaved-pair complex rotation in fp32 (llama.py:67-77), no FMA contraction
            const float xe = (r & 1) ? oth : mine, xo = (r & 1) ? mine : oth;
            val = (r & 1) ? __fadd_rn(__fmul_rn(xe, cs[hh].y), __fmul_rn(xo, cs[hh].x))
                          : __fsub_rn(__fmul_rn(xe, cs[hh].x), __fmul_rn(xo, cs[hh].y));
          }
          const __half o16 = __float2half_rn(val);
          const unsigned o_other = __shfl_xor_sync(0xffffffffu, (unsigned)__half_as_ushort(o16), 8);
          if (c == 0 && row >= p.n_q_rows) {  // cache append for the following steps (llama.py:166-168)
            if (!is_v)
              p.kcache[((size_t)head * p.cache_seq + ps) * 128 + ((((d >> 3) ^ ((ps & 1) << 2)) << 3) | (d & 7))] = o16;
            else
              p.vtcache[(size_t)head * p.cache_seq * 128 + (size_t)(ps >> 5) * 4096 + d * 32 + (ps & 31)] = o16;
          }
          if (storer) {
            const unsigned pay = (unsigned)__half_as_ushort(o16) | (o_other << 16);
            if (row < p.n_q_rows)
              ll_store(comm + mp.lay.yq + (size_t)row * 4, pay, seq);
            else
              ll_store(comm + mp.lay.ykv + ((size_t)(head * 2 + (is_v ? 1 : 0)) * 128 + d) * 4, pay, seq);
          }
        }
      }
    }
  }
  lt_io = lt;
}

// ---- attention phase ----------------------------------------------------------------------------------------------------
struct AttnItem {
  int kvh, split, s_begin, s_end, n_tiles;
};
__device__ __forceinline__ AttnItem attn_item(const Params& mp, int item, int kv_len) {
  AttnItem it;
  it.kvh = item / mp.n_split;
  it.split = item % mp.n_split;
  const int chunk = ((kv_len + mp.n_split - 1) / mp.n_split + kTileKV - 1) / kTileKV * kTileKV;
  it.s_begin = it.split * chunk;
  it.s_end = min(kv_len, it.s_begin + chunk);
  it.n_tiles = it.s_end > it.s_begin ? (it.s_end - it.s_begin + kTileKV - 1) / kTileKV : 0;
  return it;
}

__device__ __forceinline__ void attn_producer_phase(const Params& mp, const G1Smem& sm, int layer, int cta, int n_cta,
                                                    G1State& st) {
  const int kv_len = mp.pos[0] + 1;
  const int n_items = mp.Hkv * mp.n_split;
  const __half* kc = mp.kcache + (size_t)layer * mp.kv_layer_stride;
  const __half* vt = mp.vtcache + (size_t)layer * mp.kv_layer_stride;
  int stage = st.stage;
  uint32_t par = st.par;
  for (int item = cta; item < n_items; item += n_cta) {
    const AttnItem it = attn_item(mp, item, kv_len);
    const size_t kv_base = (size_t)it.kvh * mp.cache_seq * 128;
    for (int i = 0; i < it.n_tiles; ++i) {
      mbar_wait(&sm.empty[stage], par ^ 1);
      const int s0 = it.s_begin + i * kTileKV;
      uint8_t* dst = sm.ring + (size_t)stage * kSlotBytes;
      mbar_arrive_expect_tx(&sm.full[stage], 2 * kTileKV * 256);
      bulk_g2s(dst, kc + kv_base + (size_t)s0 * 128, kTileKV * 256, &sm.full[stage]);
      bulk_g2s(dst + kTileKV * 256, vt + kv_base + (size_t)s0 * 128, kTileKV * 256, &sm.full[stage]);
      if (++stage == mp.stages) stage = 0, par ^= 1;
    }
  }
  st.stage = stage, st.par = par;
}

__device__ __forceinline__ int k_swz1(int row) { return (row & 1) << 2; }

__device__ __forceinline__ void attn_mma_phase(const Params& mp, const G1Smem& sm, uint32_t seq_in, uint32_t seq_out, int warp,
                                               int lane, int cta, int n_cta, G1State& st, unsigned* err) {
  const int g = lane >> 2, t4 = lane & 3;
  const int kv_len = mp.pos[0] + 1;
  const int n_rep = mp.Hq / mp.Hkv;
  const int n_items = mp.Hkv * mp.n_split;
  const uint8_t* comm = mp.comm[mp.tp_rank];
  float* mo = reinterpret_cast<float*>(sm.xq);  // merge area [16 warps][4 rows][128] + [16][4][2] in the digit-plane area
  float* mml = mo + kConsumerWarps * 4 * 128;
  int stage = st.stage;
  uint32_t par = st.par;
  for (int item = cta; item < n_items; item += n_cta) {
    const AttnItem it = attn_item(mp, item, kv_len);
    // ---- Q fragments: row g = query head kvh*n_rep + g (zero beyond n_rep), 4 chunks of 32 d; LL vector yq ----
    uint32_t qf[4][4];
    {
      const uint8_t* qptr[4];
      bool qon[4];
      uint4 qv[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        qon[c] = g < n_rep;
        qptr[c] = comm + mp.lay.yq + (size_t)((it.kvh * n_rep + min(g, n_rep - 1)) * 128 + c * 32 + t4 * 8) * 4;
        qv[c] = make_uint4(0, 0, 0, 0);
      }
      ll_poll32<4>(qptr, qon, seq_in, qv, err);
#pragma unroll
      for (int c = 0; c < 4; ++c) qf[c][0] = qv[c].x, qf[c][1] = qv[c].y, qf[c][2] = qv[c].z, qf[c][3] = qv[c].w;
    }
    float oacc[16][2];
    float m_run = -INFINITY, l_run = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) oacc[j][0] = oacc[j][1] = 0.f;

    for (int i = 0; i < it.n_tiles; ++i) {
      mbar_wait(&sm.full[stage], par);
      if ((i & (kConsumerWarps - 1)) == warp) {
        uint8_t* ks = sm.ring + (size_t)stage * kSlotBytes;
        uint8_t* vs = ks + kTileKV * 256;
        const int s0 = it.s_begin + i * kTileKV;
        if (s0 + kTileKV >= kv_len) {
          // this tile holds the position being decoded: its K / V row is being written to the cache right now, so patch
          // the shared-memory copy from the LL copy of the fresh rows (only this warp reads this tile)
          const int prow = (kv_len - 1) - s0;
          const uint8_t* kvp[2] = {comm + mp.lay.ykv + ((size_t)(it.kvh * 2 + 0) * 128 + lane * 4) * 4,
                                   comm + mp.lay.ykv + ((size_t)(it.kvh * 2 + 1) * 128 + lane * 4) * 4};
          const bool kvon[2] = {true, true};
          uint2 kvv[2];
          ll_poll16<2>(kvp, kvon, seq_in, kvv, err);
          const uint2 kk = kvv[0], vv = kvv[1];
          const int d = lane * 4;  // 4 consecutive dims per lane
          *reinterpret_cast<uint2*>(ks + prow * 256 + ((((d >> 3) ^ k_swz1(prow)) << 4) | ((d & 7) * 2))) = kk;
          __half* vsh = reinterpret_cast<__half*>(vs);
          vsh[(d + 0) * 32 + prow] = __ushort_as_half((unsigned short)(vv.x & 0xffff));
          vsh[(d + 1) * 32 + prow] = __ushort_as_half((unsigned short)(vv.x >> 16));
          vsh[(d + 2) * 32 + prow] = __ushort_as_half((unsigned short)(vv.y & 0xffff));
          vsh[(d + 3) * 32 + prow] = __ushort_as_half((unsigned short)(vv.y >> 16));
          __syncwarp();
        }
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
        const float m_new = fmaxf(m_run, tmax);
        const float corr = exp2f(m_run - m_new);
        m_run = m_new;
        l_run *= corr;
        uint32_t pa[2][2];
#pragma unroll
        for (int X = 0; X < 4; ++X) {
          const __half2 h01 = __floats2half2_rn(exp2f(sacc[X][0] - m_run), exp2f(sacc[X][1] - m_run));
          const float2 f01 = __half22float2(h01);
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
    for (int r0 = 0; r0 < n_rep; r0 += 4) {
      if (g >= r0 && g < r0 + 4) {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          *reinterpret_cast<float2*>(mo + ((size_t)warp * 4 + (g - r0)) * 128 + 8 * j + 2 * t4) = make_float2(oacc[j][0], oacc[j][1]);
        if (t4 == 0) mml[(warp * 4 + (g - r0)) * 2 + 0] = m_run, mml[(warp * 4 + (g - r0)) * 2 + 1] = l_run;
      }
      named_bar_sync(1, kConsumerThreads);
      const int row = threadIdx.x >> 7, d = threadIdx.x & 127;
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
        uint8_t* base = mp.comm[mp.tp_rank] + mp.lay.att + ((size_t)hq * mp.n_split + it.split) * 130 * 8;
        ll_store(base + (size_t)d * 8, __float_as_uint(o), seq_out);
        if (d == 0) {
          ll_store(base + 128 * 8, __float_as_uint(M), seq_out);
          ll_store(base + 129 * 8, __float_as_uint(Lsum), seq_out);
        }
      }
      named_bar_sync(1, kConsumerThreads);
    }
  }
  st.stage = stage, st.par = par;
}

// ---- the kernel -----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 1) decode_step1_ll_kernel(const __grid_constant__ Params mp) {
  extern __shared__ __align__(128) uint8_t smem[];
  G1Smem sm;
  sm.ring = smem;
  sm.full = reinterpret_cast<uint64_t*>(smem + (size_t)mp.stages * kSlotBytes);
  sm.empty = sm.full + mp.stages;
  sm.red_full = sm.empty + mp.stages;
  sm.red_empty = sm.red_full + 2;
  uint64_t* x_ready = sm.red_empty + 2;
  sm.red = reinterpret_cast<int*>(x_ready + 2);
  sm.scratch = reinterpret_cast<float*>(sm.red + 2 * kConsumerWarps * 128);
  __half* hs = reinterpret_cast<__half*>(sm.scratch + 32);  // [D] this CTA's copy of the residual stream
  sm.xq = reinterpret_cast<uint8_t*>(hs + mp.D);

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
  uint8_t* const comm = mp.comm[mp.tp_rank];
  unsigned* const ctl = reinterpret_cast<unsigned*>(comm + mp.lay.ctl);  // [0] exit counter [1] epoch [2] error [3] final barrier

  if (warp == kConsumerWarps) {
    // ================= producer: every phase's HBM stream, back to back; waits for nothing but free ring slots =================
    if (lane == 0) {
      G1State st;
      bool dep = false;
      for (int l = 0; l < L; ++l) {
        {
          const GemvParams p = make_phase(mp, l, PH_QKV);
          g1_producer_phase(p, sm, cta, n_cta, st);
        }
        if (!dep) {
          pdl_wait();  // pos[] of this step is final
          dep = true;
        }
        attn_producer_phase(mp, sm, l, cta, n_cta, st);
        {
          const GemvParams p = make_phase(mp, l, PH_WO);
          g1_producer_phase(p, sm, cta, n_cta, st);
        }
        {
          const GemvParams p = make_phase(mp, l, PH_W13);
          g1_producer_phase(p, sm, cta, n_cta, st);
        }
        {
          const GemvParams p = make_phase(mp, l, PH_W2);
          g1_producer_phase(p, sm, cta, n_cta, st);
        }
      }
      const GemvParams p = make_head(mp);
      g1_producer_phase(p, sm, cta, n_cta, st);
    }
    return;
  }

  if (warp > kConsumerWarps) {
    // ================= epilogue warps =================
    const int etid = tid - (kConsumerWarps + 1) * 32;
    pdl_wait();
    const unsigned epoch = ctl[1];
    const uint32_t seq0 = epoch * (unsigned)n_ph + 1u;
    int lt = 0;
    __shared__ __half2 sz_buf[2][kMaxLocal * 16];
    __shared__ float2 rope_buf[kMaxLocal * 16];
    const EpiStage es = {sz_buf, rope_buf};
    // phase q (GEMV phases only, numbered 0, 1, 2, ... in execution order) reads buffer q & 1; its scales are prefetched
    // while phase q - 1 runs
    {
      const GemvParams p0 = make_phase(mp, 0, PH_QKV);
      epi_prefetch(mp, p0, es, 0, true, etid, cta, n_cta);
    }
    int q = 0;
    auto run = [&](int l, int kind, auto tag) {
      constexpr int KIND = decltype(tag)::value;
      const GemvParams p = make_phase(mp, l, KIND);
      // next GEMV phase in execution order: QKV -> WO -> W13 -> W2 -> QKV(l+1); none after the last W2 (the head is fp16)
      const int nk = KIND == PH_QKV ? PH_WO : KIND == PH_WO ? PH_W13 : KIND == PH_W13 ? PH_W2 : PH_QKV;
      const int nl = KIND == PH_W2 ? l + 1 : l;
      if (nl < L) {
        const GemvParams pn = make_phase(mp, nl, nk);
        epi_prefetch(mp, pn, es, (q + 1) & 1, nk == PH_QKV, etid, cta, n_cta);
      } else {
        cp_async_commit();  // keep the group accounting uniform
      }
      epilogue_ll<KIND>(mp, p, sm, es, q & 1, seq0 + 5 * l + KIND, etid, lane, cta, n_cta, lt);
      asm volatile("bar.sync 2, %0;" ::"n"(kEpiWarps * 32) : "memory");  // both epilogue warps have issued their stores
      if (etid == 0) hint_bump(mp, 5 * l + KIND, n_ph), mtl(mp, 5 * l + KIND, 3);
      ++q;
    };
    for (int l = 0; l < L; ++l) {
      run(l, PH_QKV, std::integral_constant<int, PH_QKV>{});
      run(l, PH_WO, std::integral_constant<int, PH_WO>{});
      run(l, PH_W13, std::integral_constant<int, PH_W13>{});
      run(l, PH_W2, std::integral_constant<int, PH_W2>{});
    }
    {
      const GemvParams p = make_head(mp);
      epilogue_role<16, 1>(p, 1, nullptr, 1, false, etid, lane, reinterpret_cast<const float*>(sm.red), sm.red_full, sm.red_empty,
                           x_ready, nullptr, lt, 0);
    }
    asm volatile("bar.sync 2, %0;" ::"n"(kEpiWarps * 32) : "memory");
    if (etid == 0) {
      mtl(mp, n_ph - 1, 3);
      const unsigned epoch1 = epoch + 1u;
      if (mp.tp_world > 1) {
        // the vocabulary-sharded logits are the one place that needs a barrier: every rank must hold every slice when its
        // kernel completes (ColumnParallelLinear gather_output, llama.py:308,426)
        __threadfence_system();
        for (int r = 0; r < mp.tp_world; ++r)
          asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(reinterpret_cast<unsigned*>(mp.comm[r] + mp.lay.ctl) + 3), "r"(1u) : "memory");
        const unsigned target = epoch1 * (unsigned)(n_cta * mp.tp_world);
        unsigned v, spins = 0;
        do {
          asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(ctl + 3) : "memory");
        } while ((int)(v - target) < 0 && ++spins < kSpinCap);
        if (spins >= kSpinCap) ctl[2] = 2u;
      }
      __threadfence();
      // the CTA that leaves last advances the epoch (sequence numbers of the next launch); nothing is ever reset
      const unsigned old = atomicAdd(ctl + 0, 1u);
      if (old + 1u == epoch1 * (unsigned)n_cta) {
        ctl[1] = epoch1;
        __threadfence();
      }
    }
    return;
  }

  // ================= MMA warps =================
  G1State st;
  pdl_wait();  // token / pos / caches / epoch of the previous step are final
  const unsigned epoch = ctl[1];
  const uint32_t seq0 = epoch * (unsigned)n_ph + 1u;
  unsigned err = 0;
  const __half* emb_row = mp.tok_emb + (size_t)mp.token[0] * mp.D;  // ParallelEmbedding row (llama.py:399)
  const unsigned epoch1 = epoch + 1u;
  auto gate = [&](int producer_ph) {  // wait (one thread) until the producing phase's hint says its outputs are on their way
    if (!(mp.flags & 2)) {
      if (tid == 0) hint_wait(mp, producer_ph, n_ph, epoch1, n_cta);
      named_bar_sync(1, kConsumerThreads);
    }
  };
  for (int l = 0; l < L; ++l) {
    {
      const GemvParams p = make_phase(mp, l, PH_QKV);
      if (l > 0) gate(5 * (l - 1) + PH_W2);
      const float xs_w = stage_norm(mp, p, sm, hs, comm + mp.lay.pf, seq0 + 5 * (l - 1) + PH_W2, l > 0, l == 0 ? emb_row : nullptr,
                                    nullptr, warp, lane, &err);
      if (tid == 0) mtl(mp, 5 * l + PH_QKV, 1);
      g1_mma_tiles(p, sm, warp, lane, cta, n_cta, st, xs_w);
      if (tid == 0) mtl(mp, 5 * l + PH_QKV, 2);
    }
    {
      gate(5 * l + PH_QKV);
      attn_mma_phase(mp, sm, seq0 + 5 * l + PH_QKV, seq0 + 5 * l + PH_ATTN, warp, lane, cta, n_cta, st, &err);
      if (tid == 0) hint_bump(mp, 5 * l + PH_ATTN, n_ph), mtl(mp, 5 * l + PH_ATTN, 2);  // after the named barrier that ends the merge
    }
    {
      const GemvParams p = make_phase(mp, l, PH_WO);
      gate(5 * l + PH_ATTN);
      const float xs_w = stage_attn_merge(mp, p, sm, comm + mp.lay.att, seq0 + 5 * l + PH_ATTN, warp, lane, &err);
      if (tid == 0) mtl(mp, 5 * l + PH_WO, 1);
      g1_mma_tiles(p, sm, warp, lane, cta, n_cta, st, xs_w);
      if (tid == 0) mtl(mp, 5 * l + PH_WO, 2);
    }
    {
      const GemvParams p = make_phase(mp, l, PH_W13);
      gate(5 * l + PH_WO);
      const float xs_w = stage_norm(mp, p, sm, hs, comm + mp.lay.po, seq0 + 5 * l + PH_WO, true, nullptr, nullptr, warp, lane, &err);
      if (tid == 0) mtl(mp, 5 * l + PH_W13, 1);
      g1_mma_tiles(p, sm, warp, lane, cta, n_cta, st, xs_w);
      if (tid == 0) mtl(mp, 5 * l + PH_W13, 2);
    }
    {
      const GemvParams p = make_phase(mp, l, PH_W2);
      gate(5 * l + PH_W13);
      const float xs_w = stage_plain(mp, p, sm, comm + mp.lay.act, seq0 + 5 * l + PH_W13, warp, lane, &err);
      if (tid == 0) mtl(mp, 5 * l + PH_W2, 1);
      g1_mma_tiles(p, sm, warp, lane, cta, n_cta, st, xs_w);
      if (tid == 0) mtl(mp, 5 * l + PH_W2, 2);
    }
  }
  {
    // fp16 lm_head on the HMMA path (gemv_core.cuh); its fp16 x row lives in the digit-plane area
    const GemvParams p = make_head(mp);
    __half* xs = reinterpret_cast<__half*>(sm.xq);
    gate(5 * (L - 1) + PH_W2);
    stage_norm(mp, p, sm, hs, comm + mp.lay.pf, seq0 + 5 * (L - 1) + PH_W2, true, nullptr, xs, warp, lane, &err);
    if (lane == 0) mbar_arrive(x_ready);
    if (tid == 0) mtl(mp, n_ph - 1, 1);
    long long c0 = 0, c1 = 0;
    mma_phase<16, 1, 0>(p, 1, 1, false, sm.ring, sm.full, sm.empty, reinterpret_cast<float*>(sm.red), sm.red_full, sm.red_empty,
                        xs, nullptr, st.stage, st.par, st.lt, warp, lane, c0, c1, false);
    if (tid == 0) mtl(mp, n_ph - 1, 2);
  }
  if (err) ctl[2] = 1u;
}

static CommLayout make_layout(int L, int D, int Hq, int Hkv, int F, int V, int n_split, int tp) {
  auto al = [](size_t v) { return (int)((v + 255) / 256 * 256); };
  CommLayout c;
  size_t off = 0;
  c.ctl = (int)off, off = al(off + 64 + (size_t)(5 * L + 1) * 4);
  c.yq = (int)off, off = al(off + (size_t)Hq * 128 * 4);
  c.ykv = (int)off, off = al(off + (size_t)Hkv * 2 * 128 * 4);
  c.att = (int)off, off = al(off + (size_t)Hq * n_split * 130 * 8);
  c.po = (int)off, off = al(off + (size_t)tp * D * 4);
  c.act = (int)off, off = al(off + (size_t)F * 4);
  c.pf = (int)off, off = al(off + (size_t)tp * D * 4);
  c.logits = (int)off, off = al(off + (size_t)V * tp * 4);
  c.total = (int)off;
  return c;
}

}  // namespace ll
}  // namespace b200

using namespace b200;

static int ll_split(int Hkv) {
  static const int force = getenv("B200_STEP1_SPLIT") ? atoi(getenv("B200_STEP1_SPLIT")) : 0;
  if (force > 0) return std::min(force, ll::kMaxSplit);
  return std::max(1, std::min(ll::kMaxSplit, sm_count() / std::max(Hkv, 1)));
}

extern "C" size_t b200_step1_ll_comm_bytes(int n_layers, int dim, int n_heads, int n_kv_heads, int ffn, int vocab_local,
                                           int tp_world) {
  return (size_t)ll::make_layout(n_layers, dim, n_heads, n_kv_heads, ffn, vocab_local, ll_split(n_kv_heads), tp_world).total;
}
extern "C" size_t b200_step1_ll_logits_offset(int n_layers, int dim, int n_heads, int n_kv_heads, int ffn, int vocab_local,
                                              int tp_world) {
  return (size_t)ll::make_layout(n_layers, dim, n_heads, n_kv_heads, ffn, vocab_local, ll_split(n_kv_heads), tp_world).logits;
}

extern "C" int b200_decode_step1_ll(const b200_step1_args_t* a, b200_stream_t stream) {
  if (!a || a->n_layers < 1 || a->n_layers > ll::kMaxLayers) {
    set_error("step1_ll: n_layers must be in 1..96");
    return B200_E_INVAL;
  }
  if (a->dim <= 0 || (a->dim & 127) || a->ffn <= 0 || (a->ffn & 127) || a->dim > 8192 || a->ffn > 16384 || a->n_heads < 1 ||
      a->n_kv_heads < 1 || a->n_heads % a->n_kv_heads || a->n_heads / a->n_kv_heads > 8 || a->n_heads * 128 > 16384 ||
      (a->vocab & 15) || (a->cache_seq % ll::kTileKV) || a->cache_seq < ll::kTileKV) {
    set_error("step1_ll: unsupported shape (dim/ffn multiples of 128, head_dim 128, n_rep <= 8, vocab % 16 == 0, cache_seq % 32 == 0)");
    return B200_E_UNSUPPORTED;
  }
  if (!a->token || !a->tok_emb || !a->pos || !a->rope || !a->kcache || !a->vtcache || !a->comm || !a->wqkv || !a->wo || !a->w13 ||
      !a->w2 || !a->attn_norm || !a->ffn_norm || !a->final_norm || a->tp_world < 1 || a->tp_world > 8 || a->tp_rank < 0 ||
      a->tp_rank >= a->tp_world) {
    set_error("step1_ll: null pointer or bad tensor-parallel rank");
    return B200_E_INVAL;
  }
  static ll::Params mp;
  memset(&mp, 0, sizeof(mp));
  mp.n_layers = a->n_layers, mp.D = a->dim, mp.Hq = a->n_heads, mp.Hkv = a->n_kv_heads, mp.F = a->ffn, mp.V = a->vocab;
  mp.cache_seq = a->cache_seq;
  mp.tp_world = a->tp_world, mp.tp_rank = a->tp_rank;
  static const int flags = getenv("B200_STEP1_FLAGS") ? atoi(getenv("B200_STEP1_FLAGS")) : 0;
  mp.flags = flags;
  mp.eps = a->eps;
  mp.scale_log2 = (1.0f / sqrtf(128.0f)) * 1.4426950408889634f;
  mp.token = reinterpret_cast<const long long*>(a->token);
  mp.tok_emb = static_cast<const __half*>(a->tok_emb);
  mp.pos = a->pos;
  mp.rope = reinterpret_cast<const float2*>(a->rope);
  mp.kcache = static_cast<__half*>(a->kcache), mp.vtcache = static_cast<__half*>(a->vtcache);
  mp.kv_layer_stride = a->kv_layer_stride;
  mp.final_norm = static_cast<const __half*>(a->final_norm);
  mp.tl = static_cast<unsigned long long*>(a->timeline);
  for (int r = 0; r < a->tp_world; ++r) {
    if (!a->comm[r]) {
      set_error("step1_ll: null communication block");
      return B200_E_INVAL;
    }
    mp.comm[r] = static_cast<uint8_t*>(a->comm[r]);
  }
  const int Nqkv = (a->n_heads + 2 * a->n_kv_heads) * 128;
  auto chk = [&](const b200_linear_t& l, int N, int K, int bits, const char* what) {
    if (l.bits != bits || l.N != N || l.K != K || !l.qweight || (bits != 16 && (!l.scales || (l.group_size > 0 && l.group_size < K)))) {
      set_error(std::string("step1_ll: ") + what + " must be a per-channel W4 (lm_head: fp16) linear of the model's shape");
      return false;
    }
    return true;
  };
  for (int i = 0; i < a->n_layers; ++i) {
    if (!chk(a->wqkv[i], Nqkv, a->dim, 4, "wqkv") || !chk(a->wo[i], a->dim, a->n_heads * 128, 4, "wo") ||
        !chk(a->w13[i], 2 * a->ffn, a->dim, 4, "w13") || !chk(a->w2[i], a->dim, a->ffn, 4, "w2"))
      return B200_E_UNSUPPORTED;
    ll::Layer& Lr = mp.layer[i];
    Lr.wqkv = static_cast<const uint8_t*>(a->wqkv[i].qweight), Lr.sqkv = static_cast<const __half2*>(a->wqkv[i].scales);
    Lr.wo = static_cast<const uint8_t*>(a->wo[i].qweight), Lr.so = static_cast<const __half2*>(a->wo[i].scales);
    Lr.w13 = static_cast<const uint8_t*>(a->w13[i].qweight), Lr.s13 = static_cast<const __half2*>(a->w13[i].scales);
    Lr.w2 = static_cast<const uint8_t*>(a->w2[i].qweight), Lr.s2 = static_cast<const __half2*>(a->w2[i].scales);
    Lr.attn_norm = static_cast<const __half*>(a->attn_norm[i]), Lr.ffn_norm = static_cast<const __half*>(a->ffn_norm[i]);
  }
  if (!chk(a->lm_head, a->vocab, a->dim, 16, "lm_head")) return B200_E_UNSUPPORTED;
  mp.lm_head = static_cast<const uint8_t*>(a->lm_head.qweight);
  mp.n_split = ll_split(a->n_kv_heads);
  mp.lay = ll::make_layout(a->n_layers, a->dim, a->n_heads, a->n_kv_heads, a->ffn, a->vocab, mp.n_split, a->tp_world);

  // shared memory: ring | barriers | red (16 KB) | scratch | h [D] | digit planes of the widest K (also: fp16 x of the head,
  // attention merge which starts in `red`)
  const int Kmax = std::max(std::max(a->dim, a->ffn), a->n_heads * 128);
  size_t xq = (size_t)kPlanes * ((((size_t)Kmax + 127) / 128) * 128 + 64);
  xq = std::max(xq, (size_t)(a->dim + kXPad) * 2);
  xq = std::max(xq, (size_t)kConsumerWarps * 4 * 130 * 4);
  const size_t fixed = 6 * 8 + (size_t)2 * kConsumerWarps * 128 * 4 + 32 * 4 + (size_t)a->dim * 2 + xq;
  const size_t cap = std::min<size_t>(smem_optin(), 227 * 1024) - 6144;  // static: sz_s / rope_s of the epilogue instances
  static const int ring_kb = getenv("B200_STEP1_RING_KB") ? atoi(getenv("B200_STEP1_RING_KB")) : 192;
  int stages = std::max(2, std::min(ring_kb * 1024 / kSlotBytes, 12));
  while (stages > 2 && (size_t)stages * (kSlotBytes + 16) + fixed > cap) --stages;
  if ((size_t)stages * (kSlotBytes + 16) + fixed > cap) {
    set_error("step1_ll: shared memory budget exceeded");
    return B200_E_UNSUPPORTED;
  }
  mp.stages = stages;
  const size_t smem = (size_t)stages * (kSlotBytes + 16) + fixed;
  static size_t configured[16] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  dev &= 15;
  if (smem > configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(ll::decode_step1_ll_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      set_error(std::string("step1_ll: cudaFuncSetAttribute: ") + cudaGetErrorString(e));
      return (int)e;
    }
    configured[dev] = smem;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(sm_count());  // one CTA per SM: every CTA must be resident (consumers poll what other CTAs produce)
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
  cudaError_t e = cudaLaunchKernelEx(&cfg, ll::decode_step1_ll_kernel, mp);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    set_error(std::string("step1_ll: launch: ") + cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}
