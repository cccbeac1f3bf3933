// GQA decode attention with split-KV (flash-decoding) for sm_90a.
//
// Replaces repeat_kv + F.scaled_dot_product_attention / flash_attn_func for seqlen-1 queries
// (accessory/model/LLM/llama.py:170-206).  The KV cache is stored as shared-memory images (see below), written
// in place by the fused QKV GEMV epilogue, so a 32-position tile of K or V is one contiguous 8 KB TMA bulk copy.
//
// One CTA = one (split, kv-head, token).  A producer warp bulk-copies K and V tiles (cp.async.bulk + mbarriers) into
// one small ring per consumer warp; the 4 consumer warps take tiles round-robin, each from its own ring, and only
// meet (at a named barrier, without the producer) for the in-CTA merge.  All n_rep query heads of the group ride in the M dimension of the
// HMMAs, so K/V are read once per group (never materialising repeat_kv):
//     S[h][s]  = Q[h][:] . K[s][:]        A = Q (16 x 16 per step), B = K rows   (k-slot permutation in d)
//     O[h][d] += P[h][s] * Vt[d][s]       A = P straight from the S accumulators (FA2 register reuse)
// Softmax is online in fp32 with exp2; P is rounded to fp16 for the second GEMM (as flash-attn does).
// Partials (m, l, O) go to a workspace; the last CTA of a (token, kv-head) merges them in fixed order.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>
#include <cstdlib>
#include <string>

#include "../../include/b200_decode.h"
#include "common.cuh"

namespace b200 {
void set_error(const std::string& s);
int sm_count();
unsigned long long* timeline_slot();
unsigned long long* timeline_cta_slot();
int prefetch_window_bytes();
int tune_get(const char* name, int dflt);

constexpr int kAttnWarps = 4;                 // consumer warps; one more warp produces
constexpr int kAttnThreads = (kAttnWarps + 1) * 32;
constexpr int kConsumerThreads = kAttnWarps * 32;
constexpr int kTile = 32;                     // kv positions per tile
constexpr int kHalfBytes = kTile * 256;       // one K tile or one V tile: 8 KB, one bulk copy, one ring slot
// Per-warp rings.  Warp w computes tiles w, w + 4, w + 8, ... and its ring receives exactly their halves, in the order the
// warp uses them: K(w), V(w), K(w + 4), V(w + 4), ...  Each slot has its own full / empty mbarrier and one consumer, so a
// slot is free again as soon as its warp has read it: a K slot after the scores, a V slot after P.V.
// Tiles are dealt from warp 0, so warp 0 never has fewer than any other warp and gets the deepest ring:
//   5 + 3 + 3 + 3 = 14 slots x 8 KB = 112 KB per CTA; two CTAs per SM: 2 x (112 KB + ~0.3 KB static + 1 KB reserved)
//   <= 228 KB.  At the bench shape (LLaMA2-7B, kv length 2049 - 2304: 8 splits of 9 tiles; warp 0 has 3 tiles, warps 1-3
//   have 2) that is every K tile plus V of tiles 0 - 4 (104 of 144 KB) in flight before the QKV launch resolves; the last
//   V of each warp is requested as soon as that warp has scored its first tile.
constexpr int kSlots0 = 5, kSlotsW = 3;
constexpr int kSlots = kSlots0 + (kAttnWarps - 1) * kSlotsW;
constexpr int kSmemBytes = kSlots * kHalfBytes;
// the merge of more than 16 splits stages (m, l) pairs, rescale factors and L of a group in the first 96 KB of the slots
constexpr int kMergeStageBytes = 96 * 1024;
constexpr int kChunkAlign = kAttnWarps * kTile;
static_assert(kSmemBytes <= 112 * 1024 && kMergeStageBytes <= kSmemBytes, "two CTAs per SM");

__device__ __forceinline__ int ring_base(int warp) { return warp == 0 ? 0 : kSlots0 + (warp - 1) * kSlotsW; }
__device__ __forceinline__ int ring_depth(int warp) { return warp == 0 ? kSlots0 : kSlotsW; }

struct AttnParams {
  const __half* q;
  const __half* kc;
  const __half* vt;
  const int* pos;
  __half* out;
  float* ws_o;   // [T][Hq][n_split][128]
  float2* ws_ml; // [T][Hq][n_split]
  int* counters; // [T][Hkv]
  int T, Hq, Hkv, S, tps, n_split, chunk, n_rep;
  float scale_log2;
  const uint8_t* next_w;  // the next kernel's weight stream (L2 prefetch of its per-CTA region heads)
  int next_bytes, next_tiles, next_grid, next_window;
  unsigned long long* tl;
  unsigned long long* tlc;  // per-CTA stamps (b200_timeline_cta)
  int stream_ef; // K/V bulk copies carry the L2 evict_first policy (B200_KV_EF)
  int even;      // keys dealt out to the splits in whole tiles, evenly (B200_ATTN_EVEN)
  int pf_early;  // next-stream L2 prefetch as soon as the producer would block instead of after its last copy
};

// KV-cache layouts are "shared-memory images" so that one 32-position tile is ONE contiguous 8 KB bulk copy:
//   K  [B][Hkv][S][128]          with the 16-byte chunk index XOR-swizzled by the row parity: chunk ^ ((s&1)<<2)
//   V  [B][Hkv][S/32][128][32]   (transposed inside each 32-position block)
__device__ __forceinline__ int k_swz(int row) { return (row & 1) << 2; }

__device__ __forceinline__ int atomic_add_acq_rel(int* addr, int v) {
  int old;
  asm volatile("atom.acq_rel.gpu.global.add.s32 %0, [%1], %2;" : "=r"(old) : "l"(addr), "r"(v) : "memory");
  return old;
}

__global__ void __launch_bounds__(kAttnThreads, 2) attn_decode_kernel(const __grid_constant__ AttnParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ int s_last;
  __shared__ __align__(8) uint64_t bars[2 * kSlots];
  uint64_t* full = bars;
  uint64_t* empty = bars + kSlots;
  // grid (Hkv, n_split, T): CTAs are dispatched kv head fastest, so the last and lightest split (the remainder of the keys)
  // goes to the SMs the QKV launch frees last
  const int kvh = blockIdx.x, split = blockIdx.y, tok = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kSlots; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 1);
    }
    fence_mbar_init();
  }
  __syncthreads();  // the only CTA-wide barrier
  const int cta_lin = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  if (threadIdx.x == 0) tl_min(p.tl, 0), tl_cta(p.tlc, cta_lin, 0);
  pdl_launch_dependents();
  // pos[] is written by a kernel that is not part of the programmatic-launch chain (advance_pos / host copies are
  // full stream dependencies), so it may be read before the dependency on the QKV kernel resolves.  Everything the
  // predecessor writes -- q and cache row pos[tok] -- is only touched after pdl_wait() below.
  const int kv_len = p.pos[tok] + 1;
  const int brow = tok / p.tps;
  // equal work per split for the ACTUAL kv length (the grid is sized once, for max_kv_len, when a graph is captured)
  int s_begin, s_end, n_tiles;
  if (p.even) {
    // the 32-position tiles that hold keys are dealt out evenly (split i gets floor or ceil of n_t / n_split): with equal
    // rounded-up chunks 2048 keys over 9 splits became 8 x 8 tiles + an idle split, i.e. 256 busy CTAs on 132 SMs (about 2 : 1)
    const int n_t = (kv_len + kTile - 1) / kTile;
    const int t_begin = (int)(((long long)n_t * split) / p.n_split), t_end = (int)(((long long)n_t * (split + 1)) / p.n_split);
    s_begin = t_begin * kTile;
    s_end = min(kv_len, t_end * kTile);
    n_tiles = t_end - t_begin;
  } else {
    const int chunk = min(p.chunk, ((kv_len + p.n_split - 1) / p.n_split + kTile - 1) / kTile * kTile);
    s_begin = split * chunk;
    s_end = min(kv_len, s_begin + chunk);
    n_tiles = s_end > s_begin ? (s_end - s_begin + kTile - 1) / kTile : 0;
  }
  const size_t kv_base = ((size_t)brow * p.Hkv + kvh) * p.S * 128;  // same element offset for K and V planes

  if (warp == kAttnWarps) {
    // ---------------- producer: each warp's halves into that warp's ring ----------------
    // Lane 0 polls the four rings and issues whatever half is next for a warp whose slot is free, so a full ring never holds
    // back the halves of the other warps.  Only the tile holding a row the QKV kernel is appending waits for the dependency:
    // its halves are skipped until nothing else can be issued, then the producer waits once.  The producer takes no part in
    // the tail and returns when every copy is issued.
    if (lane == 0) {
      const bool stream_ef = p.stream_ef != 0;
      const uint64_t pol = stream_ef ? l2_policy_evict_first() : 0;
      bool waited = false, pf_done = !(p.next_w && p.next_bytes > 0);
      auto prefetch_next = [&]() {  // pull the next kernel's weights into L2
        pf_done = true;
        const int n_cta = gridDim.x * gridDim.y * gridDim.z;
        prefetch_next_stream(p.next_w, p.next_bytes, p.next_tiles, p.next_grid, p.next_window, cta_lin, n_cta);
      };
      // the QKV kernel appends the rows of every token of this sequence in the launch, not just row pos[tok]: a prompt chunk
      // whose positions cross a 32-row tile writes into the tile before the one holding pos[tok] as well
      int first_new = kv_len - 1;
      for (int j = brow * p.tps; j < min(p.T, (brow + 1) * p.tps); ++j) first_new = min(first_new, p.pos[j]);
      int next[kAttnWarps], slot[kAttnWarps], n_half[kAttnWarps];  // per ring: next half, its slot, halves in all
      uint32_t par[kAttnWarps];
      int left = 0;
#pragma unroll
      for (int w = 0; w < kAttnWarps; ++w) {
        next[w] = 0, slot[w] = ring_base(w), par[w] = 0;
        n_half[w] = n_tiles > w ? 2 * ((n_tiles - w + kAttnWarps - 1) / kAttnWarps) : 0;
        left += n_half[w];
      }
      while (left > 0) {
        bool issued = false, held = false;
#pragma unroll
        for (int w = 0; w < kAttnWarps; ++w) {
          if (next[w] == n_half[w]) continue;
          const int s0 = s_begin + (w + kAttnWarps * (next[w] >> 1)) * kTile;
          if (!waited && s0 + kTile > first_new) {  // this tile holds a row the QKV kernel is appending right now
            held = true;
            continue;
          }
          if (!mbar_try_wait(&empty[slot[w]], par[w] ^ 1)) continue;
          uint8_t* dst = smem + (size_t)slot[w] * kHalfBytes;
          const __half* src = ((next[w] & 1) ? p.vt : p.kc) + kv_base + (size_t)s0 * 128;
          mbar_arrive_expect_tx(&full[slot[w]], kHalfBytes);
          if (stream_ef)
            bulk_g2s_hint(dst, src, kHalfBytes, &full[slot[w]], pol);
          else
            bulk_g2s(dst, src, kHalfBytes, &full[slot[w]]);
          ++next[w], --left, issued = true;
          if (++slot[w] == ring_base(w) + ring_depth(w)) slot[w] = ring_base(w), par[w] ^= 1;
        }
        if (!issued) {
          // pf_early: the hint goes out as soon as this producer would block (rings full / dependency), not after its last copy
          if (p.pf_early && !pf_done) prefetch_next();
          if (held) {
            pdl_wait();
            waited = true;
          }
        }
      }
      if (!pf_done) prefetch_next();  // own stream issued
    }
    return;
  }

  // ---------------- consumers ----------------
  float oacc[16][4];
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) oacc[j][i] = 0.f;

  pdl_wait();  // q comes from the previous kernel
  if (threadIdx.x == 0) {
    tl_max(p.tl, 1), tl_cta(p.tlc, cta_lin, 1);
    if (p.tlc) p.tlc[(size_t)cta_lin * 16 + 5] = (unsigned long long)n_tiles;
  }
  // ---- Q fragments: rows g and g+8 of the group's heads, 4 chunks of 32 d ----
  uint32_t qf[4][2][4];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = g + 8 * hh;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (row < p.n_rep)
        v = *reinterpret_cast<const uint4*>(p.q + ((size_t)tok * p.Hq + kvh * p.n_rep + row) * 128 + c * 32 + t4 * 8);
      qf[c][hh][0] = v.x, qf[c][hh][1] = v.y, qf[c][hh][2] = v.z, qf[c][hh][3] = v.w;
    }

  // This warp's tiles (i % 4 == warp) from its own ring: the K half, then the V half of each.  Every slot of the ring is only
  // ever waited on by this warp, in the order it was filled, so a wait never meets a barrier one phase behind.
  int slot = ring_base(warp);
  uint32_t par = 0;
  auto release = [&]() {  // hand the slot back to the producer and step to the next one
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[slot]);
    if (++slot == ring_base(warp) + ring_depth(warp)) slot = ring_base(warp), par ^= 1;
  };
  for (int i = warp; i < n_tiles; i += kAttnWarps) {
    const int s0 = s_begin + i * kTile;
    // K in `slot`, V in the next one (the tile's halves are consecutive in the ring)
    const bool wrap = slot + 1 == ring_base(warp) + ring_depth(warp);
    const int vslot = wrap ? ring_base(warp) : slot + 1;
    mbar_wait(&full[slot], par);
    mbar_wait(&full[vslot], wrap ? par ^ 1 : par);
    const uint8_t* ks = smem + (size_t)slot * kHalfBytes;
    const uint8_t* vs = smem + (size_t)vslot * kHalfBytes;

    // ---- S = Q K^T for 4 blocks of 8 positions; block X column n <-> s0 + 8*(n>>1) + 2X + (n&1) ----
    float sacc[4][4];
#pragma unroll
    for (int X = 0; X < 4; ++X) {
#pragma unroll
      for (int ii = 0; ii < 4; ++ii) sacc[X][ii] = 0.f;
      const int row = 8 * (g >> 1) + (g & 1) + 2 * X;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const uint4 kb = lds_v4(ks + row * 256 + (((4 * c + t4) ^ k_swz(row)) << 4));
        mma16816(sacc[X], qf[c][0][0], qf[c][1][0], qf[c][0][1], qf[c][1][1], kb.x, kb.y);
        mma16816(sacc[X], qf[c][0][2], qf[c][1][2], qf[c][0][3], qf[c][1][3], kb.z, kb.w);
      }
    }
    release();  // K read: its slot takes this warp's next half while the softmax and P.V run
    // ---- mask + online softmax (rows g and g+8) ----
    float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int X = 0; X < 4; ++X)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int s = s0 + 8 * t4 + 2 * X + e;
        const bool ok = s < s_end;
        sacc[X][e] = ok ? sacc[X][e] * p.scale_log2 : -INFINITY;
        sacc[X][2 + e] = ok ? sacc[X][2 + e] * p.scale_log2 : -INFINITY;
        tmax[0] = fmaxf(tmax[0], sacc[X][e]);
        tmax[1] = fmaxf(tmax[1], sacc[X][2 + e]);
      }
    float corr[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      tmax[hh] = fmaxf(tmax[hh], __shfl_xor_sync(0xffffffffu, tmax[hh], 1));
      tmax[hh] = fmaxf(tmax[hh], __shfl_xor_sync(0xffffffffu, tmax[hh], 2));
      const float m_new = fmaxf(m_run[hh], tmax[hh]);  // finite: every tile has >= 1 valid position
      corr[hh] = exp2f(m_run[hh] - m_new);
      m_run[hh] = m_new;
      l_run[hh] *= corr[hh];
    }
    uint32_t pa[2][4];  // A fragments of P for the two PV steps
#pragma unroll
    for (int X = 0; X < 4; ++X) {
      const float p0 = exp2f(sacc[X][0] - m_run[0]), p1 = exp2f(sacc[X][1] - m_run[0]);
      const float p2 = exp2f(sacc[X][2] - m_run[1]), p3 = exp2f(sacc[X][3] - m_run[1]);
      const __half2 h01 = __floats2half2_rn(p0, p1), h23 = __floats2half2_rn(p2, p3);
      // accumulate the row sums from the fp16-rounded P (what the second GEMM multiplies)
      const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
      l_run[0] += f01.x + f01.y;
      l_run[1] += f23.x + f23.y;
      pa[X >> 1][(X & 1) * 2 + 0] = *reinterpret_cast<const uint32_t*>(&h01);
      pa[X >> 1][(X & 1) * 2 + 1] = *reinterpret_cast<const uint32_t*>(&h23);
    }
    // ---- O = O*corr + P V ----
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      oacc[j][0] *= corr[0], oacc[j][1] *= corr[0], oacc[j][2] *= corr[1], oacc[j][3] *= corr[1];
      const uint4 vb = lds_v4(vs + (8 * j + g) * 64 + (t4 << 4));
      mma16816(oacc[j], pa[0][0], pa[0][1], pa[0][2], pa[0][3], vb.x, vb.y);
      mma16816(oacc[j], pa[1][0], pa[1][1], pa[1][2], pa[1][3], vb.z, vb.w);
    }
    release();
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l_run[hh] += __shfl_xor_sync(0xffffffffu, l_run[hh], 1);
    l_run[hh] += __shfl_xor_sync(0xffffffffu, l_run[hh], 2);
  }

  // ---- in-CTA merge: each warp parks (O, m, l) of the group's rows in its own ring (every copy into it has been consumed),
  // the four consumer warps meet at one named barrier (the producer is not waited for) and fold the warps in order ----
  auto part_o = [&](int w) { return reinterpret_cast<float*>(smem + (size_t)ring_base(w) * kHalfBytes); };  // [16][128]
  auto part_ml = [&](int w) { return part_o(w) + 16 * 128; };                                                // [16][2]
  {
    float* mo = part_o(warp);
    float* mml = part_ml(warp);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = g + 8 * hh;
      if (row >= p.n_rep) continue;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        *reinterpret_cast<float2*>(mo + (size_t)row * 128 + 8 * j + 2 * t4) = make_float2(oacc[j][2 * hh], oacc[j][2 * hh + 1]);
      if (t4 == 0) mml[row * 2 + 0] = m_run[hh], mml[row * 2 + 1] = l_run[hh];
    }
  }
  named_bar_sync(1, kConsumerThreads);

  const int d = threadIdx.x;  // consumer thread <-> output dim
  for (int h = 0; h < p.n_rep; ++h) {
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < kAttnWarps; ++w) M = fmaxf(M, part_ml(w)[h * 2]);
    float L = 0.f, o = 0.f;
#pragma unroll
    for (int w = 0; w < kAttnWarps; ++w) {
      const float mw = part_ml(w)[h * 2];
      const float f = (mw == -INFINITY) ? 0.f : exp2f(mw - M);
      L += part_ml(w)[h * 2 + 1] * f;
      o += part_o(w)[(size_t)h * 128 + d] * f;
    }
    const int hq = kvh * p.n_rep + h;
    if (p.n_split == 1) {
      p.out[((size_t)tok * p.Hq + hq) * 128 + d] = __float2half_rn(o / L);
    } else {
      p.ws_o[(((size_t)tok * p.Hq + hq) * p.n_split + split) * 128 + d] = o;
      if (d == 0) p.ws_ml[((size_t)tok * p.Hq + hq) * p.n_split + split] = make_float2(M, L);
    }
  }
  if (threadIdx.x == 0) tl_max(p.tl, 2), tl_cta(p.tlc, cta_lin, 2);
  if (p.n_split == 1) {
    if (threadIdx.x == 0) tl_max(p.tl, 3);
    return;
  }
  // ---- cross-split merge by the last CTA to arrive for this (token, kv head) ----
  // One acquire-release add by one thread instead of a sequentially consistent fence in every thread before the count and
  // again after it: the barrier orders the other consumer threads' partial stores before thread 0's release (release is
  // cumulative), and the second barrier orders the merging CTA's loads after thread 0's acquire.
  named_bar_sync(1, kConsumerThreads);  // also: every warp is done reading the parked partials
  if (threadIdx.x == 0) s_last = atomic_add_acq_rel(&p.counters[tok * p.Hkv + kvh], 1) == p.n_split - 1;
  named_bar_sync(1, kConsumerThreads);
  if (!s_last) {
    if (threadIdx.x == 0) tl_max(p.tl, 3), tl_cta(p.tlc, cta_lin, 3);
    return;
  }
  // Latency-parallel merge: (1) all (M, L) pairs of the group in one round trip -> smem, (2) one warp per head forms
  // the global max, the rescale factors and L, (3) one warp per head accumulates O with 16 independent 16-byte loads
  // in flight per lane.  (A serial loop over the splits costs one L2 round trip per split: 60 us at 33 splits x 8 heads.)
  if (p.n_split <= 16) {
    // one warp per head, ONE L2 round trip: the (m, l) pairs (lane = split) and all O partials are requested together;
    // same operations in the same order as the general path below (bit-identical results)
    const float2* ml0 = p.ws_ml + ((size_t)tok * p.Hq + (size_t)kvh * p.n_rep) * p.n_split;
    for (int h = warp; h < p.n_rep; h += kAttnWarps) {
      const int hq = kvh * p.n_rep + h;
      const float4* base = reinterpret_cast<const float4*>(p.ws_o + ((size_t)tok * p.Hq + hq) * p.n_split * 128) + lane;
      const float2 mlv = lane < p.n_split ? __ldcg(&ml0[h * p.n_split + lane]) : make_float2(-INFINITY, 0.f);
      float4 v[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) v[j] = j < p.n_split ? __ldcg(base + (size_t)j * 32) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float M = warp_max(mlv.x);
      const float f = (mlv.x == -INFINITY) ? 0.f : exp2f(mlv.x - M);
      const float L = warp_sum(mlv.y * f);
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float fj = __shfl_sync(0xffffffffu, f, j);
        acc.x = fmaf(v[j].x, fj, acc.x), acc.y = fmaf(v[j].y, fj, acc.y);
        acc.z = fmaf(v[j].z, fj, acc.z), acc.w = fmaf(v[j].w, fj, acc.w);
      }
      __half2* dst = reinterpret_cast<__half2*>(p.out + ((size_t)tok * p.Hq + hq) * 128 + lane * 4);
      dst[0] = __floats2half2_rn(acc.x / L, acc.y / L);
      dst[1] = __floats2half2_rn(acc.z / L, acc.w / L);
    }
  } else {
    float2* sml = reinterpret_cast<float2*>(smem);                    // [n_rep][n_split]
    float* sf = reinterpret_cast<float*>(sml + p.n_rep * p.n_split);   // [n_rep][n_split]
    float* sL = sf + p.n_rep * p.n_split;                              // [n_rep]
    const int nml = p.n_rep * p.n_split;
    const float2* ml0 = p.ws_ml + ((size_t)tok * p.Hq + (size_t)kvh * p.n_rep) * p.n_split;  // heads of a group are adjacent
    for (int i = threadIdx.x; i < nml; i += kConsumerThreads) sml[i] = __ldcg(&ml0[i]);
    named_bar_sync(1, kConsumerThreads);
    for (int h = warp; h < p.n_rep; h += kAttnWarps) {
      float M = -INFINITY;
      for (int sp = lane; sp < p.n_split; sp += 32) M = fmaxf(M, sml[h * p.n_split + sp].x);
      M = warp_max(M);
      float L = 0.f;
      for (int sp = lane; sp < p.n_split; sp += 32) {
        const float2 v = sml[h * p.n_split + sp];
        const float f = (v.x == -INFINITY) ? 0.f : exp2f(v.x - M);
        sf[h * p.n_split + sp] = f;
        L += v.y * f;
      }
      L = warp_sum(L);
      if (lane == 0) sL[h] = L;
    }
    named_bar_sync(1, kConsumerThreads);
    for (int h = warp; h < p.n_rep; h += kAttnWarps) {
      const int hq = kvh * p.n_rep + h;
      const float4* base = reinterpret_cast<const float4*>(p.ws_o + ((size_t)tok * p.Hq + hq) * p.n_split * 128) + lane;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int s0 = 0; s0 < p.n_split; s0 += 16) {
        float4 v[16];
#pragma unroll
        for (int j = 0; j < 16; ++j)
          v[j] = (s0 + j < p.n_split) ? __ldcg(base + (size_t)(s0 + j) * 32) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float f = (s0 + j < p.n_split) ? sf[h * p.n_split + s0 + j] : 0.f;
          acc.x = fmaf(v[j].x, f, acc.x), acc.y = fmaf(v[j].y, f, acc.y);
          acc.z = fmaf(v[j].z, f, acc.z), acc.w = fmaf(v[j].w, f, acc.w);
        }
      }
      const float L = sL[h];
      __half2* dst = reinterpret_cast<__half2*>(p.out + ((size_t)tok * p.Hq + hq) * 128 + lane * 4);
      dst[0] = __floats2half2_rn(acc.x / L, acc.y / L);
      dst[1] = __floats2half2_rn(acc.z / L, acc.w / L);
    }
  }
  if (threadIdx.x == 0) p.counters[tok * p.Hkv + kvh] = 0;  // ready for the next launch / graph replay
  if (threadIdx.x == 0) tl_max(p.tl, 3), tl_cta(p.tlc, cta_lin, 3), tl_cta(p.tlc, cta_lin, 6);
}

}  // namespace b200

using namespace b200;

extern "C" int b200_attn_choose_split(int T, int Hkv, int max_kv_len) {
  if (T <= 0 || Hkv <= 0 || max_kv_len <= 0) return 1;
  // all CTAs must be co-resident in one wave: 2 CTAs per SM (112 KB of rings each)
  const int target = 2 * sm_count();
  int want = target / (T * Hkv);
  const int max_split = (max_kv_len + kChunkAlign - 1) / kChunkAlign;
  // Every split count merges through the workspace (last CTA of a (token, kv head)), never through a thread-block cluster:
  // a cluster is only scheduled once all its CTA slots in one GPC are free at the same time, which defeats the early start
  // under programmatic dependent launch (dropping the clusters of 8 CTAs gave 8 % more decode tokens/s at bs = 1 on an H100 SXM).
  const int cap = tune_get("B200_ATTN_MAX_SPLIT", 16);
  want = std::max(1, std::min(want, max_split));
  if (want > cap && T * Hkv * cap >= sm_count()) want = std::max(cap, 1);  // keep >= one CTA per SM when capping
  int chunk = (max_kv_len + want - 1) / want;
  chunk = (chunk + kTile - 1) / kTile * kTile;
  return (max_kv_len + chunk - 1) / chunk;
}

extern "C" size_t b200_attn_workspace_bytes(int T, int Hq, int n_split) {
  if (n_split <= 1) return 16;
  return (size_t)T * Hq * n_split * (128 * 4 + 8);
}

extern "C" int b200_attn_decode(const b200_attn_args_t* a, b200_stream_t stream) {
  if (!a || !a->q || !a->kcache || !a->vtcache || !a->pos || !a->out) {
    set_error("attn: null pointer");
    return B200_E_INVAL;
  }
  if (a->T < 1 || a->Hq < 1 || a->Hkv < 1 || a->Hq % a->Hkv || a->Hq / a->Hkv > 16) {
    set_error("attn: need Hq % Hkv == 0 and at most 16 query heads per kv head");
    return B200_E_UNSUPPORTED;
  }
  if (a->cache_seq < kTile || (a->cache_seq % kTile) || a->max_kv_len < 1 || a->max_kv_len > a->cache_seq ||
      a->tokens_per_seq < 1) {
    set_error("attn: cache_seq must be a multiple of 32 and max_kv_len within it");
    return B200_E_INVAL;
  }
  int n_split = a->n_split > 0 ? a->n_split : b200_attn_choose_split(a->T, a->Hkv, a->max_kv_len);
  int chunk = (a->max_kv_len + n_split - 1) / n_split;
  chunk = (chunk + kTile - 1) / kTile * kTile;
  n_split = (a->max_kv_len + chunk - 1) / chunk;
  // the merge of more than 16 splits stages (m, l) pairs, rescale factors and L of a group in the slots
  if ((size_t)(a->Hq / a->Hkv) * (n_split * 12 + 4) > (size_t)kMergeStageBytes) {
    set_error("attn: too many splits for the merge's shared-memory staging");
    return B200_E_INVAL;
  }
  if (n_split > 1 && (!a->ws || !a->counters)) {
    set_error("attn: workspace/counters required when n_split > 1");
    return B200_E_INVAL;
  }
  AttnParams p = {};
  p.q = static_cast<const __half*>(a->q);
  p.kc = static_cast<const __half*>(a->kcache);
  p.vt = static_cast<const __half*>(a->vtcache);
  p.pos = a->pos;
  p.out = static_cast<__half*>(a->out);
  p.ws_o = static_cast<float*>(a->ws);
  p.ws_ml = reinterpret_cast<float2*>(static_cast<float*>(a->ws) + (size_t)a->T * a->Hq * n_split * 128);
  p.counters = a->counters;
  p.T = a->T, p.Hq = a->Hq, p.Hkv = a->Hkv, p.S = a->cache_seq, p.tps = a->tokens_per_seq;
  p.n_split = n_split, p.chunk = chunk, p.n_rep = a->Hq / a->Hkv;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.next_w = static_cast<const uint8_t*>(a->prefetch_next);
  p.next_bytes = a->prefetch_bytes;
  p.next_tiles = a->prefetch_tiles;
  p.next_grid = std::min(std::max(a->prefetch_tiles, 1), sm_count());
  p.next_window = prefetch_window_bytes();
  const int pf_early = tune_get("B200_PF_EARLY", 0);
  p.pf_early = pf_early;
  p.even = tune_get("B200_ATTN_EVEN", 0);
  p.stream_ef = tune_get("B200_KV_EF", 1);
  p.tl = timeline_slot();
  p.tlc = timeline_cta_slot();

  const size_t smem = kSmemBytes;
  static bool configured_dev[16] = {};  // cudaFuncSetAttribute is per device
  int dev = 0;
  cudaGetDevice(&dev);
  bool& configured = configured_dev[dev & 15];
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(attn_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      set_error(std::string("attn: cudaFuncSetAttribute: ") + cudaGetErrorString(e));
      return (int)e;
    }
    configured = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(a->Hkv, n_split, a->T);
  cfg.blockDim = dim3(kAttnThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (a->use_pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  cudaError_t e = cudaLaunchKernelEx(&cfg, attn_decode_kernel, p);
  if (e != cudaSuccess) {
    set_error(std::string("attn: launch: ") + cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}
