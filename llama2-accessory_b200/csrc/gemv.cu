// Fused W{2,3,4,16}A16 dequant-GEMV family for decode (T <= 32 tokens), sm_90a.
//
//   prologue : optional residual add + RMSNorm (components.py:41-53), x staged once per CTA in smem
//   main loop: packed weights streamed HBM -> smem ring by 1-D TMA bulk copies (UBLKCP) issued by a
//              producer warp that never waits on the previous kernel (weights are constants), so
//              under programmatic dependent launch the ring is already full when x arrives;
//              8 consumer warps split K, unpack W-bit fields straight into HMMA A fragments
//              (fp16 denormal trick: a masked field IS the half q*2^-24, no int->float ALU work)
//              and accumulate sum_k q[n,k]*x[k] in fp32 on the tensor pipe;
//   epilogue : cross-warp fixed-order reduction, y = s*(sum q x - z*sum x), then fp16 rounding and one of
//              plain store / fp32 logits / RoPE + KV-cache append / SiLU(a)*b.
//
// Arithmetic contract (DESIGN.md "numerics"): y[n] = sum_g s[n,g] * ( sum_{k in g} q[n,k] x[k]
//                                                               - z[n,g] sum_{k in g} x[k] )  in fp32.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <string>

#include "../../include/b200_decode.h"
#include "common.cuh"

#include "gemv_core.cuh"

namespace b200 {

// ------------------------------------------------------------------------------------------------
// Warp roles: 0..7 MMA consumers (split K inside a 16-row tile) | 8 producer (TMA bulk copies) |
// 9..10 epilogue (cross-warp reduction, scales, fused epilogue, global stores).  Everything between the
// roles is mbarrier-synchronised, so the dependent global loads of the epilogue never stall the MMA warps.
// ------------------------------------------------------------------------------------------------
template <int BITS, int NT, bool GROUPED, bool BIAS>
__device__ __forceinline__ void gemv_body(const GemvParams& p, GemvBias bias) {
  using C = Codec<BITS>;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* ring = smem;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * kSlotBytes);
  uint64_t* empty = full + p.stages;
  uint64_t* red_full = empty + p.stages;   // [2]
  uint64_t* red_empty = red_full + 2;      // [2]
  uint64_t* x_ready = red_empty + 2;       // [1] (+1 pad)
  float* red = reinterpret_cast<float*>(x_ready + 2);               // [2][8][NT*128]
  float* scratch = red + 2 * kConsumerWarps * NT * 128;             // [32*8]
  float* xsum = scratch + 32 * kConsumerWarps;                      // [32]
  float* csum = xsum + 32;                                          // [T][n_chunk64]
  __half* xs = reinterpret_cast<__half*>(csum + ((p.T * p.n_chunk64 + 3) & ~3));  // [T][x_stride]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  __shared__ int s_cols[32];
  __shared__ int s_T;
  if (tid == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kConsumerWarps);
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(&red_full[b], kConsumerWarps);
      mbar_init(&red_empty[b], kEpiWarps);
    }
    mbar_init(x_ready, kConsumerWarps);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) tl_min(p.tl, 0);
  pdl_launch_dependents();  // the next kernel may start prefetching its weights now

  // MoE: the column set (slots routed to this expert) comes from the router kernel
  int T = p.T;
  const int* cols = nullptr;
  if (p.slot_expert) {
    pdl_wait();
    if (tid == 0) {
      // [slot_lo, slot_hi) is a range of RANKS among the slots routed to this expert (in slot order), not of slot ids:
      // the launches of a token-group split then walk the weights ceil(routed / group) times instead of once per slot
      // group, and the launches past the routed count return without streaming anything.
      int n = 0, rank = 0;
      for (int sl = 0; sl < p.n_slots; ++sl)
        if (p.slot_expert[sl] == p.expert_id) {
          if (rank >= p.slot_lo && rank < p.slot_hi) s_cols[n++] = sl;
          ++rank;
        }
      s_T = n;
    }
    __syncthreads();
    T = s_T;
    if (T == 0) return;  // nobody routed here: stream nothing
    cols = s_cols;
  }
  const int nta = (T + 7) >> 3;
  // contiguous tile range per CTA: one CTA streams one contiguous region of the packed weights (DRAM-page friendly)
  const int tile_begin = (int)(((long long)p.n_tiles * blockIdx.x) / gridDim.x);
  const int tile_end = (int)(((long long)p.n_tiles * (blockIdx.x + 1)) / gridDim.x);
  const int slots_per_tile = (p.KB + kSlotBlocks - 1) / kSlotBlocks;
  constexpr bool grouped = GROUPED;  // p.G > 1, resolved by the host when it picks the instance

  if (warp == kConsumerWarps) {
    // ---------------- producer: weight stream, independent of any earlier kernel ----------------
    if (lane == 0) {
      if (blockIdx.x == 0 && p.const_pf && p.const_pf_bytes > 0) l2_prefetch(p.const_pf, (uint32_t)p.const_pf_bytes & ~15u);
      int stage = 0;
      uint32_t par = 0;
      for (int tile = tile_begin; tile < tile_end; ++tile) {
        const uint8_t* src = p.qw + (size_t)tile * p.KB * 512;
        for (int s = 0; s < slots_per_tile; ++s) {
          mbar_wait(&empty[stage], par ^ 1);
          const int nblk = min(kSlotBlocks, p.KB - s * kSlotBlocks);
          const uint32_t bytes = (uint32_t)nblk * 512u;
          mbar_arrive_expect_tx(&full[stage], bytes);
          if (p.stream_ef) bulk_g2s_hint(ring + (size_t)stage * kSlotBytes, src + (size_t)s * kSlotBytes, bytes, &full[stage], l2_policy_evict_first());
          else bulk_g2s(ring + (size_t)stage * kSlotBytes, src + (size_t)s * kSlotBytes, bytes, &full[stage]);
          if (++stage == p.stages) stage = 0, par ^= 1;
        }
      }
      // Own stream fully issued: pull this CTA's share of the NEXT kernel's first bytes into L2, so HBM keeps
      // streaming through our epilogue, the launch gap and the next kernel's prologue (one CTA per SM leaves
      // no room for a co-resident successor; the 50 MB L2 is the hand-over buffer instead).
      if (p.next_w && p.next_bytes > 0)
        prefetch_next_stream(p.next_w, p.next_bytes, p.next_tiles, p.next_grid, p.next_window, blockIdx.x, gridDim.x);
    }
    return;
  }

  if (warp > kConsumerWarps) {
    // ---------------- epilogue warps ----------------
    int elt = 0;
    epilogue_role<BITS, NT, BIAS>(p, T, cols, nta, grouped, tid - (kConsumerWarps + 1) * 32, lane, red, red_full, red_empty,
                            x_ready, xsum, elt, 0, bias);
    return;
  }

  // ---------------- MMA consumers ----------------
  pdl_wait();  // activations written by the previous kernel are now visible
  if (tid == 0) tl_max(p.tl, 4);
  stage_x(p, T, cols, xs, csum, xsum, scratch, tid);
  if (lane == 0) mbar_arrive(x_ready);
  if (tid == 0) tl_max(p.tl, 1);

  int stage = 0, lt = 0;
  uint32_t par = 0;
  long long c_full = 0, c_red = 0;
  const long long c_t0 = clock64();
  const bool prof = p.tl != nullptr && warp == 0;
  mma_phase<BITS, NT, GROUPED ? 1 : 0>(p, T, nta, grouped, ring, full, empty, red, red_full, red_empty, xs, csum, stage, par, lt, warp,
                      lane, c_full, c_red, prof);
  if (tid == 0) tl_max(p.tl, 2);
  if (prof && lane == 0) {  // cycles of MMA warp 0 summed over CTAs: [5] waiting for weights, [6] waiting for the epilogue, [7] whole loop
    atomicAdd(p.tl + 5, (unsigned long long)c_full);
    atomicAdd(p.tl + 6, (unsigned long long)c_red);
    atomicAdd(p.tl + 7, (unsigned long long)(clock64() - c_t0));
  }
}

template <int BITS, int NT, bool GROUPED>
__global__ void __launch_bounds__(kThreads, 1) gemv_kernel(const __grid_constant__ GemvParams p) {
  gemv_body<BITS, NT, GROUPED, false>(p, GemvBias{});
}
// the same kernel with the bias epilogue (B200_BIAS_ACC / _OUT): separate instances, so the bias-free ones are untouched
template <int BITS, int NT, bool GROUPED>
__global__ void __launch_bounds__(kThreads, 1) gemv_bias_kernel(const __grid_constant__ GemvBiasParams bp) {
  gemv_body<BITS, NT, GROUPED, true>(bp.p, bp.bias);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
template <int BITS, int NT, bool GROUPED, bool BIAS>
static int launch(const GemvParams& p, GemvBias bias, int grid, size_t smem, bool pdl, cudaStream_t st) {
  auto kfn = BIAS ? reinterpret_cast<const void*>(gemv_bias_kernel<BITS, NT, GROUPED>)
                  : reinterpret_cast<const void*>(gemv_kernel<BITS, NT, GROUPED>);
  static size_t configured_dev[16] = {};  // cudaFuncSetAttribute is per device
  int dev = 0;
  cudaGetDevice(&dev);
  size_t& configured = configured_dev[dev & 15];
  if (smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();  // do not leave the error sticky for the next launch check
      set_error(std::string("gemv: cudaFuncSetAttribute: ") + cudaGetErrorString(e));
      return (int)e;
    }
    configured = smem;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t e;
  if constexpr (BIAS) e = cudaLaunchKernelEx(&cfg, gemv_bias_kernel<BITS, NT, GROUPED>, GemvBiasParams{p, bias});
  else e = cudaLaunchKernelEx(&cfg, gemv_kernel<BITS, NT, GROUPED>, p);
  if (e != cudaSuccess) {
    set_error(std::string("gemv: launch: ") + cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

template <int BITS, bool GROUPED, bool BIAS>
static int launch_gb(int NT, const GemvParams& p, GemvBias bias, int grid, size_t smem, bool pdl, cudaStream_t st) {
  switch (NT) {
    case 1: return launch<BITS, 1, GROUPED, BIAS>(p, bias, grid, smem, pdl, st);
    case 2: return launch<BITS, 2, GROUPED, BIAS>(p, bias, grid, smem, pdl, st);
    default: return launch<BITS, 4, GROUPED, BIAS>(p, bias, grid, smem, pdl, st);
  }
}

template <int BITS, bool GROUPED>
static int launch_g(int NT, const GemvParams& p, GemvBias bias, int grid, size_t smem, bool pdl, cudaStream_t st) {
  return bias.b ? launch_gb<BITS, GROUPED, true>(NT, p, bias, grid, smem, pdl, st)
                : launch_gb<BITS, GROUPED, false>(NT, p, bias, grid, smem, pdl, st);
}

template <int BITS>
static int launch_nt(int NT, const GemvParams& p, GemvBias bias, int grid, size_t smem, bool pdl, cudaStream_t st) {
  // grouped scales exist for the W4 and W2 codecs only (build_gemv_params rejects the rest)
  if constexpr (BITS == 4 || BITS == 2) {
    if (p.G > 1) return launch_g<BITS, true>(NT, p, bias, grid, smem, pdl, st);
  }
  return launch_g<BITS, false>(NT, p, bias, grid, smem, pdl, st);
}

static size_t fixed_smem(int NT, int T, int n_chunk64, int x_stride, int stages) {
  size_t b = (size_t)stages * kSlotBytes + (size_t)stages * 16 + 6 * 8;
  b += (size_t)2 * kConsumerWarps * NT * 128 * 4;
  b += (size_t)32 * kConsumerWarps * 4 + 32 * 4;
  b += (size_t)((T * n_chunk64 + 3) & ~3) * 4;
  b += (size_t)T * x_stride * 2;
  return b;
}

}  // namespace b200

using namespace b200;

extern "C" size_t b200_gemv_weight_bytes(const b200_linear_t* lin) {
  if (!lin) return 0;
  size_t b = b200_packed_weight_bytes(lin->bits, lin->N, lin->K);
  if (lin->bits != 16) b += b200_packed_scale_bytes(lin->N, lin->K, lin->group_size);
  return b;
}

int b200::build_gemv_params(const b200_gemv_args_t* a, GemvParams* pp) {
  if (!a) return B200_E_INVAL;
  GemvParams& p = *pp;
  const b200_linear_t& L = a->lin;
  const int bits = L.bits;
  if (!(bits == 2 || bits == 3 || bits == 4 || bits == 16)) {
    set_error("gemv: bits must be 2, 3, 4 or 16");
    return B200_E_INVAL;
  }
  if (L.N <= 0 || (L.N & 15) || L.K <= 0 || (L.K & 63)) {
    set_error("gemv: N must be a multiple of 16 and K a multiple of 64");
    return B200_E_INVAL;
  }
  if (bits == 2 && (L.K & 127)) {
    set_error("gemv: W2 needs K % 128 == 0");
    return B200_E_INVAL;
  }
  if (a->T < 1 || a->T > 32) {
    set_error("gemv: T must be in 1..32 (loop over token groups on the host)");
    return B200_E_UNSUPPORTED;
  }
  if (!L.qweight || (bits != 16 && !L.scales) || !a->out) {
    set_error("gemv: null weight/scale/out pointer");
    return B200_E_INVAL;
  }
  const int kblk = bits == 4 ? 64 : bits == 2 ? 128 : bits == 3 ? 80 : 16;
  p = GemvParams{};
  p.bits = bits;
  p.qw = static_cast<const uint8_t*>(L.qweight);
  p.sz = static_cast<const __half2*>(L.scales);
  p.N = L.N;
  p.K = L.K;
  p.KB = (L.K + kblk - 1) / kblk;
  p.Kpad = p.KB * kblk;
  p.n_tiles = L.N / 16;
  const int gsz = (L.group_size <= 0 || L.group_size >= L.K) ? 0 : L.group_size;
  if (gsz) {
    if (bits == 3 || bits == 16) {
      set_error("gemv: grouped scales are supported for W4 (g64/g128) and W2 (g128); pack W3-grouped in the W4 container");
      return B200_E_UNSUPPORTED;
    }
    if ((gsz % kblk) || (L.K % gsz) || (gsz != 64 && gsz != 128)) {
      set_error("gemv: group_size must be 64 or 128 and a multiple of the codec k-block");
      return B200_E_UNSUPPORTED;
    }
    p.G = L.K / gsz;
    p.gb_mask = gsz / kblk - 1;
    p.gb_shift = (gsz / kblk) == 2 ? 1 : 0;
    p.gs_chunks = gsz / 64;
  } else {
    p.G = 1;
    p.gb_mask = 0x7fffffff;
    p.gb_shift = 0;
    p.gs_chunks = 0;
  }
  p.T = a->T;
  p.pro = a->prologue;
  if (p.pro == B200_PRO_RMSNORM) {
    if (!a->resid || !a->gamma || L.K > 8192) {
      set_error("gemv: RMSNorm prologue needs resid, gamma and K <= 8192");
      return B200_E_INVAL;
    }
  } else if (p.pro == B200_PRO_NONE) {
    if (!a->xin) {
      set_error("gemv: xin is NULL");
      return B200_E_INVAL;
    }
    if (L.K > 8192 * 2) {
      set_error("gemv: K > 16384 unsupported");
      return B200_E_UNSUPPORTED;
    }
  } else {
    return B200_E_INVAL;
  }
  p.xin = static_cast<const __half*>(a->xin);
  p.resid = static_cast<const __half*>(a->resid);
  p.delta = static_cast<const __half*>(a->delta);
  p.h_out = static_cast<__half*>(a->h_out);
  p.gamma = static_cast<const __half*>(a->gamma);
  p.eps = a->eps;
  p.epi = a->epilogue;
  p.out = a->out;
  if (p.epi == B200_EPI_QKV) {
    if (!a->rope || !a->pos || !a->kcache || !a->vtcache || a->tokens_per_seq < 1 || (a->n_q_rows & 127) ||
        (a->n_kv_rows & 127) || a->n_q_rows + 2 * a->n_kv_rows != L.N) {
      set_error("gemv: bad QKV epilogue arguments");
      return B200_E_INVAL;
    }
  } else if (p.epi == B200_EPI_SILU) {
    if (L.N & 31) return B200_E_INVAL;
  } else if (p.epi != B200_EPI_F16 && p.epi != B200_EPI_F32) {
    return B200_E_INVAL;
  }
  p.n_q_rows = a->n_q_rows;
  p.n_kv_rows = a->n_kv_rows;
  p.rope = reinterpret_cast<const float2*>(a->rope);
  p.pos = a->pos;
  p.tokens_per_seq = a->tokens_per_seq;
  p.kcache = static_cast<__half*>(a->kcache);
  p.vtcache = static_cast<__half*>(a->vtcache);
  p.cache_seq = a->cache_seq;
  p.hkv = a->n_kv_rows / 128;
  p.slot_expert = a->slot_expert;
  p.expert_id = a->expert_id;
  p.n_slots = a->n_slots;
  p.src_div = a->src_div > 0 ? a->src_div : 1;
  p.slot_lo = 0;
  p.slot_hi = a->n_slots;
  p.t_base = 0;
  if (a->slot_expert && (a->n_slots < 1 || a->n_slots > 32 || a->n_slots != a->T || a->epilogue == B200_EPI_QKV)) {
    set_error("gemv: MoE slot indirection needs 1 <= n_slots == T <= 32 and a non-QKV epilogue");
    return B200_E_INVAL;
  }
  if (a->bias_mode < B200_BIAS_NONE || a->bias_mode > B200_BIAS_OUT) {
    set_error("gemv: bias_mode must be 0 (none), 1 (B200_BIAS_ACC) or 2 (B200_BIAS_OUT)");
    return B200_E_INVAL;
  }
  if ((a->bias != nullptr) != (a->bias_mode != B200_BIAS_NONE)) {
    set_error("gemv: a bias needs bias_mode 1 or 2, and bias_mode 1 or 2 needs a bias");
    return B200_E_INVAL;
  }
  if (a->bias) {
    if (p.epi != B200_EPI_F16 && p.epi != B200_EPI_QKV) {
      set_error("gemv: a bias is supported with the fp16 and QKV epilogues only");
      return B200_E_INVAL;
    }
    if (a->slot_expert) {
      set_error("gemv: a bias cannot be combined with MoE slot indirection");
      return B200_E_INVAL;
    }
    if (a->ar_world > 1) {
      set_error("gemv: a bias cannot be combined with the fused all-reduce (it is added after the reduction)");
      return B200_E_INVAL;
    }
  }
  p.x_stride = p.Kpad + kXPad;
  p.n_chunk64 = L.K / 64;
  if (a->ar_world > 1) {
    // tensor-parallel all-reduce fused into this launch (bs = 1 only): LL push by the epilogue and / or LL sum by the prologue
    if (a->T != 1 || a->ar_world > 8 || a->ar_rank < 0 || a->ar_rank >= a->ar_world || !a->ar_step || a->ar_period < 1) {
      set_error("gemv: the fused all-reduce needs T == 1, 2 <= ar_world <= 8, a step counter and a sequence period");
      return B200_E_INVAL;
    }
    p.ll_step = a->ar_step;
    p.ll_period = a->ar_period;
    p.ll_err = a->ar_error;
    if (a->ar_out_peers) {
      if (p.epi != B200_EPI_F16 || (L.N & 1)) {
        set_error("gemv: ar_out_peers needs the fp16 epilogue");
        return B200_E_INVAL;
      }
      // every kernel pushes all N rows once; a MoE launch whose expert gets no routed token pushes nothing
      if (a->slot_expert) {
        set_error("gemv: ar_out_peers cannot be combined with MoE slot indirection");
        return B200_E_INVAL;
      }
      p.ll_out = 1;
      p.ll_out_id = a->ar_out_id;
      p.n_bcast = a->ar_world;
      for (int r = 0; r < a->ar_world; ++r) p.bcast[r] = static_cast<uint8_t*>(a->ar_out_peers[r]) + (size_t)a->ar_rank * L.N * 4;
      p.bcast_off = 0;
    }
    if (a->ar_in) {
      if (p.pro != B200_PRO_RMSNORM) {
        set_error("gemv: ar_in needs the RMSNorm prologue (the summed vector is the residual delta)");
        return B200_E_INVAL;
      }
      p.ll_in = 1;
      p.ll_in_id = a->ar_in_id;
      p.delta = static_cast<const __half*>(a->ar_in);
      p.n_delta = a->ar_world;
    }
  }

  return 0;
}

// Largest token group whose staged activations fit next to a ring of at least kMinStages slots.
static int pick_token_group(int T, int n_chunk64, int x_stride, size_t cap, int want_stages, int* stages_out) {
  constexpr int kMinStages = 3;
  for (int tg = T; tg >= 1; tg = (tg > 16 ? 16 : tg > 8 ? 8 : tg / 2)) {
    const int NT = tg <= 8 ? 1 : tg <= 16 ? 2 : 4;
    int stages = want_stages;
    while (stages > 2 && fixed_smem(NT, tg, n_chunk64, x_stride, stages) > cap) --stages;
    const bool fits = fixed_smem(NT, tg, n_chunk64, x_stride, stages) <= cap;
    if (fits && (stages >= kMinStages || stages == want_stages || tg == 1)) {
      *stages_out = stages;
      return tg;
    }
  }
  return 0;
}

extern "C" int b200_gemv(const b200_gemv_args_t* a, b200_stream_t stream) {
  GemvParams p0;
  const int rc = build_gemv_params(a, &p0);
  if (rc) return rc;
  if (gemv1_supported(a, p0)) return gemv1_launch(a, p0, static_cast<cudaStream_t>(stream));
  const b200_linear_t& L = a->lin;
  const int bits = L.bits;
  // dynamic shared memory budget: the opt-in limit minus the kernel's static shared memory (sz_s, rope_s, s_cols: 3.3 KB)
  const size_t cap = std::min<size_t>(smem_optin(), 227 * 1024) - 4096;
  static const int ring_kb = getenv("B200_GEMV_RING_KB") ? atoi(getenv("B200_GEMV_RING_KB")) : 128;
  int want = a->ring_bytes > 0 ? a->ring_bytes / kSlotBytes : (ring_kb * 1024) / kSlotBytes;
  want = std::max(2, std::min(want, 24));
  // The activations of all tokens of a launch are staged in shared memory beside the weight ring.  When T*K is too
  // large for that (e.g. T = 32 at K = 4096, T = 8 at K = 11008) the batch is walked in token groups: one launch per
  // group over the same weights, which the second and later groups find in the 50 MB L2.
  int stages = 0;
  const int tg = pick_token_group(a->T, p0.n_chunk64, p0.x_stride, cap, want, &stages);
  if (tg <= 0) {
    set_error("gemv: one token's activations do not fit in shared memory (K too large)");
    return B200_E_UNSUPPORTED;
  }
  static const int dbg = getenv("B200_GEMV_DBG") ? atoi(getenv("B200_GEMV_DBG")) : 0;
  static const int grid_mult = getenv("B200_GEMV_GRID_MULT") ? atoi(getenv("B200_GEMV_GRID_MULT")) : 1;
  const int grid = std::min(p0.n_tiles, sm_count() * std::max(1, grid_mult));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int t0 = 0; t0 < a->T; t0 += tg) {
    GemvParams p = p0;
    const int tn = std::min(tg, a->T - t0);
    p.T = tn;
    if (p.slot_expert) {
      p.slot_lo = t0, p.slot_hi = t0 + tn;  // ranks among the routed slots; rows of xin / out are addressed through the slot ids
    } else if (t0) {
      const size_t ko = (size_t)t0 * p.K;
      if (p.xin) p.xin += ko;
      if (p.resid) p.resid += ko;
      if (p.delta) p.delta += ko;
      if (p.h_out) p.h_out += ko;
      if (p.pos) p.pos += t0;
      p.t_base = t0;
      switch (p.epi) {
        case B200_EPI_F32: p.out = static_cast<float*>(p.out) + (size_t)t0 * p.N; break;
        case B200_EPI_SILU: p.out = static_cast<__half*>(p.out) + (size_t)t0 * (p.N >> 1); break;
        case B200_EPI_QKV: p.out = static_cast<__half*>(p.out) + (size_t)t0 * p.n_q_rows; break;
        default: p.out = static_cast<__half*>(p.out) + (size_t)t0 * p.N; break;
      }
    }
    const int NT = tn <= 8 ? 1 : tn <= 16 ? 2 : 4;
    const size_t smem = fixed_smem(NT, tn, p.n_chunk64, p.x_stride, stages);
    p.stages = stages;
    p.dbg = dbg;
    p.tl = timeline_slot();
    p.keep_const = tune_get("B200_KEEP_CONST", 1);
    p.stream_ef = tune_get("B200_STREAM_EF", 1);
    p.const_pf = (t0 == 0 && tune_get("B200_CONST_PF", 1)) ? static_cast<const uint8_t*>(a->prefetch_const) : nullptr;
    p.const_pf_bytes = a->prefetch_const_bytes;
    const bool last = t0 + tn >= a->T;
    p.next_w = last ? static_cast<const uint8_t*>(a->prefetch_next) : nullptr;
    p.next_bytes = last ? a->prefetch_bytes : 0;
    p.next_tiles = a->prefetch_tiles;
    p.next_grid = std::min(std::max(a->prefetch_tiles, 1), sm_count());
    p.next_window = prefetch_window_bytes();
    const GemvBias bias{static_cast<const __half*>(a->bias), a->bias_mode};
    int r;
    switch (bits) {
      case 4: r = launch_nt<4>(NT, p, bias, grid, smem, a->use_pdl != 0, st); break;
      case 2: r = launch_nt<2>(NT, p, bias, grid, smem, a->use_pdl != 0, st); break;
      case 3: r = launch_nt<3>(NT, p, bias, grid, smem, a->use_pdl != 0, st); break;
      default: r = launch_nt<16>(NT, p, bias, grid, smem, a->use_pdl != 0, st); break;
    }
    if (r) return r;
  }
  return 0;
}
