// Mixtral top-k MoE glue (accessory/model/LLM/mixtral.py:266-294, mixtral_sparse.py:405-489): router, expert FFN
// driver, combine.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <string>

#include "../../include/b200_decode.h"
#include "common.cuh"

namespace b200 {
void set_error(const std::string& s);

constexpr int kRouteThreads = 256;
constexpr int kMaxExperts = 64;

struct RouteParams {
  int T, D, E, topk;
  const __half* resid;
  const __half* delta;
  __half* h_out;
  const __half* gamma;
  float eps;
  const __half* gate_w;
  __half* xn_out;
  __half* slot_weight;
  int* slot_expert;
};

// One CTA per token: residual add, RMSNorm (components.py:41-53), gate logits (fp16 F.linear), then one of two score
// rules:
//   kScoresF32 = false (mixtral.py:272-281): softmax in fp32 -> fp16, top-k on the fp16 scores, renormalise in fp16;
//   kScoresF32 = true  (mixtral_sparse.py:417-428): softmax in fp32, top-k on the fp32 scores, fp32 sum of the chosen
//                      scores, weight = fp16(score / sum) rounded once.
template <bool kScoresF32>
__global__ void __launch_bounds__(kRouteThreads) moe_route_kernel(const __grid_constant__ RouteParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  __half* xs = reinterpret_cast<__half*>(smem);  // [D]
  __shared__ float s_part[kRouteThreads / 32];
  __shared__ float s_logit[kMaxExperts];
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nvec = p.D >> 3;
  float ssq = 0.f;
  for (int u = tid; u < nvec; u += kRouteThreads) {
    uint4 a = *reinterpret_cast<const uint4*>(p.resid + (size_t)t * p.D + (size_t)u * 8);
    if (p.delta) {
      const uint4 b = *reinterpret_cast<const uint4*>(p.delta + (size_t)t * p.D + (size_t)u * 8);
      __half2* ha = reinterpret_cast<__half2*>(&a);
      const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
      for (int j = 0; j < 4; ++j) ha[j] = __hadd2(ha[j], hb[j]);
    }
    if (p.h_out) *reinterpret_cast<uint4*>(p.h_out + (size_t)t * p.D + (size_t)u * 8) = a;
    *reinterpret_cast<uint4*>(xs + (size_t)u * 8) = a;
    const __half2* h = reinterpret_cast<const __half2*>(&a);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      ssq = fmaf(f.x, f.x, ssq);
      ssq = fmaf(f.y, f.y, ssq);
    }
  }
  ssq = warp_sum(ssq);
  if (lane == 0) s_part[warp] = ssq;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < kRouteThreads / 32; ++w) tot += s_part[w];
  const float rstd = 1.0f / sqrtf(tot / (float)p.D + p.eps);
  for (int u = tid; u < nvec; u += kRouteThreads) {
    const uint4 a = *reinterpret_cast<const uint4*>(xs + (size_t)u * 8);
    const uint4 gm = *reinterpret_cast<const uint4*>(p.gamma + (size_t)u * 8);
    uint4 o;
    const __half2* h = reinterpret_cast<const __half2*>(&a);
    const __half2* gh = reinterpret_cast<const __half2*>(&gm);
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      oh[j] = __hmul2(__floats2half2_rn(f.x * rstd, f.y * rstd), gh[j]);
    }
    *reinterpret_cast<uint4*>(xs + (size_t)u * 8) = o;
    *reinterpret_cast<uint4*>(p.xn_out + (size_t)t * p.D + (size_t)u * 8) = o;
  }
  __syncthreads();
  // gate logits: one warp per expert
  for (int e = warp; e < p.E; e += kRouteThreads / 32) {
    float acc = 0.f;
    for (int u = lane; u < nvec; u += 32) {
      const uint4 a = *reinterpret_cast<const uint4*>(xs + (size_t)u * 8);
      const uint4 w = *reinterpret_cast<const uint4*>(p.gate_w + (size_t)e * p.D + (size_t)u * 8);
      const __half2* h = reinterpret_cast<const __half2*>(&a);
      const __half2* wh = reinterpret_cast<const __half2*>(&w);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]), g = __half22float2(wh[j]);
        acc = fmaf(f.x, g.x, acc);
        acc = fmaf(f.y, g.y, acc);
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) s_logit[e] = __half2float(__float2half_rn(acc));  // F.linear output is fp16
  }
  __syncthreads();
  if (tid == 0) {
    float mx = -INFINITY;
    for (int e = 0; e < p.E; ++e) mx = fmaxf(mx, s_logit[e]);
    float den = 0.f;
    for (int e = 0; e < p.E; ++e) den += expf(s_logit[e] - mx);
    float sc[kMaxExperts];
    for (int e = 0; e < p.E; ++e) {
      const float v = expf(s_logit[e] - mx) / den;
      sc[e] = kScoresF32 ? v : __half2float(__float2half_rn(v));
    }
    // top-k on the scores (fp16-valued or fp32); ties -> lowest index first
    int idx[8];
    float val[8];
    for (int j = 0; j < p.topk; ++j) {
      int b = -1;
      float bv = -INFINITY;
      for (int e = 0; e < p.E; ++e) {
        bool used = false;
        for (int q = 0; q < j; ++q) used |= (idx[q] == e);
        if (!used && sc[e] > bv) bv = sc[e], b = e;
      }
      idx[j] = b, val[j] = bv;
    }
    float sum = 0.f;
    for (int j = 0; j < p.topk; ++j) sum += val[j];
    // fp16 rule: .sum(dim=-1) of a half tensor is rounded to fp16; fp32 rule: the sum stays fp32
    const float den_k = kScoresF32 ? sum : __half2float(__float2half_rn(sum));
    for (int j = 0; j < p.topk; ++j) {
      p.slot_expert[t * p.topk + j] = idx[j];
      p.slot_weight[t * p.topk + j] = __float2half_rn(val[j] / den_k);
    }
  }
}

// out[t][d] = fp16( sum_j fp16(w[t,j] * y_slot[t*topk+j][d]) ) over the slots whose expert lives here.
__global__ void moe_combine_kernel(const __half* __restrict__ y_slot, const __half* __restrict__ w,
                                   const int* __restrict__ slot_expert, int e_first, int e_count,
                                   __half* __restrict__ out, int D, int topk) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = 0.f;
    for (int j = 0; j < topk; ++j) {
      const int sl = t * topk + j, e = slot_expert[sl];
      if (e >= e_first && e < e_first + e_count)
        acc += __half2float(__hmul(y_slot[(size_t)sl * D + d], w[sl]));
    }
    out[(size_t)t * D + d] = __float2half_rn(acc);
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_moe_route(const b200_moe_route_args_t* a, b200_stream_t stream) {
  if (!a || !a->resid || !a->gamma || !a->gate_w || !a->xn_out || !a->slot_weight || !a->slot_expert) {
    set_error("moe_route: null pointer");
    return B200_E_INVAL;
  }
  if (a->T < 1 || a->D < 8 || (a->D & 7) || a->E < 1 || a->E > kMaxExperts || a->topk < 1 || a->topk > 8 ||
      a->topk > a->E) {
    set_error("moe_route: unsupported shape");
    return B200_E_UNSUPPORTED;
  }
  if (a->scores_f32 != 0 && a->scores_f32 != 1) {
    set_error("moe_route: scores_f32 must be 0 (fp16 scores) or 1 (fp32 scores)");
    return B200_E_INVAL;
  }
  RouteParams p = {};
  p.T = a->T, p.D = a->D, p.E = a->E, p.topk = a->topk;
  p.resid = static_cast<const __half*>(a->resid);
  p.delta = static_cast<const __half*>(a->delta);
  p.h_out = static_cast<__half*>(a->h_out);
  p.gamma = static_cast<const __half*>(a->gamma);
  p.eps = a->eps;
  p.gate_w = static_cast<const __half*>(a->gate_w);
  p.xn_out = static_cast<__half*>(a->xn_out);
  p.slot_weight = static_cast<__half*>(a->slot_weight);
  p.slot_expert = a->slot_expert;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(a->T);
  cfg.blockDim = dim3(kRouteThreads);
  cfg.dynamicSmemBytes = (size_t)a->D * 2;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = a->use_pdl ? 1 : 0;
  cudaError_t e = a->scores_f32 ? cudaLaunchKernelEx(&cfg, moe_route_kernel<true>, p)
                                 : cudaLaunchKernelEx(&cfg, moe_route_kernel<false>, p);
  if (e != cudaSuccess) {
    set_error(std::string("moe_route: ") + cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

extern "C" int b200_moe_expert_ffn(const b200_moe_ffn_args_t* a, b200_stream_t stream) {
  if (!a || !a->w13 || !a->w2 || !a->xn || !a->slot_expert || !a->act || !a->y_slot) {
    set_error("moe_expert_ffn: null pointer");
    return B200_E_INVAL;
  }
  const int n_slots = a->T * a->topk;
  if (n_slots < 1 || n_slots > 32) {
    set_error("moe_expert_ffn: T*topk must be in 1..32 (split the token batch)");
    return B200_E_UNSUPPORTED;
  }
  for (int i = 0; i < a->e_count; ++i) {
    b200_gemv_args_t g = {};
    g.lin = a->w13[i];
    g.T = n_slots;
    g.prologue = B200_PRO_NONE;
    g.xin = a->xn;
    g.epilogue = B200_EPI_SILU;
    g.out = a->act;
    g.slot_expert = a->slot_expert;
    g.expert_id = a->e_first + i;
    g.n_slots = n_slots;
    g.src_div = a->topk;
    g.use_pdl = a->use_pdl;
    int rc = b200_gemv(&g, stream);
    if (rc) return rc;
    b200_gemv_args_t d = {};
    d.lin = a->w2[i];
    d.T = n_slots;
    d.prologue = B200_PRO_NONE;
    d.xin = a->act;
    d.epilogue = B200_EPI_F16;
    d.out = a->y_slot;
    d.slot_expert = a->slot_expert;
    d.expert_id = a->e_first + i;
    d.n_slots = n_slots;
    d.src_div = 1;
    d.use_pdl = a->use_pdl;
    rc = b200_gemv(&d, stream);
    if (rc) return rc;
  }
  return 0;
}

extern "C" int b200_moe_combine(const void* y_slot, const void* slot_weight, const int32_t* slot_expert,
                                int e_first, int e_count, void* out, int T, int D, int topk,
                                b200_stream_t stream) {
  if (!y_slot || !slot_weight || !slot_expert || !out || T < 1 || D < 1 || topk < 1) return B200_E_INVAL;
  moe_combine_kernel<<<T, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(y_slot), static_cast<const __half*>(slot_weight), slot_expert, e_first, e_count,
      static_cast<__half*>(out), D, topk);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error(std::string("moe_combine: ") + cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}
