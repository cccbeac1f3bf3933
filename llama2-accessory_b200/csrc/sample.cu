// Device-side token selection and generate-loop bookkeeping (SURVEY.md 8f rank 2): what MetaModel.generate does
// on the host after every forward_inference call (meta.py:434-461, 550-565), moved into two small kernels so that
// a whole decode step -- model, sampling, prompt forcing, stop detection -- replays as one CUDA graph with no
// per-token host synchronisation.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <string>

#include "../../include/b200_decode.h"
#include "common.cuh"

namespace b200 {

void set_error(const std::string& s);
size_t smem_optin();

constexpr int kSampleThreads = 1024;

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();  // previous use of red[] is over
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < kSampleThreads / 32; ++w) t += red[w];  // fixed order: same value in every thread
  return t;
}

__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = -INFINITY;
#pragma unroll
  for (int w = 0; w < kSampleThreads / 32; ++w) t = fmaxf(t, red[w]);
  return t;
}

// Top-p (nucleus) sampling of one row per CTA, meta.py:550-565 without the sort:
//   p = softmax(logits / temperature)
//   keep token i  <=>  sum of the probabilities strictly larger than p_i  <=  top_p
//       (= "cumsum before it in descending order <= top_p", the reference's mask; tokens of equal probability
//        are kept or dropped together, the only difference from torch.sort's arbitrary order among ties)
//   draw from the kept tokens, renormalised, by inverse CDF in index order with the caller's uniform u[t] in [0, 1).
// The cut is found by bisection on the bit pattern of the threshold (positive floats order like integers): 30 passes
// over the V probabilities held in shared memory.
__global__ void __launch_bounds__(kSampleThreads, 1)
sample_top_p_kernel(const float* __restrict__ logits, const float* __restrict__ u, long long* __restrict__ next, int V,
                    float inv_temperature, float top_p) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float prob[];  // [V]
  __shared__ float red[kSampleThreads / 32];
  __shared__ float wtot[kSampleThreads / 32];
  __shared__ int s_tok;
  const int t = blockIdx.x, tid = threadIdx.x;
  const float* row = logits + (size_t)t * V;

  float m = -INFINITY;
  for (int i = tid; i < V; i += kSampleThreads) m = fmaxf(m, row[i]);
  m = block_max(m, red);
  float s = 0.f;
  for (int i = tid; i < V; i += kSampleThreads) {
    const float e = expf((row[i] - m) * inv_temperature);
    prob[i] = e;
    s += e;
  }
  s = block_sum(s, red);
  const float inv = 1.0f / s;
  for (int i = tid; i < V; i += kSampleThreads) prob[i] *= inv;
  __syncthreads();

  // smallest threshold x (as a bit pattern) with  G(x) = sum_{p_j > x} p_j <= top_p ;  G(p_max) = 0 always qualifies
  unsigned lo = 0u, hi = __float_as_uint(inv);  // p_max = exp(0) / s
  if (top_p < 1.0f) {
    while (lo < hi) {
      const unsigned mid = lo + ((hi - lo) >> 1);
      const float x = __uint_as_float(mid);
      float g = 0.f;
      for (int i = tid; i < V; i += kSampleThreads) {
        const float p = prob[i];
        if (p > x) g += p;
      }
      g = block_sum(g, red);
      if (g <= top_p) hi = mid; else lo = mid + 1;
    }
  } else {
    hi = 0u;
  }
  const float cut = __uint_as_float(hi);  // keep p_i >= cut

  // inverse CDF over the kept tokens in index order: thread tid owns the contiguous chunk [c0, c1)
  const int chunk = (V + kSampleThreads - 1) / kSampleThreads;
  const int c0 = min(V, tid * chunk), c1 = min(V, c0 + chunk);
  float part = 0.f;
  for (int i = c0; i < c1; ++i) {
    const float p = prob[i];
    if (p >= cut && p > 0.f) part += p;
  }
  // block-wide exclusive scan of the chunk sums (warp scan, then scan of the 32 warp totals)
  float incl = part;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_up_sync(0xffffffffu, incl, o);
    if ((tid & 31) >= o) incl += v;
  }
  if ((tid & 31) == 31) wtot[tid >> 5] = incl;
  if (tid == 0) s_tok = -1;
  __syncthreads();
  float base = 0.f, total = 0.f;
#pragma unroll
  for (int w = 0; w < kSampleThreads / 32; ++w) {
    if (w < (tid >> 5)) base += wtot[w];
    total += wtot[w];
  }
  const float excl = base + incl - part;
  const float target = u[t] * total;
  if (part > 0.f && excl <= target && target < excl + part) {
    float acc = excl;
    int pick = -1;
    for (int i = c0; i < c1; ++i) {
      const float p = prob[i];
      if (p >= cut && p > 0.f) {
        pick = i;
        acc += p;
        if (target < acc) break;
      }
    }
    s_tok = pick;
  }
  __syncthreads();
  const bool unclaimed = s_tok < 0;  // read by everybody before anybody may write again
  __syncthreads();
  if (unclaimed) {
    // u * total rounded onto (or past) the end of the last interval: take the last kept token
    int last = -1;
    for (int i = c1 - 1; i >= c0; --i)
      if (prob[i] >= cut && prob[i] > 0.f) { last = i; break; }
    if (last >= 0) atomicMax(&s_tok, last);
  }
  __syncthreads();
  if (tid == 0) next[t] = s_tok < 0 ? 0 : s_tok;
}

// Top-p sampling for vocabularies whose probabilities do not fit in shared memory (V > ~57800 on the H100): the same
// rule and the same draw as sample_top_p_kernel, with nothing stored per token.  Every pass re-reads the logits row
// (L2-resident: 412 KB at V = 103168) and recomputes p_i = exp((l_i - max) / T) / sum, bit for bit the value the other
// kernel keeps in shared memory.  The threshold is found by a radix descent on the bit pattern of p (4 passes of 8 bits,
// most significant first) instead of 30 bisection passes: each pass histograms the probability mass of the tokens that
// share the prefix fixed so far, and keeps the lowest non-empty bin whose largest member still has at most top_p of
// mass strictly above it.  The masses are summed in 2^-56 fixed point (exact for every p >= 2^-33; a smaller p counts
// as 2^-56), so the integer atomics are order-independent and the cut is the same on every run.  A 64-bit sum is kept as
// two 32-bit words with the carry taken from the low word's atomic: shared-memory atomics are native at 32 bits, while a
// 64-bit add is a compare-and-swap loop that spins under the contention of a whole vocabulary landing in a few bins.
constexpr int kRadixBins = 256;
constexpr float kFix = 72057594037927936.0f;  // 2^56

__device__ __forceinline__ unsigned long long fixed_mass(float p) {
  const unsigned long long f = __float2ull_rz(p * kFix);
  return f ? f : 1ull;  // p > 0 always counts, so a bin is non-empty iff its mass is
}

__device__ __forceinline__ void add_mass(unsigned* lo, unsigned* hi, unsigned long long v) {
  const unsigned vl = (unsigned)v, vh = (unsigned)(v >> 32);
  const unsigned old = atomicAdd(lo, vl);
  const unsigned up = vh + (old + vl < old ? 1u : 0u);  // + the carry out of the low word
  if (up) atomicAdd(hi, up);
}

__global__ void __launch_bounds__(kSampleThreads, 1)
sample_top_p_radix_kernel(const float* __restrict__ logits, const float* __restrict__ u, long long* __restrict__ next,
                          int V, float inv_temperature, float top_p) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ unsigned hist_lo[kRadixBins], hist_hi[kRadixBins];
  __shared__ float red[kSampleThreads / 32];
  __shared__ float wtot[kSampleThreads / 32];
  __shared__ unsigned s_prefix;
  __shared__ unsigned long long s_above;
  __shared__ int s_tok;
  const int t = blockIdx.x, tid = threadIdx.x;
  const float* row = logits + (size_t)t * V;

  float m = -INFINITY;
  for (int i = tid; i < V; i += kSampleThreads) m = fmaxf(m, row[i]);
  m = block_max(m, red);
  float s = 0.f;
  for (int i = tid; i < V; i += kSampleThreads) s += expf((row[i] - m) * inv_temperature);
  s = block_sum(s, red);
  const float inv = 1.0f / s;
  const auto prob = [&](int i) { return expf((row[i] - m) * inv_temperature) * inv; };

  unsigned prefix = 0u;  // bit pattern of the cut, fixed from the top down
  if (top_p < 1.0f) {
    const unsigned long long limit = __float2ull_rz(top_p * kFix);
    unsigned long long above = 0ull;  // mass of the tokens whose pattern is above every pattern with this prefix
    for (int shift = 24; shift >= 0; shift -= 8) {
      if (tid < kRadixBins) hist_lo[tid] = hist_hi[tid] = 0u;
      __syncthreads();
      const unsigned fixed = shift == 24 ? 0u : ~0u << (shift + 8);
      for (int i = tid; i < V; i += kSampleThreads) {
        const float p = prob(i);
        const unsigned b = __float_as_uint(p);
        const int d = (b >> shift) & (kRadixBins - 1);
        if (p > 0.f && (b & fixed) == prefix) add_mass(&hist_lo[d], &hist_hi[d], fixed_mass(p));
      }
      __syncthreads();
      if (tid < 32) {
        // lane l owns bins [8l, 8l + 8); mass of the bins above lane l's = suffix sum over the higher lanes
        unsigned long long h[8], own = 0ull;
#pragma unroll
        for (int j = 0; j < 8; ++j) own += (h[j] = (unsigned long long)hist_hi[8 * tid + j] << 32 | hist_lo[8 * tid + j]);
        unsigned long long higher = own;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned long long v = __shfl_down_sync(0xffffffffu, higher, o);
          if (tid + o < 32) higher += v;
        }
        unsigned long long a = above + higher - own;  // mass above bin 8l + 7
        int bin = -1;
        unsigned long long bin_above = 0ull;
#pragma unroll
        for (int j = 7; j >= 0; --j) {
          if (h[j] && a <= limit) { bin = 8 * tid + j; bin_above = a; }
          a += h[j];
        }
        // the lowest qualifying bin: masses above grow towards lower bins, so the qualifying lanes are the upper ones
        const unsigned have = __ballot_sync(0xffffffffu, bin >= 0);
        if (have && tid == __ffs(have) - 1) {
          s_prefix = prefix | ((unsigned)bin << shift);
          s_above = bin_above;
        }
      }
      __syncthreads();
      prefix = s_prefix;
      above = s_above;
    }
  }

  // inverse CDF over the kept tokens in index order, as in sample_top_p_kernel: thread tid owns the chunk [c0, c1)
  const float cut = __uint_as_float(prefix);  // keep p_i >= cut
  const int chunk = (V + kSampleThreads - 1) / kSampleThreads;
  const int c0 = min(V, tid * chunk), c1 = min(V, c0 + chunk);
  float part = 0.f;
  for (int i = c0; i < c1; ++i) {
    const float p = prob(i);
    if (p >= cut && p > 0.f) part += p;
  }
  // block-wide exclusive scan of the chunk sums (warp scan, then scan of the 32 warp totals)
  float incl = part;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_up_sync(0xffffffffu, incl, o);
    if ((tid & 31) >= o) incl += v;
  }
  if ((tid & 31) == 31) wtot[tid >> 5] = incl;
  if (tid == 0) s_tok = -1;
  __syncthreads();
  float base = 0.f, total = 0.f;
#pragma unroll
  for (int w = 0; w < kSampleThreads / 32; ++w) {
    if (w < (tid >> 5)) base += wtot[w];
    total += wtot[w];
  }
  const float excl = base + incl - part;
  const float target = u[t] * total;
  if (part > 0.f && excl <= target && target < excl + part) {
    float acc = excl;
    int pick = -1;
    for (int i = c0; i < c1; ++i) {
      const float p = prob(i);
      if (p >= cut && p > 0.f) {
        pick = i;
        acc += p;
        if (target < acc) break;
      }
    }
    s_tok = pick;
  }
  __syncthreads();
  const bool unclaimed = s_tok < 0;  // read by everybody before anybody may write again
  __syncthreads();
  if (unclaimed) {
    // u * total rounded onto (or past) the end of the last interval: take the last kept token
    int last = -1;
    for (int i = c1 - 1; i >= c0; --i) {
      const float p = prob(i);
      if (p >= cut && p > 0.f) { last = i; break; }
    }
    if (last >= 0) atomicMax(&s_tok, last);
  }
  __syncthreads();
  if (tid == 0) next[t] = s_tok < 0 ? 0 : s_tok;
}

// One thread per sequence: meta.py:446-461 for position cur = *cur_pos.
//   forced token while the position is still inside the sequence's own prompt (input_text_mask, :446-448),
//   tokens[:, cur] = next (:449), stop bookkeeping in the reference's order (:451-459: first matching stop sequence
//   wins, a match ending on a prompt token does not count), then the engine's inputs for the next step:
//   step_tokens[b] = next, step_pos[b] = cur, *cur_pos = cur + 1, *n_stopped = number of finished sequences.
__global__ void generate_update_kernel(const long long* __restrict__ sampled, long long* __restrict__ tokens,
                                       const unsigned char* __restrict__ text_mask, int total_len, int bsz,
                                       const long long* __restrict__ stop_seqs, const int* __restrict__ stop_lens,
                                       int n_stop, int max_stop_len, unsigned char* __restrict__ stopped,
                                       int* __restrict__ stop_pos, long long* __restrict__ step_tokens,
                                       int* __restrict__ step_pos, int* __restrict__ cur_pos, int* __restrict__ n_stopped) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ int s_count;
  if (threadIdx.x == 0) s_count = 0;
  __syncthreads();
  const int b = threadIdx.x;
  const int cur = *cur_pos;
  if (b < bsz && cur < total_len) {
    long long* row = tokens + (size_t)b * total_len;
    const bool forced = text_mask[(size_t)b * total_len + cur] != 0;
    const long long nt = forced ? row[cur] : sampled[b];
    row[cur] = nt;
    bool st = stopped[b] != 0;
    int sp = st ? stop_pos[b] : cur + 1;
    for (int s = 0; s < n_stop; ++s) {
      const int L = stop_lens[s];
      if (L < 1 || cur + 1 - L < 0) continue;
      bool match = true;
      for (int j = 0; j < L; ++j) match = match && (row[cur + 1 - L + j] == stop_seqs[(size_t)s * max_stop_len + j]);
      if (match && !forced && !st) {
        sp = cur + 1 - L;
        st = true;
      }
    }
    stopped[b] = st ? 1 : 0;
    stop_pos[b] = sp;
    step_tokens[b] = nt;
    step_pos[b] = cur;
    if (st) atomicAdd(&s_count, 1);
  } else if (b < bsz) {
    if (stopped[b]) atomicAdd(&s_count, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    *n_stopped = s_count;
    if (cur < total_len) *cur_pos = cur + 1;
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_sample_top_p(const float* logits, const float* uniform, int64_t* next, int T, int V,
                                 float temperature, float top_p, b200_stream_t stream) {
  if (!logits || !uniform || !next || T < 1 || V < 1) {
    set_error("sample_top_p: bad arguments");
    return B200_E_INVAL;
  }
  if (!(temperature > 0.f) || !(top_p > 0.f)) {
    set_error("sample_top_p: temperature and top_p must be > 0 (temperature 0 is b200_argmax)");
    return B200_E_INVAL;
  }
  const size_t smem = (size_t)V * sizeof(float);
  if (smem + 1024 > smem_optin()) {
    // the probabilities do not fit in shared memory: recompute them from the logits row on every pass
    sample_top_p_radix_kernel<<<T, kSampleThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        logits, uniform, reinterpret_cast<long long*>(next), V, 1.0f / temperature, top_p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      set_error(std::string("sample_top_p: ") + cudaGetErrorString(e));
      return (int)e;
    }
    return 0;
  }
  static size_t configured_dev[16] = {};  // cudaFuncSetAttribute is per device
  int dev = 0;
  cudaGetDevice(&dev);
  size_t& configured = configured_dev[dev & 15];
  if (smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(sample_top_p_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      set_error(std::string("sample_top_p: cudaFuncSetAttribute: ") + cudaGetErrorString(e));
      return (int)e;
    }
    configured = smem;
  }
  sample_top_p_kernel<<<T, kSampleThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      logits, uniform, reinterpret_cast<long long*>(next), V, 1.0f / temperature, top_p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error(std::string("sample_top_p: ") + cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

extern "C" int b200_generate_update(const b200_generate_state_t* s, const int64_t* sampled, b200_stream_t stream) {
  if (!s || !sampled || !s->tokens || !s->text_mask || !s->stopped || !s->stop_pos || !s->step_tokens || !s->step_pos ||
      !s->cur_pos || !s->n_stopped || s->bsz < 1 || s->bsz > 1024 || s->total_len < 1 ||
      (s->n_stop > 0 && (!s->stop_seqs || !s->stop_lens || s->max_stop_len < 1))) {
    set_error("generate_update: bad arguments");
    return B200_E_INVAL;
  }
  const int threads = (s->bsz + 31) / 32 * 32;
  generate_update_kernel<<<1, threads, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(sampled), reinterpret_cast<long long*>(s->tokens), s->text_mask, s->total_len,
      s->bsz, reinterpret_cast<const long long*>(s->stop_seqs), s->stop_lens, s->n_stop, s->max_stop_len, s->stopped,
      s->stop_pos, reinterpret_cast<long long*>(s->step_tokens), s->step_pos, s->cur_pos, s->n_stopped);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error(std::string("generate_update: ") + cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}
