// Library plumbing (errors, device info) and the small glue kernels of the decode step.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdlib>
#include <cstring>
#include <string>

#include "../../include/b200_decode.h"
#include "common.cuh"

namespace b200 {

static thread_local std::string g_err;
void set_error(const std::string& s) { g_err = s; }

static unsigned long long* g_tl = nullptr;
static int g_tl_cap = 0, g_tl_next = 0;
// Tuning knobs: b200_tune(name, value) overrides, else the environment variable of that name, else the default.
// Read at ENQUEUE time (a captured graph keeps the values it was captured with).
struct TuneEntry { char name[40]; int value; };
static TuneEntry g_tune[32];
static int g_n_tune = 0;
int tune_get(const char* name, int dflt) {
  for (int i = 0; i < g_n_tune; ++i)
    if (!strcmp(g_tune[i].name, name)) return g_tune[i].value;
  const char* e = getenv(name);
  return e ? atoi(e) : dflt;
}
int prefetch_window_bytes() { return tune_get("B200_PF_KB", 96) * 1024; }
static unsigned long long* g_tlc = nullptr;
static int g_tlc_first = 0, g_tlc_rows = 0, g_tlc_ctas = 0;
unsigned long long* timeline_slot() {
  if (!g_tl || g_tl_next >= g_tl_cap) return nullptr;
  return g_tl + 8 * (size_t)(g_tl_next++);
}
// per-CTA stamp block of the launch that just took timeline row `g_tl_next - 1` (call right after timeline_slot())
unsigned long long* timeline_cta_slot() {
  const int row = g_tl_next - 1;
  if (!g_tl || !g_tlc || row < g_tlc_first || row >= g_tlc_first + g_tlc_rows) return nullptr;
  return g_tlc + (size_t)(row - g_tlc_first) * g_tlc_ctas * 16;
}

}  // namespace b200
extern "C" int b200_tune(const char* name, int value) {
  using namespace b200;
  if (!name || strlen(name) >= sizeof(g_tune[0].name)) return B200_E_INVAL;
  for (int i = 0; i < g_n_tune; ++i)
    if (!strcmp(g_tune[i].name, name)) {
      g_tune[i].value = value;
      return 0;
    }
  if (g_n_tune >= 32) return B200_E_INVAL;
  strcpy(g_tune[g_n_tune].name, name);
  g_tune[g_n_tune++].value = value;
  return 0;
}
namespace b200 {
static int g_sm = 0;
static size_t g_smem = 0;
static void query() {
  if (g_sm) return;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    g_sm = 132;
    g_smem = 227 * 1024;
    return;
  }
  int v = 0;
  cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
  g_sm = v > 0 ? v : 132;
  cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  g_smem = v > 0 ? (size_t)v : 227 * 1024;
}
int sm_count() {
  query();
  return g_sm;
}
size_t smem_optin() {
  query();
  return g_smem;
}

__global__ void embed_kernel(const long long* __restrict__ tokens, const uint4* __restrict__ table,
                             uint4* __restrict__ h, int D8, int vocab) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x;
  long long id = tokens[t];
  if (id < 0) id = 0;
  if (id >= vocab) id = vocab - 1;
  for (int i = threadIdx.x; i < D8; i += blockDim.x) h[(size_t)t * D8 + i] = table[(size_t)id * D8 + i];
}

__global__ void argmax_kernel(const float* __restrict__ logits, long long* __restrict__ next, int V) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sv[32];
  __shared__ int si[32];
  const int t = blockIdx.x;
  const float* row = logits + (size_t)t * V;
  float best = -INFINITY;
  int bi = 0;
  // 128-bit loads, all issued before the compares (V % 4 == 0 fast path; scalar tail otherwise)
  const int V4 = ((reinterpret_cast<uintptr_t>(row) & 15) == 0) ? (V >> 2) : 0;
  const float4* row4 = reinterpret_cast<const float4*>(row);
  for (int i0 = threadIdx.x; i0 < V4; i0 += 4 * blockDim.x) {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = i0 + u * blockDim.x;
      v[u] = i < V4 ? row4[i] : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = (i0 + u * blockDim.x) * 4;
      // ascending index order inside the thread + strict '>' keeps the lowest index on ties
      if (v[u].x > best) best = v[u].x, bi = i;
      if (v[u].y > best) best = v[u].y, bi = i + 1;
      if (v[u].z > best) best = v[u].z, bi = i + 2;
      if (v[u].w > best) best = v[u].w, bi = i + 3;
    }
  }
  for (int i = V4 * 4 + threadIdx.x; i < V; i += blockDim.x) {
    const float v = row[i];
    if (v > best || (v == best && i < bi)) best = v, bi = i;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) best = ov, bi = oi;
  }
  if ((threadIdx.x & 31) == 0) sv[threadIdx.x >> 5] = best, si[threadIdx.x >> 5] = bi;
  __syncthreads();
  if (threadIdx.x < 32) {
    const int nw = blockDim.x >> 5;
    best = threadIdx.x < nw ? sv[threadIdx.x] : -INFINITY;
    bi = threadIdx.x < nw ? si[threadIdx.x] : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) best = ov, bi = oi;
    }
    if (threadIdx.x == 0) next[t] = bi;
  }
}

__global__ void advance_pos_kernel(int* pos, int T, int inc) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < T) pos[i] += inc;
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error(std::string(what) + ": " + cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_version(void) { return 100; }
extern "C" int b200_timeline(void* buf, int capacity) {
  g_tl = static_cast<unsigned long long*>(buf);
  g_tl_cap = buf ? capacity : 0;
  g_tl_next = 0;
  return 0;
}
extern "C" int b200_timeline_cta(void* buf, int first_row, int n_rows, int ctas_per_row) {
  g_tlc = static_cast<unsigned long long*>(buf);
  g_tlc_first = first_row, g_tlc_rows = buf ? n_rows : 0, g_tlc_ctas = ctas_per_row;
  return 0;
}
extern "C" const char* b200_last_error(void) { return g_err.c_str(); }

extern "C" int b200_device_info(int* sm, int* major, int* minor, size_t* smem) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    set_error(std::string("device_info: ") + cudaGetErrorString(e));
    return (int)e;
  }
  int v = 0;
  if (sm) *sm = sm_count();
  if (major) {
    cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, dev);
    *major = v;
  }
  if (minor) {
    cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, dev);
    *minor = v;
  }
  if (smem) *smem = smem_optin();
  return 0;
}

extern "C" int b200_embed(const int64_t* tokens, const void* table, void* h, int T, int D, int vocab,
                          b200_stream_t stream) {
  if (!tokens || !table || !h || T < 1 || D < 8 || (D & 7) || vocab < 1) {
    set_error("embed: bad arguments");
    return B200_E_INVAL;
  }
  embed_kernel<<<T, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(tokens), static_cast<const uint4*>(table), static_cast<uint4*>(h), D / 8, vocab);
  return check_launch("embed");
}

extern "C" int b200_argmax(const float* logits, int64_t* next, int T, int V, b200_stream_t stream) {
  if (!logits || !next || T < 1 || V < 1) return B200_E_INVAL;
  argmax_kernel<<<T, 1024, 0, static_cast<cudaStream_t>(stream)>>>(logits, reinterpret_cast<long long*>(next), V);
  return check_launch("argmax");
}

extern "C" int b200_advance_pos(int32_t* pos, int T, int inc, b200_stream_t stream) {
  if (!pos || T < 1) return B200_E_INVAL;
  advance_pos_kernel<<<(T + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(pos, T, inc);
  return check_launch("advance_pos");
}


// ------------------------------------------------------------------------------------------------------------------
// Peer-mapped buffers for the fused tensor-parallel data paths (one process per GPU, one node): plain CUDA IPC.
// The caller exchanges the 64-byte handles through its process group (torch.distributed all_gather) -- plumbing only.
// ------------------------------------------------------------------------------------------------------------------
extern "C" int b200_ipc_alloc(size_t bytes, void** dev_ptr, void* handle64) {
  if (!dev_ptr || !handle64 || bytes == 0) return B200_E_INVAL;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e == cudaSuccess) e = cudaMemset(p, 0, bytes);
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    if (p) cudaFree(p);
    b200::set_error(std::string("ipc_alloc: ") + cudaGetErrorString(e));
    return (int)e;
  }
  memcpy(handle64, &h, 64);
  *dev_ptr = p;
  return 0;
}

extern "C" int b200_ipc_open(const void* handle64, void** dev_ptr) {
  if (!handle64 || !dev_ptr) return B200_E_INVAL;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    b200::set_error(std::string("ipc_open: ") + cudaGetErrorString(e));
    return (int)e;
  }
  *dev_ptr = p;
  return 0;
}

extern "C" int b200_ipc_close(void* peer_ptr) { return peer_ptr ? (int)cudaIpcCloseMemHandle(peer_ptr) : 0; }
extern "C" int b200_ipc_free(void* own_ptr) { return own_ptr ? (int)cudaFree(own_ptr) : 0; }
