/*
 * b200_decode.h -- C ABI of libb200decode.so: the H100 (sm_90a) quantised-decode hot path that
 * sits behind LLaMA2-Accessory's Transformer.forward_inference (accessory/model/LLM/llama.py:394-427,
 * mixtral.py:441-474) and its quantised-linear plug-in hook (accessory/util/quant.py:18-46,95-163).
 *
 * The reference is 100 % Python; it has no FFI of its own.  The binding a maintainer adds is the
 * ctypes stub in llama2-accessory_b200/_cabi.py (shown in INTEGRATION.md).  Every entry point below
 * names the reference code it replaces.
 *
 * Conventions
 *   - plain pointers and sizes only; all tensor pointers are DEVICE pointers unless marked host;
 *   - the caller owns every buffer (weights, KV cache, activations, workspaces); the library
 *     allocates nothing on the device;
 *   - enqueue-only: every launch goes to `stream`, never synchronises, and is CUDA-graph capturable;
 *   - return value: 0 = ok, <0 = invalid argument / unsupported shape (B200_E_*), >0 = cudaError_t;
 *     b200_last_error() returns a thread-local human readable message;
 *   - activations are fp16 (north star: W{2,3,4}A16); accumulation is fp32;
 *   - there is no CPU fallback anywhere.
 */
#ifndef B200_DECODE_H_
#define B200_DECODE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* b200_stream_t; /* cudaStream_t */

#define B200_E_INVAL (-1)
#define B200_E_UNSUPPORTED (-2)
#define B200_E_NOT_BUILT (-3)

int b200_version(void);
const char* b200_last_error(void);
/* sm count / compute capability of the current device (host query, no launch). */
int b200_device_info(int* sm_count, int* cc_major, int* cc_minor, size_t* smem_optin);
/* Debug/measurement aid: buf = device uint64 [capacity][8]; every subsequent b200_gemv / b200_attn_decode
 * launch takes the next row and records %globaltimer ns: [0] first CTA start (atomicMin; init to ~0ull),
 * [1] activations staged, [2] main loop done, [3] last CTA end, [4] dependency wait returned (atomicMax; init 0).
 * NULL = off. */
int b200_timeline(void* buf, int capacity);
/* Per-CTA detail for the launches that take timeline rows [first_row, first_row + n_rows): buf = device uint64
 * [n_rows][ctas_per_row][16]: columns 0..7 as in a timeline row but one row per CTA (plain stores; [5] = tiles / KV tiles
 * of the CTA), 8.. = finer stamps inside the activation staging ([8] loads returned, [9] norm barrier passed).  ctas_per_row must cover the largest grid among those launches.  NULL = off. */
int b200_timeline_cta(void* buf, int first_row, int n_rows, int ctas_per_row);
/* Measurement aid: override a tuning knob (the same names as the B200_* environment variables the kernels' launchers
 * read -- ring depth, L2-prefetch windows, attention split cap ...) for the launches enqueued from now on.  Not part of
 * the reference interface; a captured CUDA graph keeps the values it was captured with. */
int b200_tune(const char* name, int value);

/* ------------------------------------------------------------------------------------------------
 * Offline packer (HOST memory in, HOST memory out).  Replaces the weight-side half of
 * accessory/util/quant.py:116-130 (bnb.nn.Params4bit creation) with the OmniQuant-style
 * uniform-affine format (q, scale, zero) -- SURVEY.md 8c.
 *
 * bits in {2,3,4}: q is uint8 [N,K] row-major, values < 2^bits.  bits == 16: use b200_pack_f16.
 * N must be a multiple of 16.  K must be a multiple of 64 (bits 4), 128 (bits 2), 16 (bits 16);
 * bits 3 pads K to a multiple of 80 internally (5 weights per 16-bit half-word, 3.2 bit/weight).
 * The packed layout is the per-lane HMMA fragment order described in DESIGN.md ("packed formats").
 * ---------------------------------------------------------------------------------------------- */
size_t b200_packed_weight_bytes(int bits, int N, int K);
int b200_pack_weight(int bits, int N, int K, const uint8_t* q, void* out);
int b200_unpack_weight(int bits, int N, int K, const void* packed, uint8_t* q_out); /* inverse, for tests */
int b200_pack_f16(int N, int K, const uint16_t* w_fp16, void* out);
int b200_unpack_f16(int N, int K, const void* packed, uint16_t* w_out);
/* scale/zero -> interleaved half2 (s, z): per-channel [N]; grouped [N/16][K/group][16]. */
size_t b200_packed_scale_bytes(int N, int K, int group_size);
int b200_pack_scales(int N, int K, int group_size, const uint16_t* scale_fp16, const uint16_t* zero_fp16,
                     void* out);

/* A packed linear layer living in device memory. */
typedef struct {
  int bits;            /* 2, 3, 4 or 16 */
  int N;               /* output rows of this shard (multiple of 16) */
  int K;               /* input features of this shard */
  int group_size;      /* 0 = per output channel */
  const void* qweight; /* packed weights (b200_pack_weight / b200_pack_f16) */
  const void* scales;  /* packed (s,z) half2; NULL when bits == 16 */
} b200_linear_t;

/* ------------------------------------------------------------------------------------------------
 * Fused W-bit GEMV family (T <= 32 tokens).  One kernel = optional prologue + dequant-GEMV +
 * epilogue, weights streamed HBM -> shared memory by 1-D TMA bulk copies.
 *
 * prologue
 *   B200_PRO_NONE     x = xin[T,K] (fp16)
 *   B200_PRO_RMSNORM  h = resid[T,K] (+ delta[T,K] if non-NULL), written back to h_out if non-NULL;
 *                     x = fp16(h * rsqrt(mean(h^2)+eps)) * gamma        components.py:41-53
 *                     (the residual add is x + attention(...) / h + feed_forward(...), llama.py:276-288)
 * epilogue
 *   B200_EPI_F16      out fp16 [T,N]                                    F.linear, quant.py:22 / :39
 *   B200_EPI_F32      out fp32 [T,N] = float(fp16(y))                   llama.py:426-427
 *   B200_EPI_QKV      rows = [q | k | v]; RoPE (llama.py:59-77) on q,k; q -> out fp16 [T,n_q];
 *                     k, v -> the engine's KV-cache layouts (see b200_attn_decode)      llama.py:151-168
 *   B200_EPI_SILU     rows interleaved 8 x w1 / 8 x w3 per 16-row tile; out fp16 [T,N/2] =
 *                     silu(w1 x) * (w3 x)                                llama.py:252-256
 * ---------------------------------------------------------------------------------------------- */
enum { B200_PRO_NONE = 0, B200_PRO_RMSNORM = 1 };
enum { B200_EPI_F16 = 0, B200_EPI_F32 = 1, B200_EPI_QKV = 2, B200_EPI_SILU = 3 };
/* Optional fp16 bias b[N] of the linear (InternLM's Wqkv / out_proj, internlm.py:75-89), two rounding points:
 *   B200_BIAS_ACC  out = fp16(acc + b)           (fp32 add, one rounding: F.linear(x, W, b))
 *   B200_BIAS_OUT  out = fp16(fp16(acc) + b)     (fp16 add of the rounded output: RowParallelLinear's y + bias)
 * In EPI_QKV the bias is added before RoPE. */
enum { B200_BIAS_NONE = 0, B200_BIAS_ACC = 1, B200_BIAS_OUT = 2 };

typedef struct {
  b200_linear_t lin;
  int T; /* tokens in this call, 1..32 */
  /* prologue */
  int prologue;
  const void* xin;   /* fp16 [T,K]                        (PRO_NONE) */
  const void* resid; /* fp16 [T,K]                        (PRO_RMSNORM) */
  const void* delta; /* fp16 [T,K] or NULL                (PRO_RMSNORM) */
  void* h_out;       /* fp16 [T,K] or NULL: resid + delta (PRO_RMSNORM); must NOT alias resid/delta
                        (every CTA re-reads resid while CTA 0 writes h_out: ping-pong the stream) */
  const void* gamma; /* fp16 [K]                          (PRO_RMSNORM) */
  float eps;
  /* epilogue */
  int epilogue;
  void* out;
  /* EPI_QKV */
  int n_q_rows;         /* local q rows = Hq_local*128 */
  int n_kv_rows;        /* local k rows (= v rows) = Hkv_local*128 */
  const float* rope;    /* fp32 [max_pos][64][2] = (cos, sin), from precompute_freqs_cis llama.py:46-56 */
  const int32_t* pos;   /* int32 [T]: absolute position of every token */
  int tokens_per_seq;   /* cache row of token t is t / tokens_per_seq */
  void* kcache;         /* fp16 K cache, engine layout (b200_attn_decode) */
  void* vtcache;        /* fp16 V cache, engine layout (b200_attn_decode) */
  int cache_seq;        /* S */
  /* MoE slot indirection (slot_expert == NULL for dense layers).  The kernel scans
   * slot_expert[0..n_slots) and takes the slots routed to `expert_id` as its columns (at most T of
   * them, T = n_slots <= 32); x row of a slot = slot / src_div, output row = slot. */
  const int32_t* slot_expert;
  int expert_id;
  int n_slots;
  int src_div;
  /* launch */
  int use_pdl;    /* programmatic dependent launch attribute on this kernel */
  int ring_bytes; /* 0 = default; shared-memory weight ring size */
  /* Optional: once this kernel has issued all of its own weight loads, it prefetches the head of the NEXT
   * kernel's weight stream into L2, so HBM does not idle across the launch gap and the next kernel's
   * prologue.  prefetch_next = the next linear's qweight, prefetch_bytes = its packed size,
   * prefetch_tiles = its N/16: the next b200_gemv gives CTA r the contiguous tiles
   * [tiles*r/grid, tiles*(r+1)/grid), and the first B200_PF_KB (env, default 96) KB of every such region
   * are prefetched.  prefetch_tiles = 0: the first prefetch_bytes of the stream, as one range.  NULL/0 = off. */
  const void* prefetch_next;
  int prefetch_bytes;
  int prefetch_tiles;
  /* EPI_QKV only: the producer also pulls cache rows [0, pos] of every kv head (what the b200_attn_decode launch that
   * follows will stream) into L2 once its own weight stream is issued. */
  int prefetch_kv;
  /* Tensor parallelism at T == 1 without a collective kernel (replaces reduce_from_model_parallel_region, quant.py:41, around
   * a RowParallelLinear): the partial sums travel as 8-byte {half2, sequence number} units (the LL protocol of low-latency
   * collectives) through peer-mapped buffers of ar_world * N/2 units per rank.
   *   producer launch (wo / w2, EPI_F16): ar_out_peers = HOST array [ar_world] of the ranks' buffers; this rank's rows go to
   *     slot ar_rank of EVERY buffer (`out` is not written), for every codec and both kernels (the integer-path gemv1 and
   *     the generic HMMA kernel); not with MoE slot indirection;
   *   consumer launch (PRO_RMSNORM): ar_in = this rank's buffer; delta = sum over slots in rank order (fp32, one rounding).
   * sequence number = *ar_step * ar_period + id + 1: ar_step is a device counter the caller advances once per decode step,
   * ids distinguish the buffers' uses inside a step (< ar_period).  ar_error (optional, device u32) is set when a poll times
   * out.  ar_world <= 1: off. */
  int ar_world, ar_rank;
  void* const* ar_out_peers;
  const void* ar_in;
  const uint32_t* ar_step;
  int ar_out_id, ar_in_id, ar_period;
  uint32_t* ar_error;
  /* Optional: small constants of a LATER launch (e.g. the norm weight of the next RMSNorm prologue, components.py:41-53),
   * prefetched into L2 by this launch before anything else, so that the launch that needs them does not wait for an HBM
   * miss queued behind its own weight stream.  NULL/0 = off.  bytes: multiple of 16. */
  const void* prefetch_const;
  int prefetch_const_bytes;
  /* Optional bias (B200_BIAS_*): fp16 [N] with bias_mode 1 or 2; NULL with bias_mode 0.  EPI_F16 and EPI_QKV only; not with
   * MoE slot indirection or ar_world > 1. */
  const void* bias;
  int bias_mode;
} b200_gemv_args_t;

int b200_gemv(const b200_gemv_args_t* a, b200_stream_t stream);
/* Algorithmic HBM bytes one b200_gemv call must move (packed weights + scales). */
size_t b200_gemv_weight_bytes(const b200_linear_t* lin);

/* ------------------------------------------------------------------------------------------------
 * Whole decode step of a dense LLaMA for ONE token (bs = 1) as ONE persistent kernel per tensor-parallel rank: replaces
 * the loop body of Transformer.forward_inference (llama.py:394-427: embedding, L TransformerBlocks llama.py:276-288, final
 * RMSNorm + output head) that b200_embed + 5L b200_gemv / b200_attn_decode launches (+ 2L all-reduces, + the logits
 * all-gather) implement otherwise.
 * Weights: THIS RANK's shards (fairscale Column/RowParallelLinear layout, tensor_parallel.py:34-38): per-channel W4 linears
 * of every block (wqkv = [wq;wk;wv] rows, w13 = w1/w3 interleaved 8+8 as for EPI_SILU), fp16 lm_head rows
 * [rank*vocab, (rank+1)*vocab); caches in the b200_attn_decode layouts, one [n_kv_heads][S][128] slab per layer.
 * Tensor parallelism: every rank launches the same kernel; the row-parallel partial sums of wo / w2 are PUSHED into every
 * rank's communication block over NVLink by the GEMV epilogue, the grid barrier that follows counts the CTAs of all ranks,
 * and the next phase's prologue adds the partials in rank order (fp32, one rounding) -- the all-reduce of
 * reduce_from_model_parallel_region (quant.py:41) without a collective kernel.  The vocabulary-sharded logits are pushed
 * the same way.  comm: HOST array of tp_world device pointers, comm[r] = rank r's block (b200_step1_comm_bytes bytes,
 * zeroed once, peer-mapped: torch symmetric memory / cudaIpc); tp_world = 1: one ordinary device buffer.
 * Reads token[0] / pos[0]; appends K/V row pos[0] of every layer; leaves fp32 logits [vocab * tp_world] at
 * comm[tp_rank] + b200_step1_comm_logits_offset().  timeline: optional uint64 [5L+1][4] ns stamps of CTA 0, or NULL.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int n_layers, dim, n_heads, n_kv_heads, ffn /* padded to 128 */, vocab /* rows of this rank's lm_head */, cache_seq;
  float eps;
  const int64_t* token;   /* [1] */
  const void* tok_emb;    /* fp16 [vocab_total][dim], replicated */
  const int32_t* pos;     /* [1] */
  const float* rope;      /* as in b200_gemv_args_t */
  void* kcache;           /* layer 0; layer i at + i * kv_layer_stride halfs */
  void* vtcache;
  long long kv_layer_stride;
  void *h0, *h1, *q, *act; /* fp16 scratch: [dim] [dim] [n_heads*128] [ffn] */
  void* attn_ws;
  const b200_linear_t* wqkv; /* HOST arrays [n_layers] */
  const b200_linear_t* wo;
  const b200_linear_t* w13;
  const b200_linear_t* w2;
  const void* const* attn_norm; /* HOST arrays [n_layers] of device fp16 [dim] */
  const void* const* ffn_norm;
  const void* final_norm;
  b200_linear_t lm_head;  /* bits = 16 */
  void* const* comm;      /* HOST array [tp_world] */
  int tp_world, tp_rank;
  void* timeline;
  int n_split;            /* 0 = choose (b200_step1_choose_split) */
  int use_pdl;
} b200_step1_args_t;

size_t b200_step1_attn_ws_bytes(int n_heads, int n_split);
size_t b200_step1_comm_bytes(int n_layers, int dim, int vocab_local, int tp_world);
size_t b200_step1_comm_logits_offset(int n_layers, int dim, int tp_world);
int b200_step1_choose_split(int n_kv_heads);
int b200_decode_step1(const b200_step1_args_t* a, b200_stream_t stream);
/* Same step, same arguments, DATAFLOW version (csrc/mega2.cu): no grid barriers; every vector that crosses CTAs (or
 * ranks) travels as 8-byte {payload, sequence number} units that the consumer polls (the LL protocol of low-latency
 * collectives), the residual stream lives in shared memory, the K/V row of the current position is patched into the
 * last KV tile on chip.  h0 / h1 / q / act / attn_ws are not used; the communication block is larger
 * (b200_step1_ll_comm_bytes) and the fp32 logits sit at b200_step1_ll_logits_offset inside it.  A poll that never
 * succeeds sets the u32 error word at byte 8 of the block instead of hanging. */
size_t b200_step1_ll_comm_bytes(int n_layers, int dim, int n_heads, int n_kv_heads, int ffn, int vocab_local, int tp_world);
size_t b200_step1_ll_logits_offset(int n_layers, int dim, int n_heads, int n_kv_heads, int ffn, int vocab_local,
                                   int tp_world);
int b200_decode_step1_ll(const b200_step1_args_t* a, b200_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Peer-mapped device buffers for the fused tensor-parallel paths (ar_* of b200_gemv_args_t, comm of b200_step1_args_t):
 * one process per GPU on one node, CUDA IPC.  b200_ipc_alloc returns a zeroed cudaMalloc'ed buffer and its 64-byte
 * handle; the caller exchanges handles through its own process group (the reference's mp_group) and maps the peers'
 * buffers with b200_ipc_open.  (The library allocates device memory ONLY here, on explicit request.)
 * ---------------------------------------------------------------------------------------------- */
int b200_ipc_alloc(size_t bytes, void** dev_ptr, void* handle64);
int b200_ipc_open(const void* handle64, void** dev_ptr);
int b200_ipc_close(void* peer_ptr);
int b200_ipc_free(void* own_ptr);

/* ------------------------------------------------------------------------------------------------
 * Prefill (prompt) path on the Hopper tensor cores: out[T, N] = x[T, K] . w_hat[N, K]^T with
 * w_hat = fp16(fp16(q - z) * s16), the reference's fake-quantised weight reproduced bit for bit, fp32 accumulation in
 * registers (wgmma, M = 128 weight rows per CTA, N = up to 256 tokens per launch, K = 64 per pipeline stage; 80 for W3).
 * Replaces F.linear at M = prompt tokens (quant.py:18-46) for per-channel W4 (bits 4) and W3 (bits 3) linears and fp16
 * linears (bits 16, w_hat = w) with N % 128 == 0 and K % 64 == 0 (W3: K % 16 == 0).  Group scales, W2 and any other
 * width return B200_E_UNSUPPORTED.
 * The elementwise kernels are the unfused forms of the decode GEMV's prologue / epilogues for T-token chunks:
 *   b200_prefill_rmsnorm   h = resid (+ delta) -> h_out (may be NULL); x = fp16(h * rsqrt(mean h^2 + eps)) * gamma
 *   b200_prefill_rope_kv   qkv [T][n_q + 2 n_kv] -> RoPE; q -> q_out [T][n_q]; k, v -> cache rows pos[t] (llama.py:151-168)
 *   b200_prefill_silu_mul  gu [T][2F] (w1 / w3 interleaved 8 + 8 as for EPI_SILU) -> act [T][F]
 * ---------------------------------------------------------------------------------------------- */
int b200_prefill_gemm_w4(const b200_linear_t* lin, const void* x_fp16, void* out_fp16, int T, b200_stream_t stream);
/* The same GEMM with a bias b fp16 [N] added at the store (bias_mode B200_BIAS_ACC or B200_BIAS_OUT, as in b200_gemv_args_t);
 * the codecs and shapes of b200_prefill_gemm_w4. */
int b200_prefill_gemm_w4_bias(const b200_linear_t* lin, const void* x_fp16, const void* bias_fp16, int bias_mode,
                              void* out_fp16, int T, b200_stream_t stream);
/* Grouped MoE form of the same GEMM (Mixtral prompts, mixtral.py:266-294), one launch over a rank's local experts:
 * for each local expert i (global id e_first + i), for every slot s with slot_expert[s] == e_first + i:
 *   out[s][0:N] = x[s / src_div][0:K] . w_hat_i^T   (w_hat = fp16(fp16(q - z) * s16), fp32 accumulation, fp16 out)
 * experts: HOST array of e_count (1..64) per-channel W4 linears with equal N (% 128 == 0) and K (% 64 == 0).
 * Rows of slots routed elsewhere are not written.  Slots are taken in increasing slot order, 256 per CTA, so every row is
 * bit-identical to b200_prefill_gemm_w4 on that expert over the gathered rows.  slot_expert: device int32 [n_slots];
 * x fp16 [(n_slots - 1) / src_div + 1][K]; out fp16 [n_slots][N]. */
int b200_prefill_moe_gemm_w4(const b200_linear_t* experts, int e_first, int e_count, const int32_t* slot_expert,
                             int n_slots, int src_div, const void* x_fp16, void* out_fp16, b200_stream_t stream);
int b200_prefill_rmsnorm(const void* resid, const void* delta, void* h_out, const void* gamma, float eps, void* x_out, int T,
                         int D, b200_stream_t stream);
int b200_prefill_rope_kv(const void* qkv, void* q_out, void* kcache, void* vtcache, const float* rope, const int32_t* pos, int T,
                         int n_q_rows, int n_kv_rows, int tokens_per_seq, int cache_seq, b200_stream_t stream);
int b200_prefill_silu_mul(const void* gu, void* act, int T, int F, b200_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * GQA decode attention, split-KV (flash-decoding).  Replaces llama.py:170-206 (repeat_kv +
 * F.scaled_dot_product_attention / flash_attn_func) for seqlen-1 queries and, with per-token
 * kv lengths, the causal prefill of short chunks.
 *   q      fp16 [T][Hq][128]        (post-RoPE, written by EPI_QKV)
 *   KV-cache layouts ("shared-memory images": a 32-position tile is one contiguous 8 KB TMA bulk copy;
 *   S must be a multiple of 32; allocate zero-filled):
 *     kcache  fp16 [B][Hkv][S][128], the 8-element chunk index of d XOR-swizzled by row parity:
 *             element (s, d) at  s*128 + (((d>>3) ^ ((s&1)<<2)) << 3) + (d&7)
 *     vtcache fp16 [B][Hkv][S/32][128][32] (V transposed inside each 32-position block):
 *             element (s, d) at  (s>>5)*4096 + d*32 + (s&31)
 *   pos    int32 [T]: token t attends to cache positions [0, pos[t]] of row t / tokens_per_seq
 *   out    fp16 [T][Hq*128]
 *   ws     fp32 workspace, b200_attn_workspace_bytes(T, Hq, n_split); counters int32 [T*Hkv] zeroed once
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int T, Hq, Hkv, cache_seq, tokens_per_seq;
  int n_split; /* 0 = choose */
  int max_kv_len; /* upper bound on pos[t]+1 used to size the grid (<= cache_seq) */
  const void* q;
  const void* kcache;
  const void* vtcache;
  const int32_t* pos;
  void* out;
  void* ws;
  int32_t* counters;
  float scale; /* 1/sqrt(head_dim) */
  int use_pdl;
  const void* prefetch_next; /* as in b200_gemv_args_t */
  int prefetch_bytes;
  int prefetch_tiles;
} b200_attn_args_t;

int b200_attn_choose_split(int T, int Hkv, int max_kv_len);
size_t b200_attn_workspace_bytes(int T, int Hq, int n_split);
int b200_attn_decode(const b200_attn_args_t* a, b200_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Small glue kernels.
 * ---------------------------------------------------------------------------------------------- */
/* h[t][:] = table[tokens[t]][:]   (ParallelEmbedding, llama.py:376,399; table replicated per rank) */
int b200_embed(const int64_t* tokens, const void* table_fp16, void* h_fp16, int T, int D, int vocab,
               b200_stream_t stream);
/* next[t] = argmax_v logits[t][v]  (meta.py:442), int64 out so it can feed tokens directly */
int b200_argmax(const float* logits, int64_t* next, int T, int V, b200_stream_t stream);
/* pos[t] += inc (decode loop bookkeeping kept on the device so a CUDA graph can be replayed) */
int b200_advance_pos(int32_t* pos, int T, int inc, b200_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Device-side generate loop (replaces the per-token host work of MetaModel.generate, meta.py:434-461,
 * and MetaModel.sample_top_p, meta.py:550-565).
 * ---------------------------------------------------------------------------------------------- */
/* next[t] ~ top-p(softmax(logits[t] / temperature)):  a token is kept iff the probabilities strictly larger than
 * its own sum to <= top_p (the reference's "cumsum - p > top_p" mask; equal probabilities are kept or dropped
 * together), the kept set is renormalised and sampled by inverse CDF in index order with uniform[t] in [0, 1).
 * temperature and top_p must be > 0 (temperature 0 is b200_argmax, meta.py:441-442).  One CTA per row, any V >= 1.
 * While the V fp32 probabilities fit in shared memory (V <= 57856 with the H100's 227 KB opt-in) they are held there and
 * the threshold is bisected; a larger vocabulary re-reads the logits row (L2-resident) on every pass and finds the
 * threshold by a 4-pass radix descent with the masses summed in 2^-56 fixed point.  No workspace either way. */
int b200_sample_top_p(const float* logits, const float* uniform, int64_t* next, int T, int V, float temperature,
                      float top_p, b200_stream_t stream);

typedef struct {
  int bsz, total_len;
  int64_t* tokens;              /* [bsz][total_len]  prompts left-aligned, generated tokens appended (meta.py:419-423) */
  const unsigned char* text_mask; /* [bsz][total_len]  1 = position belongs to the prompt (input_text_mask) */
  const int64_t* stop_seqs;     /* [n_stop][max_stop_len] stop token sequences (eos first, meta.py:427-430) */
  const int32_t* stop_lens;     /* [n_stop] */
  int n_stop, max_stop_len;
  unsigned char* stopped;       /* [bsz] */
  int32_t* stop_pos;            /* [bsz]  end (exclusive) of the text to return per sequence */
  int64_t* step_tokens;         /* [bsz]  out: token fed to the next decode step */
  int32_t* step_pos;            /* [bsz]  out: its position (start_pos of the next step) */
  int32_t* cur_pos;             /* [1]    position being written; incremented */
  int32_t* n_stopped;           /* [1]    out: number of finished sequences (host polls this every few steps) */
} b200_generate_state_t;

/* One step of meta.py:446-461 at position *cur_pos: prompt forcing, tokens[:, cur] = next, stop bookkeeping,
 * inputs of the next decode step.  No-op once *cur_pos == total_len. */
int b200_generate_update(const b200_generate_state_t* s, const int64_t* sampled, b200_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Mixtral top-2 MoE (mixtral.py:266-294).
 *   b200_moe_route: h = resid (+delta) -> h_out; xn = rmsnorm(h)*gamma -> xn_out fp16 [T,D];
 *     logits = fp16(gate xn); scores = softmax(logits) in fp32, then by scores_f32:
 *       0  scores rounded to fp16, top-k on them, renormalised in fp16            (mixtral.py:272-281)
 *       1  top-k on the fp32 scores, fp32 sum, weight = fp16(score / sum)        (mixtral_sparse.py:417-428)
 *     (top-k ties go to the lower expert index); writes, for slot (t, j) = t*topk + j:
 *       slot_expert  int32 [T*topk]       global expert id chosen for the slot
 *       slot_weight  fp16  [T*topk]       renormalised routing weight of the slot
 *     (the expert GEMVs scan slot_expert themselves: no atomics, deterministic column order)
 *   b200_moe_combine: y[t] = sum_j fp16(slot_weight[t,j] * y_slot[t*topk+j]) over LOCAL slots only
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int T, D, E, topk;
  const void* resid;
  const void* delta;
  void* h_out;        /* must not alias resid */
  const void* gamma;
  float eps;
  const void* gate_w; /* fp16 [E][D] row-major (unpacked, replicated on every rank) */
  void* xn_out;       /* fp16 [T][D] */
  void* slot_weight;  /* fp16 [T*topk] */
  int32_t* slot_expert; /* int32 [T*topk] */
  int use_pdl;
  int scores_f32;     /* 0: fp16 score rule (mixtral), 1: fp32 score rule (mixtral_sparse); other values refused */
} b200_moe_route_args_t;
int b200_moe_route(const b200_moe_route_args_t* a, b200_stream_t stream);

typedef struct {
  /* experts of this rank, e_count entries each */
  const b200_linear_t* w13; /* HOST array: interleaved w1/w3, N = 2*F, K = D */
  const b200_linear_t* w2;  /* HOST array: N = D, K = F */
  int T, D, F, topk, e_first, e_count;
  const void* xn;              /* fp16 [T][D] */
  const int32_t* slot_expert;  /* device int32 [T*topk] */
  void* act;                   /* fp16 [T*topk][F] scratch */
  void* y_slot;                /* fp16 [T*topk][D] (rows of non-local slots are left untouched) */
  int use_pdl;
} b200_moe_ffn_args_t;
int b200_moe_expert_ffn(const b200_moe_ffn_args_t* a, b200_stream_t stream);

int b200_moe_combine(const void* y_slot, const void* slot_weight, const int32_t* slot_expert, int e_first,
                     int e_count, void* out, int T, int D, int topk, b200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200_DECODE_H_ */
