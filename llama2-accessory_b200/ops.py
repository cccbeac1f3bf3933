"""Operator-level Python entry points: torch tensors in, one C-ABI launch each, on torch's current stream.

These mirror the operator boundary of the reference (the `quanted_layer(x)` call inside
accessory/util/quant.py:18-46 and the attention math of llama.py:170-206).  PyTorch is used only for
device memory and streams.  Every function raises if the CUDA library is missing or a launch fails.
"""
import ctypes as C

import torch

from . import _cabi
from ._cabi import (B200_BIAS_ACC, B200_BIAS_NONE, B200_BIAS_OUT, B200_EPI_F16, B200_EPI_F32, B200_EPI_QKV,  # noqa: F401
                    B200_EPI_SILU, B200_PRO_NONE, B200_PRO_RMSNORM)
from .quant import PackedLinear

launch_count = 0  # kernels launched through this module (bench.py reports it as gpu_launches)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else t.data_ptr()


def _f16(t, name):
    if t is not None and (t.dtype != torch.float16 or not t.is_cuda or not t.is_contiguous()):
        raise ValueError(f"{name} must be a contiguous CUDA fp16 tensor")


def gemv(lin: PackedLinear, T: int, *, out, epilogue=B200_EPI_F16, xin=None, resid=None, delta=None, h_out=None,
         gamma=None, eps=1e-5, qkv=None, moe=None, use_pdl=False, ring_bytes=0, prefetch=None, ar=None,
         prefetch_const=None, bias=None, bias_mode=B200_BIAS_NONE):
    """Fused [residual + RMSNorm] -> W-bit GEMV -> epilogue.  See include/b200_decode.h b200_gemv.
    bias: optional fp16 [N] added at bias_mode's rounding point (B200_BIAS_ACC / B200_BIAS_OUT)."""
    global launch_count
    a = gemv_args(lin, T, out=out, epilogue=epilogue, xin=xin, resid=resid, delta=delta, h_out=h_out, gamma=gamma,
                  eps=eps, qkv=qkv, moe=moe, use_pdl=use_pdl, ring_bytes=ring_bytes, prefetch=prefetch, bias=bias,
                  bias_mode=bias_mode)
    if prefetch_const is not None:  # a later launch's norm weight -> L2 now
        a.prefetch_const, a.prefetch_const_bytes = prefetch_const.data_ptr(), prefetch_const.numel() * prefetch_const.element_size()
    if ar is not None:  # fused tensor-parallel all-reduce (engine.DecodeEngine._ar): dict(world, rank, step, period, err, ...)
        a.ar_world, a.ar_rank = ar["world"], ar["rank"]
        a.ar_step, a.ar_period, a.ar_error = ar["step"], ar["period"], ar["err"]
        if "out_peers" in ar:
            a.ar_out_peers, a.ar_out_id = ar["out_peers"], ar["out_id"]
        if "in_buf" in ar:
            a.ar_in, a.ar_in_id = ar["in_buf"], ar["in_id"]
    _cabi.check(_cabi.lib().b200_gemv(C.byref(a), _stream()), "b200_gemv")
    launch_count += 1


def gemv_args(lin: PackedLinear, T: int, *, out, epilogue=B200_EPI_F16, xin=None, resid=None, delta=None, h_out=None,
              gamma=None, eps=1e-5, qkv=None, moe=None, use_pdl=False, ring_bytes=0, prefetch=None, bias=None,
              bias_mode=B200_BIAS_NONE):
    for t, n in ((xin, "xin"), (resid, "resid"), (delta, "delta"), (h_out, "h_out"), (gamma, "gamma"), (bias, "bias")):
        _f16(t, n)
    if bias is not None and bias.numel() != lin.N:
        raise ValueError(f"bias has {bias.numel()} elements, the linear has {lin.N} output rows")
    a = _cabi.GemvArgs()
    a.lin = lin.c_struct()
    a.T = T
    a.prologue = B200_PRO_RMSNORM if resid is not None else B200_PRO_NONE
    a.xin, a.resid, a.delta, a.h_out, a.gamma = _p(xin), _p(resid), _p(delta), _p(h_out), _p(gamma)
    a.eps = eps
    a.epilogue = epilogue
    a.out = _p(out)
    if qkv is not None:
        a.n_q_rows, a.n_kv_rows = qkv["n_q_rows"], qkv["n_kv_rows"]
        a.rope, a.pos = _p(qkv["rope"]), _p(qkv["pos"])
        a.tokens_per_seq = qkv["tokens_per_seq"]
        a.kcache, a.vtcache, a.cache_seq = _p(qkv["kcache"]), _p(qkv["vtcache"]), qkv["cache_seq"]
        a.prefetch_kv = int(bool(qkv.get("prefetch_kv", False)))
    if moe is not None:
        a.slot_expert, a.expert_id = _p(moe["slot_expert"]), moe["expert_id"]
        a.n_slots, a.src_div = moe["n_slots"], moe["src_div"]
    a.use_pdl = int(use_pdl)
    a.ring_bytes = ring_bytes
    if prefetch is not None:  # (tensor, nbytes[, tiles]): head of the next kernel's HBM stream -> L2
        a.prefetch_next, a.prefetch_bytes = prefetch[0].data_ptr(), int(prefetch[1])
        a.prefetch_tiles = int(prefetch[2]) if len(prefetch) > 2 else 0
    a.bias, a.bias_mode = _p(bias), bias_mode
    return a


def attn_decode(q, kcache, vtcache, pos, out, *, T, Hq, Hkv, cache_seq, tokens_per_seq, max_kv_len, ws=None,
                counters=None, n_split=0, scale=None, use_pdl=False, prefetch=None):
    global launch_count
    a = _cabi.AttnArgs()
    a.T, a.Hq, a.Hkv, a.cache_seq, a.tokens_per_seq = T, Hq, Hkv, cache_seq, tokens_per_seq
    a.n_split, a.max_kv_len = n_split, max_kv_len
    a.q, a.kcache, a.vtcache, a.pos, a.out = _p(q), _p(kcache), _p(vtcache), _p(pos), _p(out)
    a.ws, a.counters = _p(ws), _p(counters)
    a.scale = scale if scale is not None else 1.0 / (128 ** 0.5)
    a.use_pdl = int(use_pdl)
    if prefetch is not None:
        a.prefetch_next, a.prefetch_bytes = prefetch[0].data_ptr(), int(prefetch[1])
        a.prefetch_tiles = int(prefetch[2]) if len(prefetch) > 2 else 0
    _cabi.check(_cabi.lib().b200_attn_decode(C.byref(a), _stream()), "b200_attn_decode")
    launch_count += 1


def decode_step1(args, dataflow=False):
    """args: _cabi.Step1Args (engine.DecodeEngine._step1_args): one persistent kernel = one whole bs = 1 decode step.
    dataflow: the barrier-free flag-in-data version (b200_decode_step1_ll)."""
    global launch_count
    if dataflow:
        _cabi.check(_cabi.lib().b200_decode_step1_ll(C.byref(args), _stream()), "b200_decode_step1_ll")
    else:
        _cabi.check(_cabi.lib().b200_decode_step1(C.byref(args), _stream()), "b200_decode_step1")
    launch_count += 1


def _dev(t, name, dtype, numel, on):
    """The prompt kernels take raw pointers: refuse a tensor they would misread or run past.  `on` is the launch's first
    fp16 tensor, already checked by _f16 to be a CUDA tensor; every other buffer must live on its device."""
    if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or t.device != on.device:
        raise ValueError(f"{name} must be a contiguous {dtype} tensor on {on.device}")
    if t.numel() < numel:
        raise ValueError(f"{name} has {t.numel()} elements, {numel} needed")


def _anchor(t, name):
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{name} must be a contiguous CUDA fp16 tensor")
    _f16(t, name)
    return t


def prefill_gemm_w4(lin: PackedLinear, x, out, T, bias=None, bias_mode=B200_BIAS_ACC):
    """out[T, N] = x[T, K] . w_hat^T on the tensor cores (wgmma): per-channel W4 or W3, or fp16 weights (w_hat = w);
    N % 128 == 0, K % 64 == 0 (W3: K % 16 == 0).  bias: optional fp16 [N] added at bias_mode's rounding point
    (b200_prefill_gemm_w4_bias)."""
    global launch_count
    on = _anchor(x, "x")
    _dev(x, "x", torch.float16, T * lin.K, on)
    _dev(out, "out", torch.float16, T * lin.N, on)
    ls = lin.c_struct()
    if bias is None:
        _cabi.check(_cabi.lib().b200_prefill_gemm_w4(C.byref(ls), _p(x), _p(out), T, _stream()), "b200_prefill_gemm_w4")
    else:
        _dev(bias, "bias", torch.float16, lin.N, on)
        _cabi.check(_cabi.lib().b200_prefill_gemm_w4_bias(C.byref(ls), _p(x), _p(bias), bias_mode, _p(out), T, _stream()),
                    "b200_prefill_gemm_w4_bias")
    launch_count += (T + 255) // 256


def prefill_moe_gemm_w4(experts, x, out, *, slot_expert, n_slots, src_div, e_first):
    """Grouped GEMM over the local experts (list of PackedLinear, global ids e_first ..): out[s] = x[s // src_div] . w_hat^T
    for every slot s routed to one of them; other rows of out are not written."""
    global launch_count
    on = _anchor(x, "x")
    if not experts:
        raise ValueError("experts must be a non-empty list of PackedLinear")
    N, K = experts[0].N, experts[0].K
    _dev(x, "x", torch.float16, ((n_slots - 1) // max(1, src_div) + 1) * K, on)
    _dev(out, "out", torch.float16, n_slots * N, on)
    _dev(slot_expert, "slot_expert", torch.int32, n_slots, on)
    arr = (_cabi.Linear * len(experts))(*[w.c_struct() for w in experts])
    _cabi.check(_cabi.lib().b200_prefill_moe_gemm_w4(arr, e_first, len(experts), _p(slot_expert), n_slots, src_div, _p(x),
                                                     _p(out), _stream()), "b200_prefill_moe_gemm_w4")
    launch_count += 1


def prefill_rmsnorm(resid, delta, h_out, gamma, eps, x_out, T, D):
    global launch_count
    on = _anchor(resid, "resid")
    for t, n in ((resid, "resid"), (delta, "delta"), (h_out, "h_out"), (x_out, "x_out")):
        if t is not None or n in ("resid", "x_out"):
            _dev(t, n, torch.float16, T * D, on)
    _dev(gamma, "gamma", torch.float16, D, on)
    _cabi.check(_cabi.lib().b200_prefill_rmsnorm(_p(resid), _p(delta), _p(h_out), _p(gamma), eps, _p(x_out), T, D, _stream()),
                "b200_prefill_rmsnorm")
    launch_count += 1


def prefill_rope_kv(qkv, q_out, kcache, vtcache, rope, pos, T, n_q_rows, n_kv_rows, tokens_per_seq, cache_seq):
    """Positions are not checked (that would need a device sync): pos[t] < cache_seq and < the rows of `rope`."""
    global launch_count
    on = _anchor(qkv, "qkv")
    _dev(qkv, "qkv", torch.float16, T * (n_q_rows + 2 * n_kv_rows), on)
    _dev(q_out, "q_out", torch.float16, T * n_q_rows, on)
    n_seq = (T - 1) // max(1, tokens_per_seq) + 1
    _dev(kcache, "kcache", torch.float16, n_seq * n_kv_rows * cache_seq, on)
    _dev(vtcache, "vtcache", torch.float16, n_seq * n_kv_rows * cache_seq, on)
    _dev(rope, "rope", torch.float32, 128, on)
    _dev(pos, "pos", torch.int32, T, on)
    _cabi.check(_cabi.lib().b200_prefill_rope_kv(_p(qkv), _p(q_out), _p(kcache), _p(vtcache), _p(rope), _p(pos), T, n_q_rows,
                                                 n_kv_rows, tokens_per_seq, cache_seq, _stream()), "b200_prefill_rope_kv")
    launch_count += 1


def prefill_silu_mul(gu, act, T, F):
    global launch_count
    on = _anchor(gu, "gu")
    _dev(gu, "gu", torch.float16, T * 2 * F, on)
    _dev(act, "act", torch.float16, T * F, on)
    _cabi.check(_cabi.lib().b200_prefill_silu_mul(_p(gu), _p(act), T, F, _stream()), "b200_prefill_silu_mul")
    launch_count += 1


def attn_split(T, Hkv, max_kv_len):
    return _cabi.lib().b200_attn_choose_split(T, Hkv, max_kv_len)


def attn_workspace_bytes(T, Hq, n_split):
    return _cabi.lib().b200_attn_workspace_bytes(T, Hq, n_split)


def embed(tokens, table, h, T, D, vocab):
    global launch_count
    _cabi.check(_cabi.lib().b200_embed(_p(tokens), _p(table), _p(h), T, D, vocab, _stream()), "b200_embed")
    launch_count += 1


def argmax(logits, out_tokens, T, V):
    global launch_count
    _cabi.check(_cabi.lib().b200_argmax(_p(logits), _p(out_tokens), T, V, _stream()), "b200_argmax")
    launch_count += 1


def advance_pos(pos, T, inc=1):
    global launch_count
    _cabi.check(_cabi.lib().b200_advance_pos(_p(pos), T, inc, _stream()), "b200_advance_pos")
    launch_count += 1


def sample_top_p(logits, uniform, out_tokens, T, V, temperature, top_p):
    """next ~ top-p(softmax(logits / temperature)) with the caller's uniforms (meta.py:438-440, 550-565)."""
    global launch_count
    if logits.dtype != torch.float32 or uniform.dtype != torch.float32 or out_tokens.dtype != torch.int64:
        raise ValueError("sample_top_p: logits/uniform must be fp32 and out_tokens int64")
    _cabi.check(_cabi.lib().b200_sample_top_p(_p(logits), _p(uniform), _p(out_tokens), T, V, float(temperature),
                                              float(top_p), _stream()), "b200_sample_top_p")
    launch_count += 1


def generate_update(state, sampled):
    """state: _cabi.GenerateState (device pointers of the generate loop); one step of meta.py:446-461."""
    global launch_count
    _cabi.check(_cabi.lib().b200_generate_update(C.byref(state), _p(sampled), _stream()), "b200_generate_update")
    launch_count += 1


def moe_route(*, T, D, E, topk, resid, delta, h_out, gamma, eps, gate_w, xn_out, slot_weight, slot_expert,
              use_pdl=False, scores_f32=False):
    """scores_f32: top-k and renormalisation on the fp32 softmax scores (mixtral_sparse.py:417-428) instead of the
    fp16-rounded ones (mixtral.py:272-281)."""
    global launch_count
    a = _cabi.MoeRouteArgs()
    a.T, a.D, a.E, a.topk = T, D, E, topk
    a.resid, a.delta, a.h_out, a.gamma = _p(resid), _p(delta), _p(h_out), _p(gamma)
    a.eps = eps
    a.gate_w, a.xn_out, a.slot_weight, a.slot_expert = _p(gate_w), _p(xn_out), _p(slot_weight), _p(slot_expert)
    a.use_pdl = int(use_pdl)
    a.scores_f32 = int(scores_f32)
    _cabi.check(_cabi.lib().b200_moe_route(C.byref(a), _stream()), "b200_moe_route")
    launch_count += 1


def moe_expert_ffn(w13, w2, *, T, D, F, topk, e_first, xn, slot_expert, act, y_slot, use_pdl=False):
    """w13 / w2: lists of PackedLinear for the experts living on this rank."""
    global launch_count
    n = len(w13)
    arr13 = (_cabi.Linear * n)(*[w.c_struct() for w in w13])
    arr2 = (_cabi.Linear * n)(*[w.c_struct() for w in w2])
    a = _cabi.MoeFfnArgs()
    a.w13, a.w2 = arr13, arr2
    a.T, a.D, a.F, a.topk, a.e_first, a.e_count = T, D, F, topk, e_first, n
    a.xn, a.slot_expert, a.act, a.y_slot = _p(xn), _p(slot_expert), _p(act), _p(y_slot)
    a.use_pdl = int(use_pdl)
    _cabi.check(_cabi.lib().b200_moe_expert_ffn(C.byref(a), _stream()), "b200_moe_expert_ffn")
    launch_count += 2 * n


def moe_combine(y_slot, slot_weight, slot_expert, out, *, T, D, topk, e_first, e_count):
    global launch_count
    _cabi.check(_cabi.lib().b200_moe_combine(_p(y_slot), _p(slot_weight), _p(slot_expert), e_first, e_count,
                                             _p(out), T, D, topk, _stream()), "b200_moe_combine")
    launch_count += 1
