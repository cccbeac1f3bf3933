"""Operator-level Python entry points: torch tensors in, one C-ABI launch each, on torch's current stream.

These mirror the operator boundary of the reference (the `quanted_layer(x)` call inside
accessory/util/quant.py:18-46 and the attention math of llama.py:170-206).  PyTorch is used only for
device memory and streams.  Every function raises if the CUDA library is missing or a launch fails.
"""
import ctypes as C

import torch

from . import _cabi
from ._cabi import (B200_EPI_F16, B200_EPI_F32, B200_EPI_QKV, B200_EPI_SILU, B200_PRO_NONE,  # noqa: F401
                    B200_PRO_RMSNORM)
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
         prefetch_const=None):
    """Fused [residual + RMSNorm] -> W-bit GEMV -> epilogue.  See include/b200_decode.h b200_gemv."""
    global launch_count
    a = gemv_args(lin, T, out=out, epilogue=epilogue, xin=xin, resid=resid, delta=delta, h_out=h_out, gamma=gamma,
                  eps=eps, qkv=qkv, moe=moe, use_pdl=use_pdl, ring_bytes=ring_bytes, prefetch=prefetch)
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
              gamma=None, eps=1e-5, qkv=None, moe=None, use_pdl=False, ring_bytes=0, prefetch=None):
    for t, n in ((xin, "xin"), (resid, "resid"), (delta, "delta"), (h_out, "h_out"), (gamma, "gamma")):
        _f16(t, n)
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


def prefill_gemm_w4(lin: PackedLinear, x, out, T):
    """out[T, N] = x[T, K] . w_hat^T on the tensor cores (wgmma) (per-channel W4, N % 128 == 0)."""
    global launch_count
    ls = lin.c_struct()
    _cabi.check(_cabi.lib().b200_prefill_gemm_w4(C.byref(ls), _p(x), _p(out), T, _stream()), "b200_prefill_gemm_w4")
    launch_count += (T + 255) // 256


def prefill_rmsnorm(resid, delta, h_out, gamma, eps, x_out, T, D):
    global launch_count
    _cabi.check(_cabi.lib().b200_prefill_rmsnorm(_p(resid), _p(delta), _p(h_out), _p(gamma), eps, _p(x_out), T, D, _stream()),
                "b200_prefill_rmsnorm")
    launch_count += 1


def prefill_rope_kv(qkv, q_out, kcache, vtcache, rope, pos, T, n_q_rows, n_kv_rows, tokens_per_seq, cache_seq):
    global launch_count
    _cabi.check(_cabi.lib().b200_prefill_rope_kv(_p(qkv), _p(q_out), _p(kcache), _p(vtcache), _p(rope), _p(pos), T, n_q_rows,
                                                 n_kv_rows, tokens_per_seq, cache_seq, _stream()), "b200_prefill_rope_kv")
    launch_count += 1


def prefill_silu_mul(gu, act, T, F):
    global launch_count
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
              use_pdl=False):
    global launch_count
    a = _cabi.MoeRouteArgs()
    a.T, a.D, a.E, a.topk = T, D, E, topk
    a.resid, a.delta, a.h_out, a.gamma = _p(resid), _p(delta), _p(h_out), _p(gamma)
    a.eps = eps
    a.gate_w, a.xn_out, a.slot_weight, a.slot_expert = _p(gate_w), _p(xn_out), _p(slot_weight), _p(slot_expert)
    a.use_pdl = int(use_pdl)
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
