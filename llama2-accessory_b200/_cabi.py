"""ctypes binding of libb200decode.so (include/b200_decode.h).

This is the stub a LLaMA2-Accessory maintainer would add (the reference is pure Python and has no
FFI of its own; see INTEGRATION.md).  There is NO fallback: if the shared library is missing or
fails to load, importing any compute entry point raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200decode.so")

B200_PRO_NONE, B200_PRO_RMSNORM = 0, 1
B200_EPI_F16, B200_EPI_F32, B200_EPI_QKV, B200_EPI_SILU = 0, 1, 2, 3


class Linear(C.Structure):
    _fields_ = [("bits", C.c_int), ("N", C.c_int), ("K", C.c_int), ("group_size", C.c_int),
                ("qweight", C.c_void_p), ("scales", C.c_void_p)]


class GemvArgs(C.Structure):
    _fields_ = [
        ("lin", Linear), ("T", C.c_int),
        ("prologue", C.c_int), ("xin", C.c_void_p), ("resid", C.c_void_p), ("delta", C.c_void_p),
        ("h_out", C.c_void_p), ("gamma", C.c_void_p), ("eps", C.c_float),
        ("epilogue", C.c_int), ("out", C.c_void_p),
        ("n_q_rows", C.c_int), ("n_kv_rows", C.c_int), ("rope", C.c_void_p), ("pos", C.c_void_p),
        ("tokens_per_seq", C.c_int), ("kcache", C.c_void_p), ("vtcache", C.c_void_p), ("cache_seq", C.c_int),
        ("slot_expert", C.c_void_p), ("expert_id", C.c_int), ("n_slots", C.c_int), ("src_div", C.c_int),
        ("use_pdl", C.c_int), ("ring_bytes", C.c_int),
        ("prefetch_next", C.c_void_p), ("prefetch_bytes", C.c_int), ("prefetch_tiles", C.c_int),
        ("prefetch_kv", C.c_int),
        ("ar_world", C.c_int), ("ar_rank", C.c_int), ("ar_out_peers", C.POINTER(C.c_void_p)), ("ar_in", C.c_void_p),
        ("ar_step", C.c_void_p), ("ar_out_id", C.c_int), ("ar_in_id", C.c_int), ("ar_period", C.c_int),
        ("ar_error", C.c_void_p),
        ("prefetch_const", C.c_void_p), ("prefetch_const_bytes", C.c_int),
    ]


class AttnArgs(C.Structure):
    _fields_ = [
        ("T", C.c_int), ("Hq", C.c_int), ("Hkv", C.c_int), ("cache_seq", C.c_int), ("tokens_per_seq", C.c_int),
        ("n_split", C.c_int), ("max_kv_len", C.c_int),
        ("q", C.c_void_p), ("kcache", C.c_void_p), ("vtcache", C.c_void_p), ("pos", C.c_void_p),
        ("out", C.c_void_p), ("ws", C.c_void_p), ("counters", C.c_void_p),
        ("scale", C.c_float), ("use_pdl", C.c_int),
        ("prefetch_next", C.c_void_p), ("prefetch_bytes", C.c_int), ("prefetch_tiles", C.c_int),
    ]


class MoeRouteArgs(C.Structure):
    _fields_ = [
        ("T", C.c_int), ("D", C.c_int), ("E", C.c_int), ("topk", C.c_int),
        ("resid", C.c_void_p), ("delta", C.c_void_p), ("h_out", C.c_void_p), ("gamma", C.c_void_p),
        ("eps", C.c_float), ("gate_w", C.c_void_p), ("xn_out", C.c_void_p),
        ("slot_weight", C.c_void_p), ("slot_expert", C.c_void_p), ("use_pdl", C.c_int),
    ]


class MoeFfnArgs(C.Structure):
    _fields_ = [
        ("w13", C.POINTER(Linear)), ("w2", C.POINTER(Linear)),
        ("T", C.c_int), ("D", C.c_int), ("F", C.c_int), ("topk", C.c_int), ("e_first", C.c_int), ("e_count", C.c_int),
        ("xn", C.c_void_p), ("slot_expert", C.c_void_p), ("act", C.c_void_p), ("y_slot", C.c_void_p),
        ("use_pdl", C.c_int),
    ]


class Step1Args(C.Structure):
    _fields_ = [
        ("n_layers", C.c_int), ("dim", C.c_int), ("n_heads", C.c_int), ("n_kv_heads", C.c_int), ("ffn", C.c_int),
        ("vocab", C.c_int), ("cache_seq", C.c_int), ("eps", C.c_float),
        ("token", C.c_void_p), ("tok_emb", C.c_void_p), ("pos", C.c_void_p), ("rope", C.c_void_p),
        ("kcache", C.c_void_p), ("vtcache", C.c_void_p), ("kv_layer_stride", C.c_longlong),
        ("h0", C.c_void_p), ("h1", C.c_void_p), ("q", C.c_void_p), ("act", C.c_void_p), ("attn_ws", C.c_void_p),
        ("wqkv", C.POINTER(Linear)), ("wo", C.POINTER(Linear)), ("w13", C.POINTER(Linear)), ("w2", C.POINTER(Linear)),
        ("attn_norm", C.POINTER(C.c_void_p)), ("ffn_norm", C.POINTER(C.c_void_p)), ("final_norm", C.c_void_p),
        ("lm_head", Linear), ("comm", C.POINTER(C.c_void_p)), ("tp_world", C.c_int), ("tp_rank", C.c_int),
        ("timeline", C.c_void_p), ("n_split", C.c_int), ("use_pdl", C.c_int),
    ]


# name -> (restype, argtypes): every symbol include/b200_decode.h declares
class GenerateState(C.Structure):
    _fields_ = [("bsz", C.c_int), ("total_len", C.c_int), ("tokens", C.c_void_p), ("text_mask", C.c_void_p),
                ("stop_seqs", C.c_void_p), ("stop_lens", C.c_void_p), ("n_stop", C.c_int), ("max_stop_len", C.c_int),
                ("stopped", C.c_void_p), ("stop_pos", C.c_void_p), ("step_tokens", C.c_void_p), ("step_pos", C.c_void_p),
                ("cur_pos", C.c_void_p), ("n_stopped", C.c_void_p)]


SYMBOLS = {
    "b200_version": (C.c_int, []),
    "b200_last_error": (C.c_char_p, []),
    "b200_device_info": (C.c_int, [C.POINTER(C.c_int)] * 3 + [C.POINTER(C.c_size_t)]),
    "b200_timeline": (C.c_int, [C.c_void_p, C.c_int]),
    "b200_tune": (C.c_int, [C.c_char_p, C.c_int]),
    "b200_timeline_cta": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "b200_packed_weight_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "b200_pack_weight": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b200_unpack_weight": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b200_pack_f16": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b200_unpack_f16": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b200_packed_scale_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "b200_pack_scales": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_gemv": (C.c_int, [C.POINTER(GemvArgs), C.c_void_p]),
    "b200_gemv_weight_bytes": (C.c_size_t, [C.POINTER(Linear)]),
    "b200_step1_attn_ws_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "b200_step1_comm_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200_step1_comm_logits_offset": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "b200_step1_choose_split": (C.c_int, [C.c_int]),
    "b200_decode_step1": (C.c_int, [C.POINTER(Step1Args), C.c_void_p]),
    "b200_step1_ll_comm_bytes": (C.c_size_t, [C.c_int] * 7),
    "b200_step1_ll_logits_offset": (C.c_size_t, [C.c_int] * 7),
    "b200_decode_step1_ll": (C.c_int, [C.POINTER(Step1Args), C.c_void_p]),
    "b200_ipc_alloc": (C.c_int, [C.c_size_t, C.POINTER(C.c_void_p), C.c_void_p]),
    "b200_ipc_open": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "b200_ipc_close": (C.c_int, [C.c_void_p]),
    "b200_ipc_free": (C.c_int, [C.c_void_p]),
    "b200_prefill_gemm_w4": (C.c_int, [C.POINTER(Linear), C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "b200_prefill_rmsnorm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int, C.c_int,
                                       C.c_void_p]),
    "b200_prefill_rope_kv": (C.c_int, [C.c_void_p] * 6 + [C.c_int] * 5 + [C.c_void_p]),
    "b200_prefill_silu_mul": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "b200_attn_choose_split": (C.c_int, [C.c_int, C.c_int, C.c_int]),
    "b200_attn_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "b200_attn_decode": (C.c_int, [C.POINTER(AttnArgs), C.c_void_p]),
    "b200_embed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200_argmax": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "b200_advance_pos": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "b200_sample_top_p": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p]),
    "b200_generate_update": (C.c_int, [C.POINTER(GenerateState), C.c_void_p, C.c_void_p]),
    "b200_moe_route": (C.c_int, [C.POINTER(MoeRouteArgs), C.c_void_p]),
    "b200_moe_expert_ffn": (C.c_int, [C.POINTER(MoeFfnArgs), C.c_void_p]),
    "b200_moe_combine": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                   C.c_int, C.c_int, C.c_int, C.c_void_p]),
}

_lib = None


def lib():
    """Load the shared library (once).  Raises if it was not built -- no CPU fallback exists."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). The decode engine has no CPU or PyTorch fallback.")
        _lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(_lib, name)  # AttributeError if a declared symbol is not exported
            fn.restype = res
            fn.argtypes = args
    return _lib


class B200Error(RuntimeError):
    pass


def check(rc, what=""):
    """C-ABI non-zero -> RuntimeError (the reference's surrounding code uses plain exceptions)."""
    if rc != 0:
        msg = lib().b200_last_error()
        raise B200Error(f"{what} failed (rc={rc}): {msg.decode() if msg else ''}")
