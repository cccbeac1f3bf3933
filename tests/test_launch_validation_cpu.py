"""CPU (no GPU present): every launch the engine would enqueue for the SURVEY.md section-8 configurations -- at their real
layer widths, per tensor-parallel rank -- goes through the REAL library's host-side code: argument validation
(csrc/gemv.cu build_gemv_params, attn.cu, moe.cu, prefill.cu), the integer-path / HMMA dispatch, token-group and ring sizing
against the H100's shared memory (the library assumes 132 SMs / 227 KB when no device is visible).  Each call must get as far
as its first CUDA runtime call (which fails here with "no driver": rc > 0); a NEGATIVE rc is the library rejecting the
shapes or pointers the engine handed it -- the failure a first run on hardware would hit.

One layer per model (the layers are identical), synthetic packed weights, prompt + decode steps through the public
forward_inference / the decode step.  Skipped when a GPU is visible: the launches would then really run, on host pointers.
"""
import ctypes as C

import pytest
import torch

import llama2_accessory_b200 as pkg
from llama2_accessory_b200 import _cabi, ops
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box WITHOUT a GPU (the launches must not run)")

L7 = dict(dim=4096, n_heads=32, vocab_size=32000, multiple_of=256)
L13 = dict(dim=5120, n_heads=40, vocab_size=32000, multiple_of=256)
L70 = dict(dim=8192, n_heads=64, n_kv_heads=8, vocab_size=32000, multiple_of=4096, ffn_dim_multiplier=1.3)
L70H = dict(dim=8192, n_heads=64, n_kv_heads=8, vocab_size=32000, multiple_of=256, ffn_dim_multiplier=0.65)  # width test
MIX = dict(dim=4096, n_heads=32, n_kv_heads=8, vocab_size=32000, hidden_dim=14336, rope_theta=1e6,
           moe=dict(num_experts=8, num_experts_per_tok=2))

#            name                       kind       args  bits gs  tp  bsz  prompt
CONFIGS = [
    ("C2_7B_W4_bs1",                "llama",   L7,   4,   0,  1,  1,  40),
    ("C2_7B_W4g128_bs1",            "llama",   L7,   4, 128,  1,  1,  40),
    ("7B_W3_bs1",                   "llama",   L7,   3,   0,  1,  1,  40),
    ("7B_W2g64_bs1",                "llama",   L7,   2,  64,  1,  1,  40),
    ("7B_W4_bs32",                  "llama",   L7,   4,   0,  1, 32,   3),
    ("C1_7B_fp16_prompt128",        "llama",   L7,  16,   0,  1,  1, 128),
    ("7B_W4_bs1_tp2_fused",         "llama",   L7,   4,   0,  2,  1,  40),
    ("7B_W4_bs1_tp4_fused",         "llama",   L7,   4,   0,  4,  1,  40),
    ("7B_W4_bs1_tp8_fused",         "llama",   L7,   4,   0,  8,  1,  40),
    ("C3_13B_W4_bs32_tp2",          "llama",   L13,  4,   0,  2, 32,   2),
    ("C3_width_13B_W4_bs1_tp1",     "llama",   L13,  4,   0,  1,  1, 128),
    ("C4_mixtral_W4_bs16_tp4",      "mixtral", MIX,  4,   0,  4, 16,   2),
    ("mixtral_W4_bs1_tp1",          "mixtral", MIX,  4,   0,  1,  1,  20),
    ("C5_70B_W3_bs8_tp8",           "llama",   L70,  3,   0,  8,  8,   4),
    ("70B_W3_bs1_tp8",              "llama",   L70,  3,   0,  8,  1,  40),
    ("70B_W4_bs1_tp2_fused",        "llama",   L70,  4,   0,  2,  1,  40),
    ("C5_width_70B_W3_bs4_tp1",     "llama",   L70H, 3,   0,  1,  4,  24),
]
LAUNCHES = ("b200_gemv", "b200_attn_decode", "b200_embed", "b200_prefill_gemm_w4", "b200_prefill_rmsnorm",
            "b200_prefill_rope_kv", "b200_prefill_silu_mul", "b200_moe_route", "b200_moe_expert_ffn", "b200_moe_combine",
            "b200_argmax", "b200_advance_pos")


class Validator:
    """Calls the real entry point; rc < 0 (rejected by the library's own checks) is collected, rc > 0 (CUDA runtime error on
    a box without a driver: the call passed every host-side check and reached its first runtime call) counts as accepted."""

    def __init__(self, real):
        self.real, self.rejected, self.accepted = real, [], {}

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        if name not in LAUNCHES:
            return fn

        def call(*args):
            rc = fn(*args)
            if rc < 0:
                self.rejected.append((name, rc, self.real.b200_last_error().decode()))
            else:
                self.accepted[name] = self.accepted.get(name, 0) + 1
            return 0
        return call


@pytest.fixture()
def validator(monkeypatch):
    pkg.build()
    v = Validator(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", v)
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0))
    monkeypatch.setattr(ops, "_f16", lambda t, name: None)
    monkeypatch.setattr(torch.distributed, "all_gather", lambda parts, t, group=None: [p.copy_(t) for p in parts])
    monkeypatch.setattr(torch.distributed, "all_reduce", lambda t, group=None, op=None: None)
    return v


@pytest.mark.parametrize("name,kind,margs,bits,gs,tp,bsz,prompt", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_library_accepts_every_launch_of_the_configuration(validator, name, kind, margs, bits, gs, tp, bsz, prompt):
    args = dict(margs, n_layers=1, max_seq_len=max(64, prompt + 32), max_batch_size=bsz)
    rank = tp - 1
    cfg = EngineConfig.from_model_args(kind, args, bits=bits, group_size=gs, tp_rank=rank, tp_world=tp)
    eng = DecodeEngine(cfg, "cpu")
    eng.load_random(seed=0)
    eng.use_graph = False
    if tp > 1:
        base = 0x7000_0000_0000
        eng._peer_buffers = lambda nbytes: (base + rank * 0x1000_0000, [base + r * 0x1000_0000 for r in range(tp)])
    g = torch.Generator().manual_seed(1)
    toks = torch.randint(1, args["vocab_size"], (bsz, prompt + 2), generator=g)
    logits = eng.forward_inference(toks[:, :prompt], 0)                       # the prompt (chunked or tensor-core path)
    assert logits.shape == (bsz, args["vocab_size"])
    for j in range(2):                                                        # two decode steps
        eng.forward_inference(toks[:, prompt + j:prompt + j + 1], prompt + j)
    assert not validator.rejected, validator.rejected[:4]
    assert validator.accepted.get("b200_gemv", 0) > 0 and validator.accepted.get("b200_attn_decode", 0) > 0
    if kind == "mixtral":
        assert all(validator.accepted.get(k, 0) > 0 for k in ("b200_moe_route", "b200_moe_expert_ffn", "b200_moe_combine"))
    if bits == 4 and not gs and kind == "llama" and prompt > 32 and bsz == 1:
        assert validator.accepted.get("b200_prefill_gemm_w4", 0) > 0           # prompts > 32 tokens take the wgmma GEMM
    if tp > 1 and bsz == 1 and bits == 4 and not gs and kind == "llama":
        assert eng._ar is not None                                             # the fused exchange was armed


def test_library_rejects_what_the_engine_refuses_up_front(validator):
    """The other direction: a shape beyond the kernels' limits IS rejected by the library (rc < 0), which is why
    engine.check_kernel_limits refuses it when the engine is built."""
    from llama2_accessory_b200.quant import random_packed
    pl = random_packed(4, 256, 28672, 0, "cpu", 0)        # K = 28672: the w2 of LLaMA2-70B at TP = 1
    x = torch.zeros(1, 28672, dtype=torch.float16)
    out = torch.zeros(1, 256, dtype=torch.float16)
    ops.gemv(pl, 1, xin=x, out=out)
    assert validator.rejected and "K > 16384" in validator.rejected[0][2]


@pytest.mark.parametrize("name,kind,margs,bits,tp,bsz,ctx", [
    ("C2_7B_ctx2048", "llama", L7, 4, 1, 1, 2048),
    ("bench_7B_tp8_ctx2400", "llama", L7, 4, 8, 1, 2400),
    ("C3_13B_tp2_ctx4096", "llama", L13, 4, 2, 4, 4096),
    ("C4_mixtral_tp4_ctx4096", "mixtral", MIX, 4, 4, 16, 4096),
    ("C5_70B_tp8_ctx8192", "llama", L70, 3, 8, 8, 8192),
])
def test_library_accepts_decode_steps_at_the_baseline_context_lengths(validator, name, kind, margs, bits, tp, bsz, ctx):
    """The attention launch at the BASELINE.json context lengths: split count, workspace size and cache addressing of a decode
    step whose sequences already hold ctx - 1 positions (the cache content does not matter for the host-side checks)."""
    args = dict(margs, n_layers=1, max_seq_len=ctx, max_batch_size=bsz)
    rank = tp - 1
    eng = DecodeEngine(EngineConfig.from_model_args(kind, args, bits=bits, group_size=0, tp_rank=rank, tp_world=tp), "cpu")
    eng.load_random(seed=0)
    eng.use_graph = False
    if tp > 1:
        base = 0x7000_0000_0000
        eng._peer_buffers = lambda nbytes: (base + rank * 0x1000_0000, [base + r * 0x1000_0000 for r in range(tp)])
    eng.allocate_kv_cache(bsz)
    out = eng.decode_step(torch.full((bsz,), 5, dtype=torch.int64), ctx - 1)
    assert out.shape == (bsz, args["vocab_size"]) and not validator.rejected, validator.rejected[:4]
    need = _cabi.lib().b200_attn_workspace_bytes(bsz, eng.Hq, _cabi.lib().b200_attn_choose_split(bsz, eng.Hkv, ctx))
    assert eng.ws.numel() >= need


def test_malformed_arguments_are_refused_before_any_cuda_call():
    """Error convention of the C ABI (include/b200_decode.h): a bad argument block returns a NEGATIVE code and sets
    b200_last_error() -- here every one of them must be caught by the host-side checks, i.e. before the first CUDA runtime call
    (which on this box would turn into a positive cudaError instead)."""
    from llama2_accessory_b200.quant import random_packed
    lib = _cabi.lib()
    x = torch.zeros(32, 4096, dtype=torch.float16)
    out = torch.zeros(32, 4096, dtype=torch.float32)
    pl = random_packed(4, 256, 512, 0, "cpu", 0)
    plg = random_packed(4, 256, 512, 128, "cpu", 0)

    def gemv(lin=pl, T=1, **kw):
        a = _cabi.GemvArgs()
        a.lin = lin.c_struct()
        a.T, a.xin, a.out = T, x.data_ptr(), out.data_ptr()
        for k, v in kw.items():
            if k.startswith("lin_"):
                setattr(a.lin, k[4:], v)
            else:
                setattr(a, k, v)
        rc = lib.b200_gemv(C.byref(a), None)
        return rc, lib.b200_last_error().decode()

    bad = [
        gemv(lin_bits=5), gemv(lin_N=250), gemv(lin_K=500), gemv(T=0), gemv(T=33), gemv(xin=None), gemv(out=None),
        gemv(lin_qweight=None), gemv(lin_scales=None),
        gemv(prologue=_cabi.B200_PRO_RMSNORM),                                  # RMSNorm prologue without resid / gamma
        gemv(epilogue=7), gemv(epilogue=_cabi.B200_EPI_QKV),                    # QKV epilogue without rope / cache arguments
        gemv(lin=plg, lin_bits=3),                                              # grouped scales on the 3-bit codec
        gemv(lin=plg, lin_group_size=96),                                       # group size that is not 64 / 128
        gemv(ar_world=2, ar_rank=0), gemv(ar_world=9, ar_rank=0, ar_step=x.data_ptr(), ar_period=4),
        gemv(T=2, ar_world=2, ar_rank=0, ar_step=x.data_ptr(), ar_period=4),    # fused all-reduce is bs = 1 only
    ]
    for rc, msg in bad:
        assert rc < 0 and msg, (rc, msg)

    def attn(**kw):
        a = _cabi.AttnArgs()
        a.T, a.Hq, a.Hkv, a.cache_seq, a.tokens_per_seq, a.n_split, a.max_kv_len = 1, 8, 2, 64, 1, 1, 64
        a.q = a.kcache = a.vtcache = a.pos = a.out = x.data_ptr()
        a.scale = 0.088
        for k, v in kw.items():
            setattr(a, k, v)
        rc = lib.b200_attn_decode(C.byref(a), None)
        return rc, lib.b200_last_error().decode()
    for rc, msg in (attn(q=None), attn(Hq=7), attn(Hq=34, Hkv=2), attn(cache_seq=48), attn(max_kv_len=128), attn(max_kv_len=0),
                    attn(tokens_per_seq=0), attn(n_split=4)):                    # n_split > 1 without workspace / counters
        assert rc < 0 and msg.startswith("attn:"), (rc, msg)

    ls = pl.c_struct()
    assert lib.b200_prefill_gemm_w4(C.byref(ls), x.data_ptr(), out.data_ptr(), 16, None) > 0      # 256 x 512 per-channel W4: fine
    ls.N = 192
    assert lib.b200_prefill_gemm_w4(C.byref(ls), x.data_ptr(), out.data_ptr(), 16, None) < 0      # N % 128 != 0
    lg = plg.c_struct()
    assert lib.b200_prefill_gemm_w4(C.byref(lg), x.data_ptr(), out.data_ptr(), 16, None) < 0      # grouped scales
    assert lib.b200_embed(None, x.data_ptr(), out.data_ptr(), 1, 4096, 10, None) < 0
    assert lib.b200_sample_top_p(out.data_ptr(), out.data_ptr(), x.data_ptr(), 1, 1000, 0.0, 0.9, None) < 0   # temperature 0
    assert lib.b200_sample_top_p(out.data_ptr(), out.data_ptr(), x.data_ptr(), 1, 1000, 1.0, 0.0, None) < 0   # top_p 0
    r = _cabi.MoeRouteArgs()
    r.T, r.D, r.E, r.topk = 1, 4096, 8, 9                                                          # top-k above the expert count
    r.resid = r.gamma = r.gate_w = r.xn_out = r.slot_weight = r.slot_expert = x.data_ptr()
    assert lib.b200_moe_route(C.byref(r), None) < 0
