"""CPU: the Mixtral prompt path on the tensor cores (engine._prefill_chunk_tc, csrc/prefill.cu b200_prefill_moe_gemm_w4),
checked without a GPU.

  * Launch trace: a recording stand-in for libb200decode.so captures every launch of a 300-token prompt at bs = 2 (TP = 1,
    and rank 1 of TP = 2) together with the collectives.  Per chunk and layer the order is rmsnorm, QKV GEMM, RoPE + cache
    write, the attention sub-launches, wo GEMM, route, grouped gate/up GEMM, SiLU*mul over the slot rows, grouped down
    GEMM, combine (mixtral.py:266-294); the data flows route -> gate/up (src_div = top-k) -> act -> down (src_div = 1)
    -> combine, the residual stream ping-pongs through the router, every grouped launch names this rank's experts, and at
    TP = 2 an all-reduce follows wo and combine.  Prompts of <= 32 tokens keep the GEMV chunks.
  * Launch validation: the same prompt at the C4 (Mixtral-8x7B) widths through the REAL library's host-side checks; a
    negative rc is a rejection, rc > 0 is the first CUDA call failing on a box without a driver, i.e. accepted.  Malformed
    arguments to the grouped GEMM are refused with rc < 0 and a message.
"""
import ctypes as C

import pytest
import torch

import llama2_accessory_b200 as pkg
from llama2_accessory_b200 import _cabi, ops
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig
from oracle import cases

LAUNCHES = {"b200_gemv", "b200_attn_decode", "b200_embed", "b200_argmax", "b200_advance_pos", "b200_moe_route",
            "b200_moe_expert_ffn", "b200_moe_combine", "b200_prefill_gemm_w4", "b200_prefill_moe_gemm_w4",
            "b200_prefill_rmsnorm", "b200_prefill_rope_kv", "b200_prefill_silu_mul"}
MIX = dict(dim=4096, n_heads=32, n_kv_heads=8, vocab_size=32000, hidden_dim=14336, rope_theta=1e6,
           moe=dict(num_experts=8, num_experts_per_tok=2))


def _snap(x):
    if hasattr(x, "_obj"):  # byref(struct)
        x = x._obj
    if isinstance(x, C.Structure):
        return {name: (_snap(getattr(x, name)) if isinstance(getattr(x, name), C.Structure) else getattr(x, name))
                for name, *_ in x._fields_}
    if isinstance(x, C.Array):  # the host array of expert linears
        return [_snap(e) for e in x]
    if isinstance(x, C.c_void_p):
        return x.value
    return x


class Recorder:
    """Stands in for the loaded library: launches are recorded and return 0, host-only helpers reach the real library."""

    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        if name not in LAUNCHES:
            return getattr(self.real, name)

        def launch(*args):
            self.calls.append((name, [_snap(a) for a in args]))
            return 0
        return launch


@pytest.fixture()
def recorder(monkeypatch):
    pkg.build()
    rec = Recorder(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", rec)
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0))
    monkeypatch.setattr(ops, "_f16", lambda t, name: None)
    monkeypatch.setattr(torch.distributed, "all_reduce", lambda t, group=None, op=None: rec.calls.append(("all_reduce", t.data_ptr())))
    monkeypatch.setattr(torch.distributed, "all_gather", lambda parts, t, group=None: [p.copy_(t) for p in parts])
    return rec


def _mixtral(tp_rank=0, tp_world=1, max_seq_len=320):
    cfg = EngineConfig.from_model_args("mixtral", dict(cases.TINY_MIXTRAL, max_seq_len=max_seq_len), bits=4, group_size=0,
                                       tp_rank=tp_rank, tp_world=tp_world)
    eng = DecodeEngine(cfg, "cpu")
    eng.load_random(seed=3)
    eng.use_graph = False
    return eng


@pytest.mark.parametrize("tp_rank,tp_world", [(0, 1), (1, 2)])
def test_mixtral_tensor_core_prompt_launch_order_and_data_flow(recorder, tp_rank, tp_world):
    eng = _mixtral(tp_rank, tp_world)
    assert eng.prefill_tc_supported()
    c, L, k = eng.cfg, len(eng.layers), eng.cfg.experts_per_tok
    bsz, seqlen = 2, 300
    toks = torch.randint(1, c.vocab_size, (bsz, seqlen), generator=torch.Generator().manual_seed(4))
    eng.forward_inference(toks, 0)
    calls = recorder.calls
    names = [n for n, _ in calls]
    assert "b200_moe_expert_ffn" not in names and "b200_gemv" in names

    ar = ["all_reduce"] if tp_world > 1 else []
    chunks = [(b, off, min(256, seqlen - off)) for b in range(bsz) for off in range(0, seqlen, 256)]

    def per_layer(ci):
        return (["b200_prefill_rmsnorm", "b200_prefill_gemm_w4", "b200_prefill_rope_kv"] + ["b200_attn_decode"] * -(-ci // 32)
                + ["b200_prefill_gemm_w4"] + ar + ["b200_moe_route", "b200_prefill_moe_gemm_w4", "b200_prefill_silu_mul",
                                                   "b200_prefill_moe_gemm_w4", "b200_moe_combine"] + ar)
    want = []
    for b, off, ci in chunks:
        want += ["b200_embed"] + per_layer(ci) * L
        if off + ci >= seqlen:
            want += ["b200_gemv"]  # lm_head on the last position
    assert names == want

    # data flow, chunk by chunk
    i = 0
    for b, off, ci in chunks:
        assert calls[i][0] == "b200_embed"
        h, delta = calls[i][1][2], None
        i += 1
        for li, lw in enumerate(eng.layers):
            seg = calls[i:i + len(per_layer(ci))]
            i += len(seg)
            norm, qkv = seg[0][1], seg[1][1]
            assert norm[0] == h and norm[1] == delta
            if delta is not None:
                h = norm[2]
            wo = seg[3 + -(-ci // 32)][1]
            j = 4 + -(-ci // 32)
            if ar:
                assert seg[j][1] == wo[2]                                  # all-reduce of the wo partial sums
                j += 1
            route, g13, silu, g2, comb = (seg[j + m][1] for m in range(5))
            route = route[0]
            assert route["T"] == ci and route["topk"] == k and route["E"] == c.num_experts
            assert route["resid"] == h and route["delta"] == wo[2] and route["h_out"] not in (None, h, wo[2])
            assert route["gamma"] == lw.ffn_norm.data_ptr() and route["gate_w"] == lw.gate.data_ptr()
            h = route["h_out"]                                              # the residual stream ping-pongs
            ns = ci * k
            # b200_prefill_moe_gemm_w4(experts, e_first, e_count, slot_expert, n_slots, src_div, x, out, stream)
            for g, ws, src_div in ((g13, lw.e_w13, k), (g2, lw.e_w2, 1)):
                assert [e["qweight"] for e in g[0]] == [w.qweight.data_ptr() for w in ws]
                assert g[1:6] == [eng.e_first, eng.E_loc, route["slot_expert"], ns, src_div]
            assert eng.e_first == tp_rank * eng.E_loc
            assert g13[6] == route["xn_out"]                                # gate/up reads the normed tokens
            assert silu[0] == g13[7] and silu[2:4] == [ns, lw.e_w2[0].K]    # SiLU*mul over every slot row
            assert g2[6] == silu[1]                                         # down reads the activations
            y_slot, slot_w, slot_e, e_first, e_count, out = comb[:6]
            assert (y_slot, slot_w, slot_e) == (g2[7], route["slot_weight"], route["slot_expert"])
            assert (e_first, e_count) == (eng.e_first, eng.E_loc) and comb[6:9] == [ci, c.dim, k]
            if ar:
                assert seg[j + 5][1] == out                                 # all-reduce of the combined expert outputs
            delta = out
        if off + ci >= seqlen:
            head = calls[i][1][0]
            assert head["epilogue"] == _cabi.B200_EPI_F32 and head["T"] == 1
            i += 1
    assert i == len(calls)


def test_short_mixtral_prompt_keeps_the_gemv_chunks(recorder):
    """<= 32 tokens: chunks of t_max = 32 / top-k tokens through the decode GEMVs and the per-expert GEMV driver."""
    eng = _mixtral()
    toks = torch.randint(1, eng.cfg.vocab_size, (1, 20), generator=torch.Generator().manual_seed(5))
    eng.forward_inference(toks, 0)
    names = [n for n, _ in recorder.calls]
    assert not any(n.startswith("b200_prefill") for n in names)
    assert names.count("b200_embed") == 2 and names.count("b200_moe_expert_ffn") == 2 * len(eng.layers)


# ------------------------------------------------------------------------------------------------ launch validation ----
class Validator:
    """Calls the real entry point; rc < 0 (rejected by the library's own checks) is collected, rc > 0 counts as accepted."""

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


no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box WITHOUT a GPU (the launches must not run)")


@no_gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("tp", [1, 4])
def test_library_accepts_every_launch_of_a_c4_prompt(monkeypatch, tp):
    pkg.build()
    v = Validator(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", v)
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0))
    monkeypatch.setattr(ops, "_f16", lambda t, name: None)
    monkeypatch.setattr(torch.distributed, "all_gather", lambda parts, t, group=None: [p.copy_(t) for p in parts])
    monkeypatch.setattr(torch.distributed, "all_reduce", lambda t, group=None, op=None: None)
    prompt = 300
    rank = tp - 1
    cfg = EngineConfig.from_model_args("mixtral", dict(MIX, n_layers=1, max_seq_len=prompt + 32, max_batch_size=1), bits=4,
                                       group_size=0, tp_rank=rank, tp_world=tp)
    eng = DecodeEngine(cfg, "cpu")
    eng.load_random(seed=0)
    eng.use_graph = False
    assert eng.prefill_tc_supported()
    toks = torch.randint(1, MIX["vocab_size"], (1, prompt + 1), generator=torch.Generator().manual_seed(1))
    assert eng.forward_inference(toks[:, :prompt], 0).shape == (1, MIX["vocab_size"])
    eng.forward_inference(toks[:, prompt:], prompt)
    assert not v.rejected, v.rejected[:4]
    assert v.accepted.get("b200_prefill_moe_gemm_w4", 0) == 2 * 2          # two chunks x (gate/up, down)
    assert v.accepted.get("b200_moe_expert_ffn", 0) == 1                    # the decode step keeps the GEMV experts


@no_gpu
def test_malformed_grouped_gemm_arguments_are_refused_before_any_cuda_call():
    from llama2_accessory_b200.quant import random_packed
    pkg.build()
    lib = _cabi.lib()
    x = torch.zeros(64, 512, dtype=torch.float16)
    out = torch.zeros(64, 256, dtype=torch.float16)
    se = torch.zeros(64, dtype=torch.int32)
    pl = [random_packed(4, 256, 512, 0, "cpu", i) for i in range(3)]
    plg = random_packed(4, 256, 512, 128, "cpu", 0)
    pl3 = random_packed(3, 256, 512, 0, "cpu", 0)

    def call(experts=pl, e_first=0, e_count=None, slot_expert=se, n_slots=64, src_div=2, x_=x, out_=out, edit=None):
        arr = (_cabi.Linear * max(1, len(experts)))(*[w.c_struct() for w in experts])
        if edit:
            edit(arr)
        rc = lib.b200_prefill_moe_gemm_w4(arr if experts else None, e_first, len(experts) if e_count is None else e_count,
                                          None if slot_expert is None else slot_expert.data_ptr(), n_slots, src_div,
                                          None if x_ is None else x_.data_ptr(), None if out_ is None else out_.data_ptr(),
                                          None)
        return rc, lib.b200_last_error().decode()

    rc, _ = call()
    assert rc > 0                                                            # valid: reaches the CUDA runtime
    bad = [call(experts=[]), call(slot_expert=None), call(x_=None), call(out_=None), call(e_count=0), call(n_slots=0),
           call(src_div=0), call(e_count=-1), call(n_slots=-5),
           call(experts=[pl[0], plg]),                                        # grouped scales
           call(experts=[pl3, pl[0]]),                                        # 3-bit expert
           call(experts=[pl[0], random_packed(4, 384, 512, 0, "cpu", 1)]),    # unequal N
           call(experts=[pl[0], random_packed(4, 256, 1024, 0, "cpu", 1)]),   # unequal K
           call(edit=lambda a: [setattr(a[i], "N", 192) for i in range(3)]),  # N % 128 != 0
           call(edit=lambda a: [setattr(a[i], "K", 480) for i in range(3)]),  # K % 64 != 0
           call(edit=lambda a: setattr(a[1], "qweight", None)),
           call(edit=lambda a: setattr(a[2], "scales", None)),
           call(experts=[pl[0]] * 65)]                                        # beyond the router's 64 experts
    for rc, msg in bad:
        assert rc < 0 and msg.startswith("prefill_moe_gemm_w4"), (rc, msg)
