"""CPU: dry run of the engine's decode step against a RECORDING stand-in for libb200decode.so -- no kernel runs, every
C-ABI call the host code would enqueue is captured with its argument block and the data flow between the launches is checked:

  * the launch sequence of a layer is QKV GEMV -> attention -> wo GEMV -> gate/up GEMV -> down GEMV (llama.py:276-288),
    preceded by the embedding and followed by the norm + lm_head GEMV (llama.py:425-427);
  * every launch reads what the launch the reference's data flow names has written (q, attention output, activations,
    residual stream ping-pong, the delta that the next RMSNorm prologue adds), `h_out` never aliases `resid` / `delta`
    (header contract of b200_gemv), layer i works on layer i's K/V cache;
  * the L2 prefetch hint of a launch names the weight stream of the launch that actually follows;
  * tensor parallel, bs = 1 (fused all-reduce): every row-parallel producer pushes with the id its consumer polls, ids are
    unique inside a step and below the period, every rank is a push target, the step counter is advanced once per step;
    world sizes 2, 4 and 8 (4 and 8 have never run on hardware: this pins the HOST side of those runs);
  * T > 1 (no fusion): the partial sums go through all_reduce between producer and consumer.

The pure host entry points of the library (split choice, workspace size, packing) are passed through to the real library.
"""
import ctypes as C

import pytest
import torch

import llama2_accessory_b200 as pkg
from llama2_accessory_b200 import _cabi, ops
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig
from oracle import cases

ARGS = dict(dim=1024, n_layers=3, n_heads=8, n_kv_heads=8, multiple_of=256, ffn_dim_multiplier=None, norm_eps=1e-5,
            rope_theta=10000.0, vocab_size=1024, max_seq_len=64, max_batch_size=4)


def _snap(x):
    if hasattr(x, "_obj"):  # byref(struct)
        x = x._obj
    if isinstance(x, C.Structure):
        d = {}
        for name, *_ in x._fields_:
            v = getattr(x, name)
            if isinstance(v, C.Structure):
                v = _snap(v)
            elif name == "ar_out_peers":
                v = [v[i] for i in range(x.ar_world)] if v else None
            elif hasattr(v, "contents"):
                v = C.cast(v, C.c_void_p).value
            d[name] = v
        return d
    if isinstance(x, C.c_void_p):
        return x.value
    return x


class Recorder:
    """Stands in for the loaded library: launches are recorded and return 0, host-only helpers reach the real library."""
    LAUNCHES = {"b200_gemv", "b200_attn_decode", "b200_embed", "b200_argmax", "b200_advance_pos", "b200_moe_route",
                "b200_moe_expert_ffn", "b200_moe_combine", "b200_prefill_gemm_w4", "b200_prefill_rmsnorm",
                "b200_prefill_rope_kv", "b200_prefill_silu_mul", "b200_decode_step1", "b200_decode_step1_ll",
                "b200_sample_top_p", "b200_generate_update"}

    def __init__(self, real):
        self.real, self.calls, self.hooks = real, [], {}

    def __getattr__(self, name):
        if name not in self.LAUNCHES:
            return getattr(self.real, name)

        def launch(*args):
            snap = [_snap(a) for a in args]
            if name in self.hooks:  # e.g. read the host buffers a launch points at, at the moment it is enqueued
                self.hooks[name](snap)
            self.calls.append((name, snap))
            return 0
        return launch


@pytest.fixture()
def recorder(monkeypatch):
    pkg.build()
    rec = Recorder(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", rec)
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0))
    monkeypatch.setattr(ops, "_f16", lambda t, name: None)
    return rec


def _engine(tp_rank=0, tp_world=1, monkeypatch=None, gathers=None, reduces=None, max_seq_len=64):
    cfg = EngineConfig.from_model_args("llama", dict(ARGS, max_seq_len=max_seq_len), bits=4, group_size=0, tp_rank=tp_rank,
                                       tp_world=tp_world)
    eng = DecodeEngine(cfg, "cpu")
    eng.load_random(seed=1)
    eng.use_graph = False
    eng.allocate_kv_cache(2)
    if tp_world > 1:
        base = 0x7000_0000_0000
        eng._peer_buffers = lambda nbytes: (base + tp_rank * 0x100_0000, [base + r * 0x100_0000 for r in range(tp_world)])

        def fake_gather(parts, t, group=None):
            gathers.append(t.data_ptr())
            for p in parts:
                p.copy_(t)

        def fake_reduce(t, group=None, op=None):
            reduces.append(t.data_ptr())
        monkeypatch.setattr(torch.distributed, "all_gather", fake_gather)
        monkeypatch.setattr(torch.distributed, "all_reduce", fake_reduce)
    return eng


def _gemvs(calls):
    return [a[0] for n, a in calls if n == "b200_gemv"]


def _check_dataflow(eng, calls, T, fused):
    L = len(eng.layers)
    names = [n for n, _ in calls if n != "b200_advance_pos"]
    assert names == ["b200_embed"] + ["b200_gemv", "b200_attn_decode", "b200_gemv", "b200_gemv", "b200_gemv"] * L + ["b200_gemv"]
    emb = next(a for n, a in calls if n == "b200_embed")
    attn = [a[0] for n, a in calls if n == "b200_attn_decode"]
    g = _gemvs(calls)
    h = emb[2]                       # residual stream after the embedding
    delta = None                     # what the next RMSNorm prologue adds (down projection of the previous layer)
    kbase, kstride = eng.kcache.data_ptr(), eng.kcache.stride(0) * 2
    for i in range(L):
        qkv, wo, w13, w2 = g[4 * i:4 * i + 4]
        at = attn[i]
        lw = eng.layers[i]
        # --- QKV: residual (+ delta of the previous layer), RoPE + cache append of THIS layer
        assert qkv["prologue"] == _cabi.B200_PRO_RMSNORM and qkv["epilogue"] == _cabi.B200_EPI_QKV
        assert qkv["lin"]["qweight"] == lw.wqkv.qweight.data_ptr() and qkv["gamma"] == lw.attn_norm.data_ptr()
        assert qkv["resid"] == h and qkv["T"] == T
        if i == 0:
            assert qkv["delta"] is None and qkv["h_out"] is None and qkv["ar_in"] is None
        elif fused:
            assert qkv["delta"] is None or qkv["ar_world"] > 1     # the partial sums arrive through the LL buffer
            assert qkv["ar_in"] is not None and qkv["h_out"] not in (None, qkv["resid"])
            assert qkv["ar_in_id"] == g[4 * i - 1]["ar_out_id"]   # polls what the previous layer's down projection pushed
        else:
            assert qkv["delta"] == delta and qkv["h_out"] not in (None, qkv["resid"], qkv["delta"])
        if qkv["h_out"] is not None:
            h = qkv["h_out"]
        assert qkv["kcache"] == kbase + i * kstride and at["kcache"] == qkv["kcache"] and at["vtcache"] == qkv["vtcache"]
        # --- attention reads the q the QKV launch wrote, wo reads the attention output
        assert at["q"] == qkv["out"] and at["T"] == T and at["Hq"] == eng.Hq and at["Hkv"] == eng.Hkv
        assert wo["xin"] == at["out"] and wo["prologue"] == _cabi.B200_PRO_NONE and wo["epilogue"] == _cabi.B200_EPI_F16
        assert wo["lin"]["qweight"] == lw.wo.qweight.data_ptr()
        # --- gate/up: h + wo output through the RMSNorm prologue, new residual stream out of place
        assert w13["prologue"] == _cabi.B200_PRO_RMSNORM and w13["epilogue"] == _cabi.B200_EPI_SILU
        assert w13["resid"] == h and w13["gamma"] == lw.ffn_norm.data_ptr()
        assert w13["h_out"] not in (None, w13["resid"], w13["delta"])
        if fused:
            assert wo["ar_out_peers"] is not None and w13["ar_in"] is not None and wo["ar_out_id"] == w13["ar_in_id"]
        else:
            assert w13["delta"] == wo["out"] and wo["ar_world"] <= 1
        h = w13["h_out"]
        assert w2["xin"] == w13["out"] and w2["lin"]["qweight"] == lw.w2.qweight.data_ptr()
        delta = w2["out"]
        # --- L2 prefetch hints name the stream that follows
        assert at["prefetch_next"] == wo["lin"]["qweight"]
        assert wo["prefetch_next"] == w13["lin"]["qweight"] and w13["prefetch_next"] == w2["lin"]["qweight"]
        nxt = eng.layers[i + 1].wqkv if i + 1 < L else eng.lm_head
        assert w2["prefetch_next"] == nxt.qweight.data_ptr()
    head = g[-1]
    assert head["epilogue"] == _cabi.B200_EPI_F32 and head["lin"]["qweight"] == eng.lm_head.qweight.data_ptr()
    assert head["resid"] == h and head["gamma"] == eng.final_norm.data_ptr() and head["h_out"] is None
    if fused:
        assert head["ar_in"] is not None and head["ar_in_id"] == g[-2]["ar_out_id"]
    else:
        assert head["delta"] == delta
    return g


def test_single_gpu_decode_step_data_flow(recorder):
    eng = _engine()
    for T in (1, 4):
        recorder.calls.clear()
        eng._step(T, 1, eng.cache_seq)
        g = _check_dataflow(eng, recorder.calls, T, fused=False)
        assert all(a["ar_world"] <= 1 and a["ar_out_peers"] is None for a in g)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_tensor_parallel_bs1_fused_all_reduce_ids_and_targets(recorder, monkeypatch, world):
    gathers, reduces = [], []
    rank = world - 1
    eng = _engine(rank, world, monkeypatch, gathers, reduces)
    assert eng.ar_fused_supported(1)
    for step in range(2):
        recorder.calls.clear()
        gathers.clear()
        eng._step(1, 1, eng.cache_seq)
        adv = [a for n, a in recorder.calls if n == "b200_advance_pos"]
        assert len(adv) == 1 and adv[0][0] == eng._ar["step"].data_ptr() and adv[0][1:3] == [1, 1]   # one tick per step
        g = _check_dataflow(eng, recorder.calls, 1, fused=True)
        st = eng._ar
        L = len(eng.layers)
        out_ids = [a["ar_out_id"] for a in g if a["ar_out_peers"] is not None]
        assert sorted(out_ids) == list(range(2 * L)) and st["period"] > max(out_ids) + 1              # unique, below the period
        for a in g:
            if a["ar_out_peers"] is not None:
                assert a["ar_world"] == world and a["ar_rank"] == rank and len(a["ar_out_peers"]) == world
                assert len(set(a["ar_out_peers"])) == world                                           # every rank is a target
                assert a["ar_step"] == st["step"].data_ptr() and a["ar_error"] == st["step"].data_ptr() + 4
            if a["ar_in"] is not None:
                assert a["ar_in"] in (st["in_o"], st["in_f"]) and a["ar_period"] == st["period"]
        # wo pushes into the 'o' half of every rank's buffer and is polled from this rank's 'o' half; w2 likewise with 'f'
        one = world * ARGS["dim"] * 4
        wo0, w13_0, w2_0 = g[1], g[2], g[3]
        assert w13_0["ar_in"] == st["in_o"] and g[4]["ar_in"] == st["in_f"] == st["in_o"] + one
        assert w2_0["ar_out_peers"][rank] == st["in_f"] and wo0["ar_out_peers"][rank] == st["in_o"]
        assert not reduces and len(gathers) == 1                                                      # only the logits are gathered


def test_tensor_parallel_batched_step_uses_the_collective_between_producer_and_consumer(recorder, monkeypatch):
    gathers, reduces = [], []
    eng = _engine(1, 2, monkeypatch, gathers, reduces)
    assert not eng.ar_fused_supported(3)
    eng._step(3, 1, eng.cache_seq)
    g = _check_dataflow(eng, recorder.calls, 3, fused=False)
    L = len(eng.layers)
    assert len(reduces) == 2 * L and reduces == [p for i in range(L) for p in (g[4 * i + 1]["out"], g[4 * i + 3]["out"])]
    assert len(gathers) == 1


def test_mixtral_step_data_flow(recorder):
    """MoE block (mixtral.py:266-294): wo -> route (residual add + RMSNorm + gate softmax / top-k) -> the local experts'
    gate/up + down GEMVs on the routed slots -> weighted combine, whose output is the delta of the next layer."""
    args = dict(cases.TINY_MIXTRAL, max_seq_len=64, max_batch_size=4)
    cfg = EngineConfig.from_model_args("mixtral", args, bits=4, group_size=0)
    eng = DecodeEngine(cfg, "cpu")
    eng.load_random(seed=2)
    eng.use_graph = False
    eng.allocate_kv_cache(2)
    T, L, k = 2, len(eng.layers), cfg.experts_per_tok
    eng._step(T, 1, eng.cache_seq)
    names = [n for n, _ in recorder.calls]
    assert names == ["b200_embed"] + ["b200_gemv", "b200_attn_decode", "b200_gemv", "b200_moe_route", "b200_moe_expert_ffn",
                                      "b200_moe_combine"] * L + ["b200_gemv"]
    calls = recorder.calls
    h, delta = calls[0][1][2], None
    for i in range(L):
        qkv, at, wo, route, ffn, comb = (calls[1 + 6 * i + j][1] for j in range(6))
        qkv, at, wo, route, ffn = qkv[0], at[0], wo[0], route[0], ffn[0]
        assert qkv["resid"] == h and qkv["delta"] == delta and at["q"] == qkv["out"] and wo["xin"] == at["out"]
        if qkv["h_out"] is not None:
            h = qkv["h_out"]
        assert route["resid"] == h and route["delta"] == wo["out"] and route["h_out"] not in (None, h, wo["out"])
        assert (route["T"], route["E"], route["topk"]) == (T, cfg.num_experts, k)
        h = route["h_out"]
        assert ffn["xn"] == route["xn_out"] and ffn["slot_expert"] == route["slot_expert"]
        assert (ffn["T"], ffn["topk"], ffn["e_first"], ffn["e_count"]) == (T, k, 0, cfg.num_experts)
        y_slot, slot_w, slot_e, e_first, e_count, out = comb[:6]
        assert (y_slot, slot_w, slot_e) == (ffn["y_slot"], route["slot_weight"], route["slot_expert"])
        assert (e_first, e_count) == (0, cfg.num_experts) and comb[6:9] == [T, cfg.dim, k]
        delta = out
    head = calls[-1][1][0]
    assert head["resid"] == h and head["delta"] == delta and head["epilogue"] == _cabi.B200_EPI_F32


def _ints(ptr, n, ctype):
    return list((ctype * n).from_address(ptr))


def _prompt_trace(recorder, eng, tokens, start_pos=0):
    """forward_inference on a prompt with, for every embedding launch, a snapshot of the token buffer it reads (CPU
    tensors: the pointers of the recorded calls are host addresses)."""
    snaps = []
    recorder.hooks["b200_embed"] = lambda a: snaps.append(dict(T=a[3], tokens=_ints(a[0], a[3], C.c_int64)))
    try:
        eng.forward_inference(tokens, start_pos)
    finally:
        recorder.hooks.clear()
    return snaps


@pytest.mark.parametrize("bsz,seqlen", [(3, 20), (1, 31), (5, 7)])
def test_chunked_prompt_covers_every_position_once_in_order(recorder, bsz, seqlen):
    """Prompts of <= 32 tokens per launch (llama.py:394-427 at seqlen > 1): every (sequence, position) is embedded exactly
    once, positions of a sequence in increasing order across the launches, tokens_per_seq = the chunk length, and the QKV /
    attention launches of a chunk address the cache rows of the sequences it holds."""
    eng = _engine()
    eng.allocate_kv_cache(bsz)
    g = torch.Generator().manual_seed(bsz * 100 + seqlen)
    toks = torch.randint(1, ARGS["vocab_size"], (bsz, seqlen), generator=g)
    pos_reads = []
    orig = ops.gemv

    def spy(lin, T, **kw):
        if kw.get("qkv") is not None and lin is eng.layers[0].wqkv:
            pos_reads.append((T, kw["qkv"]["tokens_per_seq"], kw["qkv"]["pos"][:T].tolist(), kw["qkv"]["kcache"].data_ptr()))
        return orig(lin, T, **kw)
    ops.gemv = spy
    try:
        snaps = _prompt_trace(recorder, eng, toks)
    finally:
        ops.gemv = orig
    assert len(snaps) == len(pos_reads)
    seen = {}
    row_bytes = eng.kcache.stride(1) * 2
    for sn, (T, tps, pos, kptr) in zip(snaps, pos_reads):
        assert sn["T"] == T <= 32 and T % tps == 0
        row0 = (kptr - eng.kcache[0].data_ptr()) // row_bytes
        for t in range(T):
            b, p = row0 + t // tps, pos[t]
            assert (b, p) not in seen and (p == 0 or (b, p - 1) in seen)        # once, in order
            seen[(b, p)] = sn["tokens"][t]
    assert len(seen) == bsz * seqlen
    assert all(seen[(b, p)] == int(toks[b, p]) for b in range(bsz) for p in range(seqlen))
    # logits of the last position only: one lm_head launch per group of sequences
    heads = [a for a in _gemvs(recorder.calls) if a["epilogue"] == _cabi.B200_EPI_F32]
    assert sum(a["T"] for a in heads) == bsz


def test_tensor_core_prompt_path_chunks_and_attention_sub_launches(recorder):
    """Prompts > 32 tokens of a per-channel W4 model: one sequence at a time in chunks of <= 256 positions through the
    wgmma GEMM; per chunk and layer: rmsnorm, QKV GEMM, RoPE + cache write, ceil(chunk / 32) attention launches that walk
    the chunk's queries in order, wo GEMM, rmsnorm, gate/up GEMM, SiLU*mul, down GEMM; logits from the last position only."""
    eng = _engine(max_seq_len=320)
    assert eng.prefill_tc_supported()
    bsz, seqlen = 2, 300
    eng.allocate_kv_cache(bsz)
    g = torch.Generator().manual_seed(9)
    toks = torch.randint(1, ARGS["vocab_size"], (bsz, seqlen), generator=g)
    ropes = []
    recorder.hooks["b200_prefill_rope_kv"] = lambda a: ropes.append(dict(T=a[6], pos=_ints(a[5], a[6], C.c_int32), kcache=a[2],
                                                                       tps=a[9]))
    # the position buffer is reused by later chunks: read it when the attention launch is enqueued
    orig_attn = ops.attn_decode

    def spy_attn(q, kc, vt, pos, out, **kw):
        spy_attn.pos.append(pos[:kw["T"]].tolist())
        return orig_attn(q, kc, vt, pos, out, **kw)
    spy_attn.pos = []
    ops.attn_decode = spy_attn
    try:
        snaps = _prompt_trace(recorder, eng, toks)
    finally:
        ops.attn_decode = orig_attn
    L = len(eng.layers)
    chunks = [(b, off, min(256, seqlen - off)) for b in range(bsz) for off in range(0, seqlen, 256)]
    assert [s_["T"] for s_ in snaps] == [c[2] for c in chunks]
    for s_, (b, off, ci) in zip(snaps, chunks):
        assert s_["tokens"] == toks[b, off:off + ci].tolist()
    assert len(ropes) == len(chunks) * L
    row_bytes = eng.kcache.stride(1) * 2
    for j, (b, off, ci) in enumerate(chunks):
        for i in range(L):
            r = ropes[j * L + i]
            assert r["T"] == ci == r["tps"] and r["pos"] == list(range(off, off + ci))
            assert r["kcache"] == eng.kcache[i].data_ptr() + b * row_bytes                 # layer i, cache row of sequence b
    names = [n for n, _ in recorder.calls]
    per_layer = lambda ci: (["b200_prefill_rmsnorm", "b200_prefill_gemm_w4", "b200_prefill_rope_kv"]  # noqa: E731
                            + ["b200_attn_decode"] * -(-ci // 32)
                            + ["b200_prefill_gemm_w4", "b200_prefill_rmsnorm", "b200_prefill_gemm_w4", "b200_prefill_silu_mul",
                               "b200_prefill_gemm_w4"])
    want = []
    for b, off, ci in chunks:
        want += ["b200_embed"] + per_layer(ci) * L
        if off + ci >= seqlen:
            want += ["b200_gemv"]                                                           # lm_head on the last position
    assert names == want
    # the attention sub-launches of a chunk take its queries 32 at a time, in order, all against the sequence's cache row
    attn = [a[0] for n, a in recorder.calls if n == "b200_attn_decode"]
    k = 0
    for b, off, ci in chunks:
        for i in range(L):
            q0 = None
            for t0 in range(0, ci, 32):
                a = attn[k]
                k += 1
                tn = min(32, ci - t0)
                assert a["T"] == tn and a["tokens_per_seq"] == tn and a["kcache"] == eng.kcache[i].data_ptr() + b * row_bytes
                q0 = a["q"] if q0 is None else q0
                assert a["q"] == q0 + t0 * eng.Hq * 128 * 2 and spy_attn.pos[k - 1] == list(range(off + t0, off + t0 + tn))
    heads = [a[0] for n, a in recorder.calls if n == "b200_gemv"]
    assert len(heads) == bsz and all(h["T"] == 1 and h["epilogue"] == _cabi.B200_EPI_F32 for h in heads)
