"""GPU: the `internlm` and `mixtral_sparse` serving paths audited launch by launch against float64
(test_engine_launch_audit_gpu.Audit: every launch checked against float64 of its own inputs, on the engine's own buffers,
with no stray writes), and the InternLM bias epilogue at the edges the engine cannot reach cheaply.

  * InternLM engine: the three tiny cases (fp16, W4, W4 g128) at bs 1 (a 5-token prompt, 3 decode steps: gemv1 T = 1
    launches with the engine's PDL and prefetch arguments, wo's BIAS_OUT beside prefetch_const) and bs 2 (a prompt, a
    continuation, 2 decode steps); tensor-core prompts for fp16 and per-channel W4 (300 tokens: 256 + 44, a GEMV
    continuation, a tensor-core continuation across the 384 boundary, decode); forward_full; one layer at InternLM-7B width
    (D 4096, 32 heads, F 11008) and at InternLM-20B width (D 5120, 40 heads, F 13824), random weights and biases in +-0.5
    (engine.load_random).
  * The bias epilogue kernels: every codec at the 7B and 20B Wqkv widths, gemv1 (T = 1) and the HMMA kernel (T = 2, 8, 9,
    32), with the RMSNorm prologue, EPI_QKV and B200_BIAS_ACC, at positions 0, 31, 32, 2047 and cache_seq - 1 into
    NaN-sentinel caches and outputs.  y (the F16 launch with the same bias) is held to the bound of float64 x . w_hat + b
    (Audit._y_bound), q / K / V follow from y bit for bit, and nothing else changes.  The same with more than 16 tiles per
    CTA (Hq = 2 SMs + 8: bias and RoPE factors read from global memory tile by tile), and BIAS_ACC with b = 0 bit-identical
    to the bias-free launch.
  * mixtral_sparse engine (the fp32 router rule, every expert sliced): the tiny W4 and fp16 cases through GEMV chunks and a
    batch above t_max, W4 through tensor-core prompts of 40 and 300 tokens with continuations, tied gate rows (every route
    an exact tie, to the lower index under the fp32 rule too), one layer at Mixtral-8x7B width at TP 1 (F 14336) and one
    at hidden_dim 3584 (the launches of one TP-4 rank, without the collective).
  * The audit refuses what it does not check: a bias on a launch of a model without one, and arguments no checker takes.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import engine as engine_mod, kvlayout, ops  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig, rope_table  # noqa: E402
from oracle import internlm, omniquant, sparse, weights  # noqa: E402
from oracle.numerics import SENT, gemv_tol, nan16, qkv_from_y, x_candidates  # noqa: E402
from test_engine_launch_audit_gpu import (BIAS_ADD_REL, MIXTRAL_WIDTH, Audit, _calls, _eager, _paths,  # noqa: E402
                                          _tc_paths, audit_schedule)
from test_gemv_batched_moe_gpu import _linear  # noqa: E402

DEV = "cuda"
EPS = 1e-5


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _bits16(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------ InternLM engine ---------
def _internlm_engine(name, max_seq_len=64):
    args, sd, _, recs, _ = internlm.build_case(name)
    _, bits, gs, _, _, _ = internlm.CASES[name]
    cfg = EngineConfig.from_model_args("internlm", dict(args, max_seq_len=max_seq_len), bits=bits or 16, group_size=gs)
    eng = DecodeEngine(cfg, DEV).load_master_state_dict(sd, quant_records=recs if bits else None)
    assert all(lw.bqkv is not None and lw.bo is not None for lw in eng.layers)
    return eng


def _biased(a, tc=False):
    """Every Wqkv launch carried B200_BIAS_ACC and every wo launch B200_BIAS_OUT (the checkers demand the roles)."""
    kinds = set(a.stats)
    assert "gemv QKV BIAS_ACC" in kinds and "gemv QKV" not in kinds, sorted(kinds)
    assert "gemv F16 (wo) BIAS_OUT" in kinds and "gemv F16 (wo)" not in kinds, sorted(kinds)
    if tc:
        assert any(k.endswith("wqkv BIAS_ACC)") for k in kinds) and any(k.endswith("wo BIAS_OUT)") for k in kinds), kinds


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", list(internlm.CASES))
def test_tiny_internlm_gemv_schedules(name):
    """bs 1: a 5-token prompt and 3 decode steps (T = 1: gemv1 for the quantised codecs, with the engine's use_pdl,
    prefetch and prefetch_const); bs 2: a 5-token prompt, a 7-token continuation, 2 decode steps."""
    a = audit_schedule(_internlm_engine(name), 1, _calls(5, 0, 3), f"{name} bs 1")
    assert _paths(a) == [("gemv", 5)] + [("gemv", 1)] * 3
    _biased(a)
    a = audit_schedule(_internlm_engine(name), 2, _calls(5, 7, 2), f"{name} bs 2")
    _biased(a)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", ["internlm_fp16", "internlm_w4"])
def test_tiny_internlm_tensor_core_prompts(name):
    """Batch 2: a 300-token prompt (256 + 44 per sequence), a 20-token GEMV continuation (16 + 4 per sequence), a 70-token
    tensor-core continuation at positions 320-389 (across the 384 boundary: max_kv_len 512), 2 decode steps."""
    eng = _internlm_engine(name, max_seq_len=512)
    a = audit_schedule(eng, 2, [(0, 300), (300, 20), (320, 70), (390, 1), (391, 1)], f"{name} bs 2 tc", tc=True)
    _tc_paths(a, [("tc", 256), ("tc", 44)] * 2 + [("gemv", 32), ("gemv", 8)] + [("tc", 70)] * 2 + [("gemv", 2)] * 2)
    assert [e["kv"] for e in a.done if e.get("tc") and e["T"] == 70] == [512] * 2
    _biased(a, tc=True)


@pytest.mark.timeout(600)
def test_tiny_internlm_w4_forward_full():
    """DecodeEngine.forward_full over batch 2 x 40 (GEMV chunks of 16 positions, the logits of every row)."""
    eng = _eager(_internlm_engine("internlm_w4"))
    toks = weights.synthetic_tokens(2, 40, eng.cfg.vocab_size, seed=13)
    a = Audit(eng)
    a.run_full(toks, eng.forward_full)
    a.report("forward_full internlm w4 2 x 40")
    _biased(a)


def _internlm_cfg(dim, heads, ffn, gs, max_seq_len):
    return EngineConfig(kind="llama", dim=dim, n_layers=1, n_heads=heads, ffn_hidden=ffn, vocab_size=2048,
                        max_seq_len=max_seq_len, bits=4, group_size=gs, attn_bias=True)


@pytest.mark.timeout(900)
def test_internlm_7b_width_one_layer():
    """D 4096, 32 heads, F 11008, per-channel W4: bs 1 (a 3-token prompt, 2 decode steps through gemv1), then bs 3, a
    40-token tensor-core prompt per sequence and 1 decode step."""
    torch.cuda.empty_cache()
    eng = DecodeEngine(_internlm_cfg(4096, 32, 11008, 0, 64), DEV).load_random(7)
    a = audit_schedule(eng, 1, _calls(3, 0, 2), "internlm-7b width w4 bs 1")
    assert _paths(a) == [("gemv", 3), ("gemv", 1), ("gemv", 1)]
    _biased(a)
    a = audit_schedule(eng, 3, _calls(40, 0, 1), "internlm-7b width w4 bs 3 tc", tc=True)
    _tc_paths(a, [("tc", 40)] * 3 + [("gemv", 3)])
    _biased(a, tc=True)
    del eng, a
    torch.cuda.empty_cache()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("gs", [128, 0], ids=["w4_g128", "w4_pc"])
def test_internlm_20b_width_one_layer(gs):
    """D 5120, 40 heads, F 13824.  W4 g128 runs GEMV chunks only: bs 2, a 20-token prompt (16 + 4 per sequence), 2 decode
    steps.  Per-channel W4 runs tensor-core prompts: bs 1, 40 tokens, 1 decode step."""
    torch.cuda.empty_cache()
    eng = DecodeEngine(_internlm_cfg(5120, 40, 13824, gs, 64), DEV).load_random(11 + gs)
    if gs:
        assert not eng.prefill_tc_supported()
        a = audit_schedule(eng, 2, _calls(20, 0, 2), "internlm-20b width w4 g128 bs 2", tc=True)
        _tc_paths(a, [("gemv", 32), ("gemv", 8), ("gemv", 2), ("gemv", 2)])
        _biased(a)
    else:
        a = audit_schedule(eng, 1, _calls(40, 0, 1), "internlm-20b width w4 bs 1 tc", tc=True)
        _tc_paths(a, [("tc", 40), ("gemv", 1)])
        _biased(a, tc=True)
    del eng, a
    torch.cuda.empty_cache()


def test_internlm_engine_never_takes_the_persistent_kernels():
    """The persistent whole-step kernels have no bias epilogue: with use_mega set, an InternLM engine of the one shape they
    serve (per-channel W4, bs 1, fp16 head) still runs the separate kernels, while the same LLaMA engine would not."""
    cfg = _internlm_cfg(256, 2, 768, 0, 64)
    for bias in (True, False):
        eng = DecodeEngine(EngineConfig(**dict(vars(cfg), attn_bias=bias)), DEV).load_random(0)
        eng.use_mega = True
        assert eng.mega_supported(1) == (not bias), bias


# ----------------------------------------------------------------------- InternLM bias epilogue at the edges --------
CODECS = [(4, 0), (4, 128), (3, 0), (2, 64), (16, 0)]
WIDTHS = {"7b": (4096, 32), "20b": (5120, 40)}
EDGE_POS = (0, 31, 32, 2047)  # and cache_seq - 1


def _norm_inputs(T, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    resid = torch.randn(T, K, generator=g, device=DEV).half()
    delta = (0.3 * torch.randn(T, K, generator=g, device=DEV)).half()
    gamma = (1 + 0.2 * torch.randn(K, generator=g, device=DEV)).half()
    return resid, delta, gamma


def _qkv_launch(pl, T, Hq, Hkv, S, pos, rope, resid, delta, gamma, bias):
    """One EPI_QKV launch of T tokens (one sequence each) into NaN-sentinel q / h_out (one spare row each) and caches, with
    the engine's PDL / K-V prefetch arguments -> (q, h_out, kc, vt)."""
    nq, nkv = Hq * 128, Hkv * 128
    kc = kvlayout.k_to_engine(nan16(T, Hkv, S, 128, device=DEV))
    vt = nan16(T, Hkv, S // 32, 128, 32, device=DEV)
    q, h_out = nan16(T + 1, nq, device=DEV), nan16(T + 1, pl.K, device=DEV)
    qkv = dict(n_q_rows=nq, n_kv_rows=nkv, rope=rope, pos=torch.tensor(pos, dtype=torch.int32, device=DEV),
               tokens_per_seq=1, kcache=kc, vtcache=vt, cache_seq=S, prefetch_kv=True)
    kw = {} if bias is None else dict(bias=bias, bias_mode=ops.B200_BIAS_ACC)
    ops.gemv(pl, T, out=q, resid=resid, delta=delta, h_out=h_out, gamma=gamma, eps=EPS, epilogue=ops.B200_EPI_QKV, qkv=qkv,
             use_pdl=True, **kw)
    torch.cuda.synchronize()
    return q, h_out, kc, vt


def _check_bias_qkv(pl, W, A, T, Hq, Hkv, S, pos, rope, bias, label, seed):
    """-> worst err / tol of y.  Asserts everything the module docstring lists for one launch."""
    nq, nkv = Hq * 128, Hkv * 128
    resid, delta, gamma = _norm_inputs(T, pl.K, seed)
    q, h_out, kc, vt = _qkv_launch(pl, T, Hq, Hkv, S, pos, rope, resid, delta, gamma, bias)
    h = resid + delta
    assert _bits16(h_out[:T]).equal(_bits16(h)) and bool((_bits16(h_out[T:]) == SENT).all()), (label, "h_out")
    assert bool((_bits16(q[T:]) == SENT).all()), (label, "q written past row T")
    assert int((_bits16(kc) != SENT).sum()) == T * nkv and int((_bits16(vt) != SENT).sum()) == T * nkv, (label, "cache")
    # the F16 launch with the same bias: the fp16 y RoPE starts from
    y = nan16(T, pl.N, device=DEV)
    ops.gemv(pl, T, out=y, resid=resid, delta=delta, gamma=gamma, eps=EPS, bias=bias, bias_mode=ops.B200_BIAS_ACC)
    torch.cuda.synchronize()
    b = bias.double()
    worst = 0.0
    for t in range(T):
        X = x_candidates(h[t], gamma, EPS).double()
        Y, M = X @ W.T + b[None], X.abs() @ A.T
        tol = gemv_tol(Y, M) + BIAS_ADD_REL * Y.abs()
        worst = max(worst, float(((y[t].double()[None] - Y).abs() / tol).amax(1).min()))
    assert worst <= 1.0, (label, worst)
    qr, kr, vr = qkv_from_y(y, rope, pos, nq, nkv)
    assert _bits16(q[:T]).equal(_bits16(qr)), (label, "q != RoPE(y)")
    k_can, v_can = kvlayout.k_from_engine(kc), kvlayout.v_from_engine(vt)
    for t in range(T):
        assert _bits16(k_can[t, :, pos[t]].reshape(-1)).equal(_bits16(kr[t])), (label, t, "K")
        assert _bits16(v_can[t, :, pos[t]].reshape(-1)).equal(_bits16(vr[t])), (label, t, "V")
    # B200_BIAS_ACC with b = 0 is the bias-free launch, bit for bit
    zero = torch.zeros_like(bias)
    outs = [_qkv_launch(pl, T, Hq, Hkv, S, pos, rope, resid, delta, gamma, bb) for bb in (zero, None)]
    for u, v in zip(*outs):
        assert _bits16(u).equal(_bits16(v)), (label, "BIAS_ACC with b = 0 differs from the bias-free launch")
    return worst


def _bias(N, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return ((torch.rand(N, generator=g, device=DEV) * 2 - 1) * 0.5).half()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("width", list(WIDTHS))
@pytest.mark.parametrize("bits,gs", CODECS, ids=[f"w{b}g{g}" for b, g in CODECS])
def test_bias_qkv_epilogue_at_real_widths(bits, gs, width):
    """Wqkv at InternLM-7B / 20B width (N = 3 D), every codec: T = 1 (gemv1 for the quantised codecs) at each edge position,
    then T = 2, 8, 9, 32 (the HMMA kernel; 9 and 32 across its token groups) with the positions dealt out in turn."""
    K, H = WIDTHS[width]
    S = 4096
    pl, W, A = _linear(bits, gs, 3 * K, K, seed=K + bits * 10 + gs)
    bias = _bias(3 * K, seed=bits + gs)
    rope = rope_table(128, 2 * S, 10000.0, None).to(DEV)
    edges = EDGE_POS + (S - 1,)
    rep = []
    for ps in edges:
        rep.append(_check_bias_qkv(pl, W, A, 1, H, H, S, [ps], rope, bias, f"{width} w{bits}g{gs} T=1 pos={ps}", ps + 1))
    for T in (2, 8, 9, 32):
        pos = [edges[t % len(edges)] for t in range(T)]
        rep.append(_check_bias_qkv(pl, W, A, T, H, H, S, pos, rope, bias, f"{width} w{bits}g{gs} T={T}", T * 3))
    print(f"\n[bias qkv {width} w{bits} g{gs}] y worst err/tol: T=1 {max(rep[:5]):.3f}, T=2..32 {max(rep[5:]):.3f}")


@pytest.mark.timeout(300)
@pytest.mark.parametrize("bits,gs", [(4, 0), (4, 128)], ids=["w4_pc", "w4_g128"])
def test_bias_qkv_epilogue_beyond_the_staged_tiles(bits, gs):
    """Hq = 2 SMs + 8 q heads, Hkv 8, K 256 (as test_gemv1_epilogue_beyond_the_staged_tiles sizes it): more than 16 tiles
    per CTA, so the bias and the RoPE factors of the later tiles come from global memory.  T = 1, 2, 9."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    Hq, Hkv, K, S = 2 * sms + 8, 8, 256, 64
    N = (Hq + 2 * Hkv) * 128
    assert N // 16 > 16 * sms
    pl, W, A = _linear(bits, gs, N, K, seed=N + gs)
    bias = _bias(N, seed=gs + 5)
    rope = rope_table(128, 2 * S, 10000.0, None).to(DEV)
    rep = [_check_bias_qkv(pl, W, A, T, Hq, Hkv, S, [(33, S - 1)[t % 2] for t in range(T)], rope, bias,
                           f"non-staged w{bits}g{gs} T={T}", T + 40) for T in (1, 2, 9)]
    print(f"\n[bias qkv non-staged w{bits} g{gs}] {N // 16} tiles on {sms} SMs; y worst err/tol {max(rep):.3f}")


# ---------------------------------------------------------------------------------------- mixtral_sparse engine -----
def _sparse_engine(name, max_seq_len=64, tied_gate=False):
    """tied_gate: the gate row of every odd expert copies its even neighbour, so every route is an exact tie."""
    args, sd, _, recs, _ = sparse.build_case(name)
    _, bits, gs, _, _, _ = sparse.CASES[name]
    args = dict(args, max_seq_len=max_seq_len)
    if tied_gate:
        base = weights.mixtral_state_dict(args)
        for i in range(args["n_layers"]):
            g = base[f"layers.{i}.feed_forward.gate.weight"]
            g[1::2] = g[0::2]
        recs = omniquant.fake_quantize_state_dict(base, bits, gs)[1] if bits else recs
        sd = sparse.to_sparse(base, args["moe"]["num_experts"])
    cfg = EngineConfig.from_model_args("mixtral_sparse", args, bits=bits or 16, group_size=gs)
    eng = DecodeEngine(cfg, DEV).load_master_state_dict(sd, quant_records=recs if bits else None)
    assert cfg.sparse_moe and eng.E_loc == cfg.num_experts
    return eng


def _fp32_rule(a):
    assert a.routed > 0 and all("fp32 rule" in k for k in a.stats if k.startswith("moe_route")), sorted(a.stats)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", list(sparse.CASES))
def test_tiny_sparse_gemv_schedules(name):
    """Batch 2: a 5-token prompt, a 12-token continuation, 2 decode steps (t_max 16: chunks of 8 positions); batch 17,
    above t_max: a 6-token prompt and 2 decode steps (sequence groups of 16 and 1, T = 1 launches at row0 16)."""
    a = audit_schedule(_sparse_engine(name), 2, _calls(5, 12, 2), f"{name} bs 2")
    _fp32_rule(a)
    a = audit_schedule(_sparse_engine(name), 17, _calls(6, 0, 2), f"{name} bs 17")
    _fp32_rule(a)
    assert ("gemv", 1) in _paths(a)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("p0,p1", [(40, 37), (300, 40)])
def test_tiny_sparse_w4_tensor_core_prompts(p0, p1):
    """Per-channel W4 (the only Mixtral codec on the tensor cores): batch 2, a p0-token prompt, a p1-token continuation
    (tensor cores again), 1 decode step."""
    eng = _sparse_engine("mixtral_sparse_w4", max_seq_len=384)
    assert eng.prefill_tc_supported()
    a = audit_schedule(eng, 2, _calls(p0, p1, 1), f"mixtral_sparse w4 tc ({p0}, {p1})", tc=True)
    chunks = [min(256, p0 - o) for o in range(0, p0, 256)]
    _tc_paths(a, [("tc", c) for c in chunks] * 2 + [("tc", p1)] * 2 + [("gemv", 2)])
    _fp32_rule(a)


@pytest.mark.timeout(600)
def test_tiny_sparse_fp16_stays_on_gemv_chunks():
    """fp16 Mixtral prompts never take the tensor cores: a 40-token prompt runs as GEMV chunks even with tc enabled."""
    eng = _sparse_engine("mixtral_sparse_fp16", max_seq_len=64)
    assert not eng.prefill_tc_supported()
    a = audit_schedule(eng, 2, _calls(40, 0, 1), "mixtral_sparse fp16 40 tc enabled", tc=True)
    assert all(p == "gemv" for p, _ in _paths(a))
    _fp32_rule(a)


@pytest.mark.timeout(600)
def test_tiny_sparse_w4_tied_gate_rows():
    """Experts 2i and 2i + 1 share a gate row: every route is an exact tie of fp32 scores, and goes to the lower index
    (kernel_route_f32, as torch.topk in mixtral_sparse.py).  GEMV chunks, then a 260-token tensor-core prompt."""
    a = audit_schedule(_sparse_engine("mixtral_sparse_w4", tied_gate=True), 2, _calls(20, 20, 2), "sparse tied gate")
    assert a.ties == a.routed > 0 and not a.flips, (a.ties, a.routed, a.flips[:2])
    eng = _sparse_engine("mixtral_sparse_w4", max_seq_len=320, tied_gate=True)
    a = audit_schedule(eng, 2, _calls(260, 0, 1), "sparse tied gate tc", tc=True)
    _tc_paths(a, [("tc", 256), ("tc", 4)] * 2 + [("gemv", 2)])
    assert a.ties == a.routed > 0 and not a.flips, (a.ties, a.routed, a.flips[:2])


@pytest.mark.timeout(900)
@pytest.mark.parametrize("hidden", [14336, 3584], ids=["8x7b_tp1", "tp4_rank_shape"])
def test_sparse_real_widths_one_layer(hidden):
    """Mixtral-8x7B width (D 4096, 8 experts, top-2), every expert sliced: F 14336 at TP 1, and F 3584, the launches one
    rank of TP 4 makes (the all-reduce aside).  W4 g128 through GEMV chunks (bs 2, a 24-token prompt, 2 decode steps);
    per-channel W4 through a 40-token tensor-core prompt and 1 decode step."""
    for gs in (128, 0):
        torch.cuda.empty_cache()
        args = dict(MIXTRAL_WIDTH, hidden_dim=hidden, max_seq_len=64)
        eng = DecodeEngine(EngineConfig.from_model_args("mixtral_sparse", args, bits=4, group_size=gs), DEV).load_random(3)
        assert eng.F == hidden and eng.E_loc == 8
        if gs:
            a = audit_schedule(eng, 2, _calls(24, 0, 2), f"mixtral_sparse F {hidden} w4 g128 bs 2")
        else:
            a = audit_schedule(eng, 1, _calls(40, 0, 1), f"mixtral_sparse F {hidden} w4 tc", tc=True)
            _tc_paths(a, [("tc", 40), ("gemv", 1)])
        _fp32_rule(a)
        del eng, a
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------ the audit refuses -------
def test_audit_refuses_a_bias_or_an_argument_it_does_not_check(monkeypatch):
    """A bias on wo of a model without one fails the audit end to end; so do a bias on a SiLU launch and arguments no
    checker takes (a bias to attention, a score rule to the embedding)."""
    from oracle import cases
    args = dict(cases.TINY_LLAMA, max_seq_len=64)
    sd = weights.llama_state_dict(args, seed=0)
    eng = DecodeEngine(EngineConfig.from_model_args("llama", args, bits=4, group_size=0), DEV)
    eng.load_master_state_dict(sd, quant_records=omniquant.fake_quantize_state_dict(sd, 4, 0)[1])
    zero = torch.zeros(eng.cfg.dim, dtype=torch.float16, device=DEV)
    with monkeypatch.context() as m:
        m.setattr(engine_mod, "_wo_bias", lambda lw: dict(bias=zero, bias_mode=ops.B200_BIAS_OUT))
        with pytest.raises(AssertionError, match="a bias this linear does not have"):
            audit_schedule(eng, 1, _calls(3, 0, 0), "llama with a stray wo bias")
    a = Audit(_eager(eng))

    def noop(*x, **kw):
        return None
    lw = eng.layers[0]
    with pytest.raises(AssertionError, match="a bias on a gemv epilogue without a bias checker"):
        a._wrap("gemv", noop)(lw.w13, 1, out=eng.act, epilogue=ops.B200_EPI_SILU, bias=zero, bias_mode=ops.B200_BIAS_ACC)
    with pytest.raises(AssertionError, match="an argument its checker does not check"):
        a._wrap("attn_decode", noop)(eng.q, eng.kcache[0], eng.vtcache[0], eng.pos, eng.attn, T=1, Hq=eng.Hq, Hkv=eng.Hkv,
                                     cache_seq=eng.cache_seq, tokens_per_seq=1, max_kv_len=128, bias=zero)
    with pytest.raises(AssertionError, match="an argument its checker does not check"):
        a._wrap("embed", noop)(eng.tokens, eng.tok_emb, eng.h[0], 1, eng.cfg.dim, eng.cfg.vocab_size, scores_f32=True)
