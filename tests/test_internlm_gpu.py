"""GPU: `internlm` on the H100 -- the Wqkv / out_proj bias epilogues and the engine serving InternLM checkpoints.

  * Kernels at InternLM-7B widths (D 4096: Wqkv N 12288, out_proj N 4096), every codec, T = 1 and T = 2..32: BIAS_OUT is
    bit-identical to fp16(fp16(no-bias launch) + b); BIAS_ACC with b = 0 is bit-identical to the no-bias launch; BIAS_ACC
    is within the no-bias launch's own float64 error plus one fp16 rounding of float64(x . w_hat) + b.  The same for
    b200_prefill_gemm_w4_bias against b200_prefill_gemm_w4 (W4, W3, fp16; T 48 and 300).
  * The engine on the three tiny cases against the goldens of the unmodified module and the port (oracle/internlm.py),
    with the parity rule of tests/test_model_parity_gpu.py: GEMV-chunk prompts and decode (eager = graph replay),
    tensor-core prompts (B200_FORCE_TC too), a continuation prompt at start_pos > 0, forward_full, and the K cache rows
    against the port's k_cache.
  * Serving end to end: build_engine_from_pretrained on a tiny `internlm` folder, the `internlm_b200` drop-in, greedy and
    top-p generate from a 103168-token head.
"""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import checkpoint, generation, ops  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig  # noqa: E402
from llama2_accessory_b200.quant import dequantize, pack_fp16, pack_quantized, quantize_weight  # noqa: E402
from oracle import internlm, weights  # noqa: E402
from oracle.toy_tokenizer import ToyTokenizer  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RULE_FACTOR = 1.5  # tests/test_model_parity_gpu.py
DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _ulp16(x):
    a = np.maximum(np.abs(x), 2.0 ** -14)
    return 2.0 ** (np.floor(np.log2(a)) - 10)


def _linear(bits, gs, N, K, seed):
    """(packed linear on the GPU, w_hat float64 [N, K])."""
    g = torch.Generator().manual_seed(seed)
    w = ((torch.rand(N, K, generator=g) * 2 - 1) / K ** 0.5).half()
    if bits == 16:
        return pack_fp16(w, DEV), w.double()
    q, s, z, g_ = quantize_weight(w, bits, gs)
    return pack_quantized(q, s, z, bits, 0 if g_ >= K else g_, DEV), dequantize(q, s, z, g_).double()


# ----------------------------------------------------------------------------------------- kernels -------------
CODECS = [(4, 0), (4, 128), (3, 0), (2, 64), (16, 0)]


@pytest.mark.parametrize("bits,gs", CODECS, ids=[f"w{b}g{g}" for b, g in CODECS])
@pytest.mark.parametrize("N", [12288, 4096], ids=["wqkv", "out_proj"])
def test_gemv_bias_epilogues_at_7b_widths(bits, gs, N):
    K = 4096
    lin, w64 = _linear(bits, gs, N, K, seed=N + bits)
    gen = torch.Generator(device=DEV).manual_seed(bits)
    b = ((torch.rand(N, device=DEV, generator=gen) * 2 - 1) * 0.5).half()
    zero = torch.zeros(N, dtype=torch.float16, device=DEV)
    for T in (1, 2, 7, 16, 17, 32):
        x = torch.randn(T, K, device=DEV, generator=gen).half()
        outs = {}
        for tag, kw in (("none", {}), ("out", dict(bias=b, bias_mode=ops.B200_BIAS_OUT)),
                        ("acc", dict(bias=b, bias_mode=ops.B200_BIAS_ACC)), ("acc0", dict(bias=zero, bias_mode=ops.B200_BIAS_ACC))):
            o = torch.empty(T, N, dtype=torch.float16, device=DEV)
            ops.gemv(lin, T, xin=x, out=o, **kw)
            outs[tag] = o
        torch.cuda.synchronize()
        y0 = outs["none"]
        assert torch.equal(outs["out"], (y0.float() + b.float()).half()), (bits, gs, N, T)
        assert torch.equal(outs["acc0"], y0), (bits, gs, N, T)
        ref = (x.double().cpu() @ w64.t()).numpy()
        refb = ref + b.double().cpu().numpy()
        e0 = np.abs(y0.double().cpu().numpy() - ref).max()
        err = np.abs(outs["acc"].double().cpu().numpy() - refb)
        assert (err <= e0 + _ulp16(refb)).all(), (bits, gs, N, T, err.max(), e0)


@pytest.mark.parametrize("bits", [4, 3, 16])
def test_prefill_gemm_bias_at_7b_widths(bits):
    N, K = 12288, 4096
    lin, w64 = _linear(bits, 0, N, K, seed=bits)
    gen = torch.Generator(device=DEV).manual_seed(bits)
    b = ((torch.rand(N, device=DEV, generator=gen) * 2 - 1) * 0.5).half()
    zero = torch.zeros(N, dtype=torch.float16, device=DEV)
    for T in (48, 300):
        x = torch.randn(T, K, device=DEV, generator=gen).half()
        outs = {}
        for tag, kw in (("none", {}), ("out", dict(bias=b, bias_mode=ops.B200_BIAS_OUT)),
                        ("acc", dict(bias=b, bias_mode=ops.B200_BIAS_ACC)), ("acc0", dict(bias=zero, bias_mode=ops.B200_BIAS_ACC))):
            o = torch.empty(T, N, dtype=torch.float16, device=DEV)
            ops.prefill_gemm_w4(lin, x, o, T, **kw)
            outs[tag] = o
        torch.cuda.synchronize()
        y0 = outs["none"]
        assert torch.equal(outs["out"], (y0.float() + b.float()).half())
        assert torch.equal(outs["acc0"], y0)
        ref = (x.double().cpu() @ w64.t()).numpy()
        refb = ref + b.double().cpu().numpy()
        e0 = np.abs(y0.double().cpu().numpy() - ref).max()
        err = np.abs(outs["acc"].double().cpu().numpy() - refb)
        assert (err <= e0 + _ulp16(refb)).all(), (bits, T, err.max(), e0)


# ----------------------------------------------------------------------------------------- engine --------------
def _rule(got, ref16, ref32, what):
    e16, e32 = np.abs(got - ref16).max(), np.abs(got - ref32).max()
    floor = np.abs(ref16 - ref32).max()
    print(f"\n[{what}] |eng-ref16|={e16:.3e} |eng-ref32|={e32:.3e} |ref16-ref32|={floor:.3e}")
    assert np.isfinite(got).all()
    assert e16 <= 1e-3 or e32 <= RULE_FACTOR * floor, (what, e16, e32, floor)
    top2 = np.sort(ref32, axis=-1)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 4 * floor
    assert (got.argmax(-1)[clear] == ref32.argmax(-1)[clear]).all(), what


def _engine(args, sd, recs, bits, gs, use_graph=False):
    eng = DecodeEngine(EngineConfig.from_model_args("internlm", args, bits=bits or 16, group_size=gs), DEV)
    eng.use_graph = use_graph
    return eng.load_master_state_dict(sd, quant_records=recs if bits else None)


def _run(eng, toks, sched):
    tk = toks.cuda()
    return np.stack([eng.forward_inference(tk[:, a:b], a).float().cpu().numpy() for a, b in sched])


def _port_pair(args, sd_ref, toks, sched):
    res = []
    for dt in (torch.float16, torch.float32):
        m = internlm.InternLMPortModel(args, sd_ref, dt)
        res.append(np.stack([m.forward_inference(toks[:, a:b], a).float().numpy() for a, b in sched]))
    return res


@pytest.mark.parametrize("name", list(internlm.CASES))
def test_engine_matches_the_goldens(name):
    """GEMV-chunk prompt (5 tokens) and three decode steps, eager and from CUDA graphs; K cache rows against the port."""
    args, sd, sd_ref, recs, toks = internlm.build_case(name)
    _, bits, gs, _, plen, ndec = internlm.CASES[name]
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    sched = [(0, plen)] + [(plen + j, plen + j + 1) for j in range(ndec)]
    eng = _engine(args, sd, recs, bits, gs)
    eager = _run(eng, toks, sched)
    _rule(eager, g["logits_fp16"], g["logits_fp32"], name)
    graph = _run(_engine(args, sd, recs, bits, gs, use_graph=True), toks, sched)
    assert np.array_equal(eager, graph)
    # K cache: the engine stores the port's k_cache rows (the interleaved RoPE output) in its swizzled layout
    port = internlm.InternLMPortModel(args, sd_ref, torch.float32)
    for a, b in sched:
        port.forward_inference(toks[:, a:b], a)
    S = plen + ndec
    s = torch.arange(S)[:, None]
    d = torch.arange(128)[None, :]
    phys = s * 128 + (((d >> 3) ^ ((s & 1) << 2)) << 3) + (d & 7)
    for i in range(args["num_layers"]):
        kc = eng.kcache[i, :toks.shape[0]].float().cpu().reshape(toks.shape[0], -1, eng.cache_seq * 128)
        got = kc[:, :, phys.reshape(-1)].reshape(toks.shape[0], -1, S, 128).transpose(1, 2)
        want = port.k_cache[i][:, :S].float()
        assert (got - want).abs().max() <= 2e-2 * want.abs().max(), (name, i, (got - want).abs().max())


@pytest.mark.parametrize("name", list(internlm.CASES))
@pytest.mark.parametrize("force_tc", [False, True])
def test_engine_prompts_continuation_and_forward_full(monkeypatch, name, force_tc):
    """bs 2: a 40-token prompt (tensor cores where the codec has them; B200_FORCE_TC: every call on the tensor cores), a
    37-token continuation at start_pos 40, two decode steps, then forward_full over the 79 tokens against the port's
    teacher-forced last-position logits."""
    if force_tc:
        monkeypatch.setenv("B200_FORCE_TC", "1")
    args, sd, sd_ref, recs, _ = internlm.build_case(name)
    _, bits, gs, _, _, _ = internlm.CASES[name]
    args = dict(args, max_seq_len=128)
    toks = weights.synthetic_tokens(2, 79, args["vocab_size"], seed=7)
    sched = [(0, 40), (40, 77), (77, 78), (78, 79)]
    eng = _engine(args, sd, recs, bits, gs)
    assert eng.force_tc == force_tc and eng.prefill_tc_supported() == (gs == 0)
    got = _run(eng, toks, sched)
    ref16, ref32 = _port_pair(args, sd_ref, toks, sched)
    _rule(got, ref16, ref32, f"{name} prompt 40 + continuation 37 + decode 2 (force_tc={force_tc})")
    if force_tc:
        return
    full = eng.forward_full(toks[:, :24].cuda()).float().cpu().numpy()          # [2, 24, V]
    steps = [(0, 1)] + [(j, j + 1) for j in range(1, 24)]
    r16, r32 = _port_pair(args, sd_ref, toks, steps)
    _rule(full.transpose(1, 0, 2), r16, r32, f"{name} forward_full 24")


# ----------------------------------------------------------------------------------------- serving -------------
def _folder(tmp_path, args, sd):
    torch.save({"model": {"llma." + k: v for k, v in sd.items()}}, tmp_path / "consolidated.00-of-01.model.pth")
    json.dump({"llama_type": "internlm"}, open(tmp_path / "meta.json", "w"))
    json.dump({k: v for k, v in args.items() if k not in ("max_seq_len", "max_batch_size")}, open(tmp_path / "config.json", "w"))
    return str(tmp_path)


def test_build_engine_from_pretrained_and_packed_round_trip(tmp_path):
    name = "internlm_w4"
    args, sd, sd_ref, recs, toks = internlm.build_case(name)
    _, _, _, _, plen, ndec = internlm.CASES[name]
    sched = [(0, plen)] + [(plen + j, plen + j + 1) for j in range(ndec)]
    eng, meta = checkpoint.build_engine_from_pretrained(_folder(tmp_path, args, sd_ref), fake_quantised=True, max_seq_len=64)
    eng.use_graph = False
    assert meta["llama_type"] == "internlm" and eng.cfg.attn_bias
    got = _run(eng, toks, sched)
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    _rule(got, g["logits_fp16"], g["logits_fp32"], "build_engine_from_pretrained")
    ref = _run(_engine(dict(args, max_seq_len=64), sd, recs, 4, 0), toks, sched)
    assert np.array_equal(got, ref)  # recovered records == the quantiser's own
    checkpoint.save_packed(eng, str(tmp_path / "packed"))
    e2 = checkpoint.load_packed(DecodeEngine(eng.cfg, DEV), str(tmp_path / "packed"))
    e2.use_graph = False
    assert np.array_equal(_run(e2, toks, sched), got)


def _dropin(args, sd, wbits=4):
    from llama2_accessory_b200.model import internlm_b200
    ma = internlm_b200.ModelArgs(**{k: v for k, v in args.items()}, wbits=wbits)
    model = internlm_b200.Transformer(ma)
    model.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    return model.half().cuda()


def test_dropin_module_matches_the_goldens():
    name = "internlm_fp16"
    args, sd, sd_ref, recs, toks = internlm.build_case(name)
    _, _, _, _, plen, ndec = internlm.CASES[name]
    model = _dropin(args, sd, wbits=16)
    sched = [(0, plen)] + [(plen + j, plen + j + 1) for j in range(ndec)]
    tk = toks.cuda()
    got = np.stack([model.forward_inference(tk[:, a:b], a).float().cpu().numpy() for a, b in sched])
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    _rule(got, g["logits_fp16"], g["logits_fp32"], "internlm_b200 drop-in")
    full = model.forward(tk[:, :6]).float().cpu().numpy()
    assert full.shape == (2, 6, args["vocab_size"]) and np.isfinite(full).all()


def test_generate_greedy_and_top_p_at_vocab_103168():
    V = 103168
    args = dict(internlm.TINY_INTERNLM, vocab_size=V)
    model = _dropin(args, internlm.state_dict(args), wbits=16)  # fp16 linears: the port below runs the same weights
    tok = ToyTokenizer(V, 2)
    prompts = ["the quick brown fox", "hello world", "a b c d e f g"]
    greedy = generation.generate(model, tok, prompts, max_gen_len=8)
    assert len(greedy) == 3
    torch.manual_seed(0)
    for device_loop in (True, False):
        texts = generation.generate(model, tok, prompts, max_gen_len=8, temperature=0.8, top_p=0.9, device_loop=device_loop)
        for t in texts:
            assert all(0 <= int(w[1:]) < V for w in t.split()), t
        # a nucleus holding only the arg-max is greedy
        assert generation.generate(model, tok, prompts, max_gen_len=8, temperature=1.0, top_p=1e-6,
                                   device_loop=device_loop) == greedy
    # greedy against the port: the first generated token of every prompt is the port's arg-max
    port = internlm.InternLMPortModel(args, internlm.state_dict(args), torch.float32)
    eng = model.engine
    for p in prompts:
        ids = torch.tensor([tok.encode(p, bos=True, eos=False)])
        ref = port.forward_inference(ids, 0).numpy()[0]
        got = eng.forward_inference(ids.cuda(), 0).float().cpu().numpy()[0]
        top2 = np.sort(ref)[-2:]
        if top2[1] - top2[0] > 1e-2:
            assert got.argmax() == ref.argmax()
