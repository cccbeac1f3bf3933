"""CPU: serving `internlm` checkpoints (accessory/model/LLM/internlm.py).

  * The port (oracle/internlm.py) against the unmodified module, bit for bit in fp16 and fp32, and against the goldens.
  * InternLM's RoPE equals LLaMA's on q / k rows taken in checkpoint.internlm_rope_perm order, bit for bit.
  * checkpoint.InternLMView: names, the q / k row permutation, the MLP swap, the biases.
  * EngineConfig.from_model_args('internlm'), its refusals, and the refusal of a multi-shard folder.
  * The real library's host-side checks accept every launch of InternLM-7B / 20B widths (W4 bs 1, W4g128 bs 1, W4 bs 8,
    fp16 prompt 128, W3 prompt 48) and refuse malformed bias arguments.
  * A launch trace: the bias pointers reach exactly the Wqkv and wo launches of every layer on every path.
  * A packed-shard round trip.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import llama2_accessory_b200 as pkg
from llama2_accessory_b200 import _cabi, checkpoint, ops
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig
from oracle import cases, internlm
from oracle import llama_port

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NO_GPU = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box WITHOUT a GPU (the launches must not run)")


# ------------------------------------------------------------------------------------------------ oracle --------
@pytest.mark.skipif(not internlm.reference_available(), reason="reference internlm.py absent")
@pytest.mark.parametrize("name", list(internlm.CASES))
def test_port_equals_the_unmodified_module_bit_for_bit(name):
    args, sd, sd_ref, recs, toks = internlm.build_case(name)
    _, _, _, _, plen, ndec = internlm.CASES[name]
    for dt in (torch.float16, torch.float32):
        ref = cases.run_schedule(internlm.reference_model(args, sd_ref, dt), toks, plen, ndec)
        port = cases.run_schedule(internlm.InternLMPortModel(args, sd_ref, dt), toks, plen, ndec)
        assert torch.equal(ref, port), (name, dt, (ref - port).abs().max())


@pytest.mark.parametrize("name", list(internlm.CASES))
def test_port_matches_the_goldens(name):
    """tests/test_oracle.py's rule: fp32 bit for bit, fp16 to one ulp (the fp16 CPU GEMM depends on the host ISA)."""
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    args, sd, sd_ref, recs, toks = internlm.build_case(name)
    assert np.array_equal(g["tokens"], toks.numpy())
    p32 = internlm.port_logits(name, torch.float32).numpy()
    assert np.array_equal(p32, g["logits_fp32"])
    p16 = internlm.port_logits(name, torch.float16).numpy()
    ulp = np.spacing(np.abs(g["logits_fp16"]).astype(np.float16)).astype(np.float32)
    assert (np.abs(p16 - g["logits_fp16"]) <= ulp).all()


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32, torch.float64])
def test_internlm_rope_is_llama_rope_on_permuted_rows(dtype):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 7, 3, 128, generator=g).to(dtype)
    fc = llama_port.precompute_freqs_cis(128, 64)[5:12]
    perm = checkpoint.internlm_rope_perm(128)
    assert perm[:4].tolist() == [0, 64, 1, 65] and sorted(perm.tolist()) == list(range(128))
    assert torch.equal(internlm.rope(x, fc), llama_port.rope(x[..., perm], fc))


# ------------------------------------------------------------------------------------------------ key view ------
def test_key_view_names_permutation_and_mlp_swap():
    args = internlm.TINY_INTERNLM
    sd = {("llma." + k): v for k, v in internlm.state_dict(args).items()}
    H, D = args["num_attention_heads"], args["hidden_size"]
    v = checkpoint.InternLMView(sd, H)
    assert "layers.0.mixer.Wqkv.weight" not in v and len(v) == len(sd) + 2 * 2 * args["num_layers"]
    assert torch.equal(v["tok_embeddings.weight"], sd["llma.embedding.weight"])
    assert torch.equal(v["output.weight"], sd["llma.head.weight"])
    assert torch.equal(v["norm.weight"], sd["llma.norm.weight"])
    p, q = "layers.1.", "llma.layers.1."
    W, b = sd[q + "mixer.Wqkv.weight"], sd[q + "mixer.Wqkv.bias"]
    idx = torch.cat([h * 128 + checkpoint.internlm_rope_perm(128) for h in range(H)])
    assert torch.equal(v[p + "attention.wq.weight"], W[:D][idx]) and torch.equal(v[p + "attention.wq.bias"], b[:D][idx])
    assert torch.equal(v[p + "attention.wk.weight"], W[D:2 * D][idx]) and torch.equal(v[p + "attention.wk.bias"], b[D:2 * D][idx])
    assert torch.equal(v[p + "attention.wv.weight"], W[2 * D:]) and torch.equal(v[p + "attention.wv.bias"], b[2 * D:])
    assert torch.equal(v[p + "attention.wo.weight"], sd[q + "mixer.out_proj.weight"])
    assert torch.equal(v[p + "attention.wo.bias"], sd[q + "mixer.out_proj.bias"])
    assert torch.equal(v[p + "feed_forward.w1.weight"], sd[q + "mlp.w1.weight"])
    assert torch.equal(v[p + "feed_forward.w3.weight"], sd[q + "mlp.w2.weight"])   # up
    assert torch.equal(v[p + "feed_forward.w2.weight"], sd[q + "mlp.w3.weight"])   # down
    assert torch.equal(v[p + "attention_norm.weight"], sd[q + "norm1.weight"])
    assert torch.equal(v[p + "ffn_norm.weight"], sd[q + "norm2.weight"])
    # OmniQuant records recovered from the view reproduce the permuted fake-quantised rows bit for bit
    fq = checkpoint.InternLMView(internlm.fake_quantize(internlm.state_dict(args), 4, 128), H)
    recs = checkpoint.LazyQuantRecords(fq, 4, 128)
    assert set(recs) == {k for k in fq if checkpoint.QUANTISED_KEY.search(k)} and len(recs) == 7 * args["num_layers"]
    r = recs["layers.0.attention.wk.weight"]
    assert r["group_size"] == 128 and r["q"].shape == (D, D)


# ------------------------------------------------------------------------------------------------ config --------
def test_config_mapping_at_7b_and_20b():
    c7 = EngineConfig.from_model_args("internlm", dict(num_layers=32, hidden_size=4096, num_attention_heads=32, mlp_ratio=8 / 3,
                                                       multiple_of=256, layer_norm_epsilon=1e-6, norm_eps=1e-3,
                                                       vocab_size=103168, rope_theta=10000))
    assert (c7.kind, c7.dim, c7.n_layers, c7.n_heads, c7.kv_heads, c7.ffn_hidden) == ("llama", 4096, 32, 32, 32, 11008)
    assert c7.norm_eps == 1e-6 and c7.attn_bias and c7.vocab_size == 103168 and c7.head_dim == 128
    c20 = EngineConfig.from_model_args("internlm", dict(num_layers=60, hidden_size=5120, num_attention_heads=40,
                                                        vocab_size=103168))
    assert (c20.dim, c20.ffn_hidden, c20.head_dim, c20.norm_eps) == (5120, 13824, 128, 1e-5)
    assert not EngineConfig.from_model_args("llama", cases.TINY_LLAMA).attn_bias


def test_config_refusals():
    a = dict(internlm.TINY_INTERNLM)
    with pytest.raises(ValueError, match="TP = 1"):
        EngineConfig.from_model_args("internlm", a, tp_rank=0, tp_world=2)
    with pytest.raises(ValueError, match="norm_type"):
        EngineConfig.from_model_args("internlm", dict(a, norm_type="layernorm"))
    with pytest.raises(ValueError, match="use_swiglu"):
        EngineConfig.from_model_args("internlm", dict(a, use_swiglu=False))
    with pytest.raises(ValueError, match="tp_world = 1"):
        DecodeEngine(EngineConfig.from_model_args("llama", cases.TINY_LLAMA, tp_world=2, attn_bias=True), "cpu")


def test_multi_shard_folder_is_refused(tmp_path):
    args = internlm.TINY_INTERNLM
    sd = internlm.state_dict(args)
    for i in range(2):  # two replicated shards: the file listing alone makes this a TP = 2 checkpoint
        torch.save({"model": {"llma." + k: v for k, v in sd.items()}}, tmp_path / f"consolidated.{i:02d}-of-02.model.pth")
    json.dump({"llama_type": "internlm"}, open(tmp_path / "meta.json", "w"))
    json.dump({k: v for k, v in args.items() if k not in ("max_seq_len", "max_batch_size")}, open(tmp_path / "config.json", "w"))
    with pytest.raises(ValueError, match="TP = 1"):
        checkpoint.build_engine_from_pretrained(str(tmp_path), device="cpu")


def test_single_shard_folder_loads_on_the_host(tmp_path):
    """build_engine_from_pretrained on a one-shard folder (engine on the CPU device: packing and the biases, no launch)."""
    args = internlm.TINY_INTERNLM
    sd = internlm.fake_quantize(internlm.state_dict(args), 4)
    torch.save({"model": {"llma." + k: v for k, v in sd.items()}}, tmp_path / "consolidated.00-of-01.model.pth")
    json.dump({"llama_type": "internlm"}, open(tmp_path / "meta.json", "w"))
    json.dump({k: v for k, v in args.items() if k not in ("max_seq_len", "max_batch_size")}, open(tmp_path / "config.json", "w"))
    eng, meta = checkpoint.build_engine_from_pretrained(str(tmp_path), fake_quantised=True, max_seq_len=64, device="cpu")
    assert meta["llama_type"] == "internlm" and eng.cfg.attn_bias
    v = checkpoint.InternLMView(sd, args["num_attention_heads"])
    lw = eng.layers[1]
    assert torch.equal(lw.bqkv, torch.cat([v[f"layers.1.attention.w{x}.bias"] for x in "qkv"]))
    assert torch.equal(lw.bo, sd["layers.1.mixer.out_proj.bias"])
    assert not eng.mega_supported(1)


# ------------------------------------------------------------------------------------------------ library -------
class Validator:
    """The real entry points: rc < 0 is a rejection by the library's own checks; rc > 0 is the first CUDA call failing on a
    box without a driver, i.e. every host-side check passed (tests/test_launch_validation_cpu.py)."""
    LAUNCHES = ("b200_gemv", "b200_attn_decode", "b200_embed", "b200_prefill_gemm_w4", "b200_prefill_gemm_w4_bias",
                "b200_prefill_rmsnorm", "b200_prefill_rope_kv", "b200_prefill_silu_mul", "b200_argmax", "b200_advance_pos")

    def __init__(self, real):
        self.real, self.rejected, self.accepted = real, [], {}

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        if name not in self.LAUNCHES:
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
    return v


I7 = dict(num_layers=1, hidden_size=4096, num_attention_heads=32, vocab_size=103168)
I20 = dict(num_layers=1, hidden_size=5120, num_attention_heads=40, vocab_size=103168)


@NO_GPU
@pytest.mark.parametrize("name,margs,bits,gs,bsz,prompt", [
    ("7B_W4_bs1", I7, 4, 0, 1, 40), ("7B_W4g128_bs1", I7, 4, 128, 1, 40), ("7B_W4_bs8", I7, 4, 0, 8, 3),
    ("7B_fp16_prompt128", I7, 16, 0, 1, 128), ("7B_W3_prompt48", I7, 3, 0, 1, 48),
    ("20B_W4_bs1", I20, 4, 0, 1, 40), ("20B_W4g128_bs1", I20, 4, 128, 1, 40), ("20B_W4_bs8", I20, 4, 0, 8, 3),
    ("20B_fp16_prompt128", I20, 16, 0, 1, 128), ("20B_W3_prompt48", I20, 3, 0, 1, 48),
], ids=lambda x: x if isinstance(x, str) else "")
def test_library_accepts_every_launch_at_real_widths(validator, name, margs, bits, gs, bsz, prompt):
    args = dict(margs, max_seq_len=prompt + 64)
    eng = DecodeEngine(EngineConfig.from_model_args("internlm", args, bits=bits, group_size=gs), "cpu")
    eng.load_random(seed=0)
    eng.use_graph = False
    toks = torch.randint(1, args["vocab_size"], (bsz, prompt + 2), generator=torch.Generator().manual_seed(1))
    assert eng.forward_inference(toks[:, :prompt], 0).shape == (bsz, args["vocab_size"])
    for j in range(2):
        eng.forward_inference(toks[:, prompt + j:prompt + j + 1], prompt + j)
    assert not validator.rejected, validator.rejected[:4]
    if prompt > 32 and not gs:
        assert validator.accepted.get("b200_prefill_gemm_w4_bias", 0) == 2     # Wqkv and wo of the tensor-core prompt
    assert validator.accepted.get("b200_gemv", 0) > 0


@NO_GPU
def test_malformed_bias_arguments_are_refused(validator):
    from llama2_accessory_b200.quant import random_packed
    lin = random_packed(4, 256, 256, 0, "cpu", 0)
    x, out, b = (torch.zeros(n, dtype=torch.float16) for n in (256, 256, 256))
    cases_ = [dict(bias=None, bias_mode=3), dict(bias=b, bias_mode=-1), dict(bias=b, bias_mode=0),
              dict(bias=None, bias_mode=ops.B200_BIAS_ACC), dict(bias=b, bias_mode=1, epilogue=ops.B200_EPI_F32),
              dict(bias=b, bias_mode=2, epilogue=ops.B200_EPI_SILU)]
    for kw in cases_:
        ops.gemv(lin, 1, xin=x, out=out, **kw)
    msgs = [m for _, rc, m in validator.rejected]
    assert len(msgs) == len(cases_) and all(rc == _cabi.B200_E_INVAL if hasattr(_cabi, "B200_E_INVAL") else rc == -1
                                            for _, rc, _ in validator.rejected), validator.rejected
    assert "bias_mode must be" in msgs[0] and "bias_mode must be" in msgs[1] and "needs bias_mode" in msgs[2]
    assert "needs a bias" in msgs[3] and "fp16 and QKV epilogues" in msgs[4] and "fp16 and QKV epilogues" in msgs[5]
    # MoE slot indirection and the fused all-reduce
    slot = torch.zeros(1, dtype=torch.int32)
    ops.gemv(lin, 1, xin=x, out=out, bias=b, bias_mode=1, moe=dict(slot_expert=slot, expert_id=0, n_slots=1, src_div=1))
    ops.gemv(lin, 1, xin=x, out=out, bias=b, bias_mode=2,
             ar=dict(world=2, rank=0, step=0x1000, period=4, err=None, out_peers=(C.c_void_p * 2)(0x2000, 0x3000), out_id=0))
    assert "MoE slot indirection" in validator.rejected[-2][2] and "fused all-reduce" in validator.rejected[-1][2]
    # the prompt GEMM: a bias needs a mode, and a mode outside {1, 2} is refused
    ls = lin.c_struct()
    for bias, mode in ((None, 1), (b, 0), (b, 3)):
        assert validator.real.b200_prefill_gemm_w4_bias(C.byref(ls), x.data_ptr(), None if bias is None else bias.data_ptr(),
                                                         mode, out.data_ptr(), 1, None) == -1
    # a well-formed bias call gets past every host check (rc > 0: no driver here)
    assert validator.real.b200_prefill_gemm_w4_bias(C.byref(ls), x.data_ptr(), b.data_ptr(), 2, out.data_ptr(), 1, None) > 0


# ------------------------------------------------------------------------------------------------ launch trace --
class Recorder:
    LAUNCHES = Validator.LAUNCHES

    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        if name not in self.LAUNCHES:
            return getattr(self.real, name)

        def launch(*args):
            a = [x._obj if hasattr(x, "_obj") else x for x in args]
            if name == "b200_gemv":
                g = a[0]
                self.calls.append((name, g.lin.qweight, g.bias, g.bias_mode, g.epilogue))
            elif name.startswith("b200_prefill_gemm_w4"):
                bias = a[2] if name.endswith("_bias") else None
                self.calls.append((name, a[0].qweight, bias, a[3] if bias else 0, None))
            else:
                self.calls.append((name,))
            return 0
        return launch


def test_launch_trace_bias_reaches_exactly_wqkv_and_wo(monkeypatch):
    pkg.build()
    rec = Recorder(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", rec)
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0))
    monkeypatch.setattr(ops, "_f16", lambda t, name: None)
    args = dict(internlm.TINY_INTERNLM, num_layers=3, max_seq_len=128)
    eng = DecodeEngine(EngineConfig.from_model_args("internlm", args, bits=4), "cpu")
    eng.load_random(seed=2)
    eng.use_graph = False
    want = {}
    for lw in eng.layers:
        want[lw.wqkv.qweight.data_ptr()] = (lw.bqkv.data_ptr(), ops.B200_BIAS_ACC)
        want[lw.wo.qweight.data_ptr()] = (lw.bo.data_ptr(), ops.B200_BIAS_OUT)
    toks = torch.randint(1, 1024, (3, 60), generator=torch.Generator().manual_seed(0))
    paths = {
        "gemv-chunk prompt": lambda: eng.forward_inference(toks[:2, :7], 0),
        "bs>1 decode": lambda: eng.forward_inference(toks[:2, 7:8], 7),
        "tensor-core prompt": lambda: eng.forward_inference(toks[:1, :48], 0),
        "tensor-core continuation": lambda: eng.forward_inference(toks[:1, 48:58], 48),
        "bs=1 decode": lambda: eng.forward_inference(toks[:1, 58:59], 58),
        "forward_full": lambda: eng.forward_full(toks[:3, :40]),
    }
    monkeypatch.setenv("B200_FORCE_TC", "0")
    for what, run in paths.items():
        rec.calls.clear()
        if what == "tensor-core continuation":
            eng.force_tc = True
        run()
        eng.force_tc = False
        lins = [c for c in rec.calls if c[0] in ("b200_gemv", "b200_prefill_gemm_w4", "b200_prefill_gemm_w4_bias")]
        biased = [c for c in lins if c[1] in want]
        assert biased, what
        n_wqkv = sum(1 for c in biased if want[c[1]][1] == ops.B200_BIAS_ACC)
        assert n_wqkv == sum(1 for c in biased if want[c[1]][1] == ops.B200_BIAS_OUT) and n_wqkv % 3 == 0, what
        for name, qw, bias, mode, _ in lins:
            if qw in want:
                assert (bias, mode) == want[qw], (what, name)
                assert name != "b200_prefill_gemm_w4", what   # a biased linear never takes the bias-free prompt GEMM
            else:
                assert not bias and not mode, (what, name)
        tc = any(c[0] == "b200_prefill_gemm_w4_bias" for c in lins)
        assert tc == what.startswith("tensor-core"), what


# ------------------------------------------------------------------------------------------------ packed --------
def test_packed_shard_round_trip(tmp_path):
    args = internlm.TINY_INTERNLM
    cfg = EngineConfig.from_model_args("internlm", args, bits=4)
    a = DecodeEngine(cfg, "cpu").load_random(seed=3)
    checkpoint.save_packed(a, str(tmp_path))
    b = checkpoint.load_packed(DecodeEngine(cfg, "cpu"), str(tmp_path))
    for la, lb in zip(a.layers, b.layers):
        assert torch.equal(la.bqkv, lb.bqkv) and torch.equal(la.bo, lb.bo)
        assert torch.equal(la.wqkv.qweight, lb.wqkv.qweight)
    assert a.step_bytes(1, 64)["weights"] == b.step_bytes(1, 64)["weights"]
    # a LLaMA engine refuses the shard (attn_bias differs); a shard written before attn_bias existed loads as attn_bias False
    with pytest.raises(ValueError, match="attn_bias"):
        checkpoint.load_packed(DecodeEngine(EngineConfig(**{**cfg.__dict__, "attn_bias": False}), "cpu"), str(tmp_path))
    lc = DecodeEngine(EngineConfig.from_model_args("llama", cases.TINY_MHA, bits=4), "cpu").load_random(seed=4)
    fn = checkpoint.save_packed(lc, str(tmp_path / "old"))
    blob = torch.load(fn, weights_only=False)
    del blob["config"]["attn_bias"]
    for d in blob["layers"]:
        del d["bqkv"], d["bo"]
    torch.save(blob, fn)
    old = checkpoint.load_packed(DecodeEngine(EngineConfig.from_model_args("llama", cases.TINY_MHA, bits=4), "cpu"),
                                 str(tmp_path / "old"))
    assert all(lw.bqkv is None and lw.bo is None for lw in old.layers)


def test_step_bytes_count_the_biases():
    cfg = EngineConfig.from_model_args("internlm", internlm.TINY_INTERNLM, bits=4)
    eng = DecodeEngine(cfg, "cpu").load_random(seed=0)
    w = eng.step_bytes(1, 64)["weights"]
    for lw in eng.layers:
        lw.bqkv = lw.bo = None
    D = cfg.dim
    assert w - eng.step_bytes(1, 64)["weights"] == cfg.n_layers * (3 * D + D) * 2
