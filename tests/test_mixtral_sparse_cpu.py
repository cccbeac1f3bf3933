"""CPU: `mixtral_sparse` models (accessory/model/LLM/mixtral_sparse.py) -- every expert sliced over the tensor-parallel
ranks, and the fp32 router rule.

  * the fp32 router, restated in torch (oracle.numerics.route_f32), against the routing of the unmodified module (run
    through oracle/shims/{megablocks,stk}), including logits where the fp16 rule of base Mixtral and the fp32 rule pick
    different experts; the line-by-line model of the kernel's fp32 rule (kernel_route_f32) against that statement wherever
    no near-tie exists, and its window (route_f32_explains);
  * the port (oracle/sparse.py) against the unmodified module, and the committed goldens against both;
  * checkpoint merge / split between checkpoint TP 1, 2, 4, 8 and engine TP 1, 2, 4, 8 against the module's own
    _sparse_expert_merge / _sparse_expert_split; the per-expert view the engine loads from; packed-shard config;
  * launch traces of the engine's decode step and tensor-core prompt at TP 1 and rank 1 of TP 2 (every expert, e_first 0,
    F/TP-wide linears, scores_f32 = 1 on every route), against a recording stand-in for the library;
  * C4-width launches (Mixtral-8x7B, W4, bs 16) at TP 1 / 2 / 4 / 8 through the real library's host-side checks;
  * refusals: hidden_dim / TP not a multiple of 128, a scores_f32 other than 0 / 1.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import llama2_accessory_b200 as pkg
from llama2_accessory_b200 import _cabi, checkpoint, ops
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig, check_kernel_limits
from oracle import cases, ref_import, sparse
from oracle.numerics import (fp16_sides, kernel_route, kernel_route_f32, kernel_scores_f32, route_f32, route_f32_explains,
                             route_f32_window, route_weight_window)

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# the unmodified mixtral_sparse.py is read from the reference tree; the staged copy of the hot-path modules does not include it
needs_ref = pytest.mark.skipif(
    not os.path.isfile(os.path.join(ref_import.REF_ROOT, "accessory", "model", "LLM", "mixtral_sparse.py")),
    reason="needs the reference tree's accessory/model/LLM/mixtral_sparse.py")
MIX = dict(dim=4096, n_heads=32, n_kv_heads=8, vocab_size=32000, hidden_dim=14336, rope_theta=1e6,
           moe=dict(num_experts=8, num_experts_per_tok=2))


def _ref_moe_routes(x16, gate16, k, hidden=128):
    """The unmodified MoE.forward on fp16 x [T, D] with router gate16 [E, D]: (selected experts [T, k], weights [T, k])."""
    mod = ref_import.load("mixtral_sparse")
    E, D = gate16.shape
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float16)
    try:
        moe = mod.MoE(D, hidden, E, k)
    finally:
        torch.set_default_dtype(old)
    with torch.no_grad():
        moe.gate.weight.copy_(gate16)
        for w in (moe.w1, moe.w2, moe.w3):
            w.zero_()
    moe.eval()
    got = {}
    real_bins, real_scatter = moe.indices_and_padded_bins, mod.ops.padded_scatter

    def bins(sel):
        got["sel"] = sel.clone()
        return real_bins(sel)

    def scatter(x, indices, bin_ids, weights, *a):
        got["w"] = weights.clone()
        return real_scatter(x, indices, bin_ids, weights, *a)
    moe.indices_and_padded_bins = bins
    mod.ops.padded_scatter = scatter
    try:
        with torch.no_grad():
            moe(x16[None])
    finally:
        mod.ops.padded_scatter = real_scatter
    T = x16.shape[0]
    return got["sel"].long().view(T, k), got["w"].view(T, k)


@needs_ref
def test_fp32_router_restated_matches_the_unmodified_module():
    g = torch.Generator().manual_seed(0)
    T, D, E, k = 256, 64, 8, 2
    x = (torch.randn(T, D, generator=g)).half()
    gate = (torch.randn(E, D, generator=g) * 0.3).half()
    idx_r, w_r = _ref_moe_routes(x, gate, k)
    logits = torch.nn.functional.linear(x.float(), gate.float()).half()  # the module's fp16 nn.Linear (exact here: D = 64)
    assert torch.equal(torch.nn.functional.linear(x, gate), logits)
    idx, w = route_f32(logits, k)
    assert torch.equal(idx, idx_r)
    assert torch.equal(w, w_r)


@needs_ref
def test_crafted_logits_where_the_fp16_and_fp32_rules_disagree():
    """Experts 1 and 2 have fp32 scores that round to the same fp16 value: the fp16 rule takes the lower index (1), the fp32
    rule the larger score (2); the weights differ too.  With an identity router (D = E) the module's logits are x itself."""
    E, k = 8, 2
    rows = []
    for d in (1, 2, 3, 4):  # expert 2's logit d * 2^-14 above expert 1's: scores ~0.1 apart by < half an fp16 step
        rows.append([2.0, 0.0, d * 2.0 ** -14, -2.0, -2.0, -3.0, -3.0, -4.0])
    x = torch.tensor(rows, dtype=torch.float16)
    gate = torch.eye(E, dtype=torch.float16)
    idx16, _ = kernel_route(x, k)
    idx32, w32 = route_f32(x, k)
    idx_r, w_r = _ref_moe_routes(x, gate, k)
    assert torch.equal(idx32, idx_r) and torch.equal(w32, w_r)
    differ = [t for t in range(len(rows)) if not np.array_equal(idx16[t], idx32[t].numpy())]
    assert differ, "no crafted row separates the two rules"
    for t in differ:
        assert list(idx16[t]) == [0, 1] and idx32[t].tolist() == [0, 2]


def _near_ties(lg16, k):
    """Tokens where two statements of the fp32 rule may part legitimately: two of the top k + 1 fp32 scores within the
    window route_f32_window of each other, or a weight's score / sum within route_weight_window of an fp16 midpoint."""
    sc = kernel_scores_f32(lg16).astype(np.float64)
    E = sc.shape[1]
    W, RW = route_f32_window(E), route_weight_window(E, k)
    top = -np.sort(-sc, -1)[:, :k + 1]
    close = ((top[:, :-1] - top[:, 1:]) <= W * (top[:, :-1] + top[:, 1:])).any(-1)
    r = top[:, :k] / top[:, :k].sum(-1, keepdims=True)
    _, _, dist = fp16_sides(torch.from_numpy(r))
    return close | (dist.numpy() <= 2 * RW * r).any(-1)


def _crafted_logits(E):
    """Rows with exact ties, ties one fp16 step apart at 2 and at the subnormal end, and the fp16-rule / fp32-rule
    disagreements of test_crafted_logits_where_the_fp16_and_fp32_rules_disagree (first eight experts)."""
    rows = []
    base = [-1.0 - 0.25 * e for e in range(E)]
    for a, b in ((2.0, 2.0), (2.0, 2.0 + 2.0 ** -9), (2.0 ** -24, 0.0), (0.5, 0.5), (3.0, 3.0 - 2.0 ** -10)):
        for i, j in ((0, 1), (1, 0), (E - 2, E - 1), (2, E - 1)):
            r = list(base)
            r[i], r[j] = a, b
            rows.append(r)
    rows.append([0.0] * E)
    for d in (1, 2, 3, 4):
        rows.append(([2.0, 0.0, d * 2.0 ** -14, -2.0, -2.0, -3.0, -3.0, -4.0] + base)[:E])
    return torch.tensor(rows, dtype=torch.float16)


@pytest.mark.parametrize("E,k", [(8, 2), (4, 2), (16, 4)])
def test_kernel_route_f32_matches_the_torch_statement_away_from_near_ties(E, k):
    """kernel_route_f32 (moe_route_kernel<true> line by line) against route_f32 (mixtral_sparse.py:417-428 in torch) on
    random logits and on crafted near-tie rows: bit for bit wherever no near-tie exists.  Exact ties go to the lower index
    in both; the decided crafted rows separate the fp32 rule from the fp16 rule (kernel_route)."""
    g = torch.Generator().manual_seed(E * 10 + k)
    rand = (torch.randn(4096, E, generator=g) * 2).half()
    crafted = _crafted_logits(E)
    for lg, what in ((rand, "random"), (crafted, "crafted")):
        idx, w = kernel_route_f32(lg, k)
        idx_t, w_t = route_f32(lg, k)
        near = _near_ties(lg, k)
        far = ~near
        if what == "random":
            assert far.sum() >= 0.8 * lg.shape[0], int(far.sum())
        elif k == 2:
            assert far[-4:].all() and far.sum() >= 8, far  # the fp16 / fp32 disagreement rows are decided
        assert torch.equal(idx[far], idx_t[far]), what
        assert torch.equal(w[far].view(torch.int16), w_t[far].view(torch.int16)), what
        # the model's own outcome is one its window explains
        for t in range(lg.shape[0]):
            assert route_f32_explains(lg[t], idx[t].numpy(), w[t].view(torch.int16).numpy(), k), (what, t)
    # exact ties: the lower index first, under the fp32 rule too
    idx, w = kernel_route_f32(crafted, k)
    for t, row in enumerate(crafted.tolist()):
        top = sorted(range(E), key=lambda e: (-row[e], e))[:k]
        if row[top[0]] == row[top[1]]:
            assert idx[t].tolist()[:2] == top[:2], (t, row, idx[t])
    assert idx[-4:, :2].tolist() == [[0, 2]] * 4 or E < 8
    if E >= 8:
        assert kernel_route(crafted[-4:], k)[0][:, :2].tolist() == [[0, 1]] * 4


def test_route_f32_window_is_not_vacuous():
    """On random logits (E 8, top-2) the window refuses what a wrong kernel would write: a weight one fp16 step off, the
    experts of a decided token swapped with the third, and the weights of the fp16 rule (scores rounded to fp16 before
    the top-k and the renormalisation)."""
    E, k = 8, 2
    lg = (torch.randn(512, E, generator=torch.Generator().manual_seed(3)) * 2).half()
    idx, w = kernel_route_f32(lg, k)
    near = _near_ties(lg, k)
    _, w16 = kernel_route(lg, k)
    sc = kernel_scores_f32(lg)
    refused, differ = dict(step=0, swap=0, rule16=0), 0
    for t in np.nonzero(~near)[0][:200]:
        wb = w[t].view(torch.int16).numpy().copy()
        wb[0] += 1
        refused["step"] += not route_f32_explains(lg[t], idx[t].numpy(), wb, k)
        third = int(np.argsort(-sc[t], kind="stable")[k])
        sw = idx[t].numpy().copy()
        sw[k - 1] = third
        refused["swap"] += not route_f32_explains(lg[t], sw, w[t].view(torch.int16).numpy(), k)
        if not torch.equal(w16[t], w[t]):
            differ += 1
            refused["rule16"] += not route_f32_explains(lg[t], idx[t].numpy(), w16[t].view(torch.int16).numpy(), k)
    print(f"\n[route_f32 window] refused of 200 decided tokens: {refused}; fp16-rule weights differing: {differ}")
    assert refused["step"] == 200 and refused["swap"] == 200 and refused["rule16"] == differ > 0, (refused, differ)


@needs_ref
@pytest.mark.parametrize("name", list(sparse.CASES))
def test_port_and_goldens_match_the_unmodified_module(name):
    args, sd, sd_ref, recs, toks = sparse.build_case(name)
    _, _, _, _, plen, ndec = sparse.CASES[name]
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    for dt, tag in ((torch.float16, "fp16"), (torch.float32, "fp32")):
        ref = cases.run_schedule(ref_import.build_reference_model("mixtral_sparse", dict(args), sd_ref, dt), toks, plen, ndec)
        port = cases.run_schedule(sparse.SparsePortModel(args, sd_ref, dtype=dt), toks, plen, ndec)
        gold = torch.from_numpy(g[f"logits_{tag}"])
        if dt == torch.float16:
            assert torch.equal(port, ref)
            assert (ref - gold).abs().max() <= 2 ** -9  # one fp16 ulp of logits < 4: the CPU fp16 GEMM follows the host ISA
        else:
            assert (port - ref).abs().max() <= 4e-6
            assert (ref - gold).abs().max() <= 2e-5


def test_sparse_port_rank_slicing_is_the_rank_sum_of_the_tp1_model():
    """At TP > 1 the port sums the ranks' per-token partial outputs; with fp32 weights the rank sums agree with TP = 1."""
    ref = sparse.port_logits("mixtral_sparse_fp16", dtype=torch.float32, tp=1)
    for tp in (2, 4, 8):
        got = sparse.port_logits("mixtral_sparse_fp16", dtype=torch.float32, tp=tp)
        assert (got - ref).abs().max() <= 2e-5, tp


# ----------------------------------------------------------------------------------------------- checkpoints --------
def _sparse_master(E=4, F=1024, D=64, L=2):
    g = torch.Generator().manual_seed(7)
    sd = {"tok_embeddings.weight": torch.randn(32, D, generator=g).half(), "norm.weight": torch.ones(D).half()}
    for i in range(L):
        p = f"layers.{i}.feed_forward."
        sd[p + "gate.weight"] = torch.randn(E, D, generator=g).half()
        for w in ("w1", "w2", "w3"):
            sd[p + w] = torch.randn(E * F, D, generator=g).half()
        sd[f"layers.{i}.attention.wo.weight"] = torch.randn(D, D, generator=g).half()
    return sd


@needs_ref
@pytest.mark.parametrize("ckpt_tp", [1, 2, 4, 8])
def test_checkpoint_merge_split_round_trip(tmp_path, ckpt_tp):
    mod = ref_import.load("mixtral_sparse")
    E = 4
    sd = _sparse_master(E)
    checkpoint.save_tensor_parallel_shards(sd, str(tmp_path), ckpt_tp)
    keys = [k for k in sd if k.endswith(("feed_forward.w1", "feed_forward.w2", "feed_forward.w3"))]
    # the files hold the module's split of the master
    files = [torch.load(os.path.join(tmp_path, f), weights_only=True)["model"]
             for f in checkpoint.get_tensor_parallel_shards_file_name("consolidated", ckpt_tp)]
    for k in keys:
        want = mod._sparse_expert_split(sd[k], ckpt_tp, E)
        for r in range(ckpt_tp):
            assert torch.equal(files[r]["llma." + k].view(E, -1, sd[k].shape[-1]), want[r])
    for tp in (1, 2, 4, 8):
        ranks = [checkpoint.load_tensor_parallel_state_dict(str(tmp_path), r, tp) for r in range(tp)]
        for k in keys:
            want = mod._sparse_expert_split(sd[k], tp, E)
            for r in range(tp):
                assert torch.equal(ranks[r]["llma." + k].view(E, -1, sd[k].shape[-1]), want[r]), (k, tp, r)
            assert torch.equal(mod._sparse_expert_merge([ranks[r]["llma." + k] for r in range(tp)], E), sd[k])
        # column / row / replicated tensors keep their rules
        assert torch.equal(torch.cat([x["llma.layers.0.attention.wo.weight"] for x in ranks], dim=1),
                           sd["layers.0.attention.wo.weight"])
        assert torch.equal(ranks[-1]["llma.layers.1.feed_forward.gate.weight"], sd["layers.1.feed_forward.gate.weight"])
        if ckpt_tp % tp == 0:
            lazy = checkpoint.LazyMergedStateDict(str(tmp_path), tp - 1, tp)
            for k in keys:
                assert torch.equal(lazy[k], ranks[-1]["llma." + k])


def test_sparse_expert_view_is_the_per_expert_linears():
    E, F, D = 4, 1024, 64
    sd = _sparse_master(E, F, D)
    v = checkpoint.SparseExpertView(sd, E)
    p = "layers.1.feed_forward."
    assert p + "w1" not in v and p + "gate.weight" in v
    for e in range(E):
        q = p + f"experts.{e}."
        assert torch.equal(v[q + "w1.weight"], sd[p + "w1"][e * F:(e + 1) * F])
        assert torch.equal(v[q + "w3.weight"], sd[p + "w3"][e * F:(e + 1) * F])
        assert torch.equal(v[q + "w2.weight"], sd[p + "w2"][e * F:(e + 1) * F].t())  # x @ w2 == F.linear(x, w2.t())
        assert checkpoint.QUANTISED_KEY.search(q + "w2.weight")
    with pytest.raises(ValueError, match="SparseExpertView"):
        checkpoint.recover_quant_records(sd, 4)


def test_model_plugin_has_the_reference_parameter_shapes():
    from llama2_accessory_b200.model import mixtral_sparse_b200 as m
    a = m.ModelArgs(dim=256, hidden_dim=512, n_layers=1, n_heads=2, vocab_size=64, moe={"num_experts": 4,
                                                                                       "num_experts_per_tok": 2})
    model = m.Transformer(a)
    sdk = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    for w in ("w1", "w2", "w3"):
        assert sdk[f"layers.0.feed_forward.{w}"] == (4 * 512, 256)
        prm = getattr(model.layers[0].feed_forward, w)
        assert prm.is_model_parallel
        parts = prm.model_parallel_split(torch.arange(4 * 512 * 2.0).view(-1, 2), 2)
        assert torch.equal(prm.model_parallel_merge(parts), torch.arange(4 * 512 * 2.0).view(-1, 2))
    assert sdk["layers.0.feed_forward.gate.weight"] == (4, 256)
    cfg = model._engine_config("cpu")
    assert cfg.kind == "mixtral" and cfg.sparse_moe


def test_packed_shard_records_sparse_moe(tmp_path):
    c = EngineConfig.from_model_args("mixtral_sparse", dict(sparse.TINY_SPARSE, n_layers=1), bits=4)
    assert c.kind == "mixtral" and c.sparse_moe
    eng = DecodeEngine(c, "cpu").load_random(seed=0)
    checkpoint.save_packed(eng, str(tmp_path))
    eng2 = checkpoint.load_packed(DecodeEngine(c, "cpu"), str(tmp_path))
    assert all(torch.equal(a.qweight, b.qweight) for a, b in zip(eng.layers[0].e_w13, eng2.layers[0].e_w13))
    base = EngineConfig.from_model_args("mixtral", dict(sparse.TINY_SPARSE, n_layers=1), bits=4)
    with pytest.raises(ValueError, match="sparse_moe"):
        checkpoint.load_packed(DecodeEngine(base, "cpu"), str(tmp_path))
    # a shard written before the field existed is a base Mixtral shard
    fn = os.path.join(tmp_path, checkpoint.packed_shard_file_name(0, 1))
    blob = torch.load(fn, weights_only=False)
    del blob["config"]["sparse_moe"]
    torch.save(blob, fn)
    checkpoint.load_packed(DecodeEngine(base, "cpu"), str(tmp_path))
    with pytest.raises(ValueError, match="sparse_moe"):
        checkpoint.load_packed(DecodeEngine(c, "cpu"), str(tmp_path))


# ----------------------------------------------------------------------------------------------- launch traces ------
TRACED = {"b200_gemv", "b200_attn_decode", "b200_embed", "b200_argmax", "b200_advance_pos", "b200_moe_route",
          "b200_moe_expert_ffn", "b200_moe_combine", "b200_prefill_gemm_w4", "b200_prefill_moe_gemm_w4",
          "b200_prefill_rmsnorm", "b200_prefill_rope_kv", "b200_prefill_silu_mul"}


class _Recorder:
    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        if name not in TRACED:
            return getattr(self.real, name)

        def launch(*args):
            self.calls.append((name, args))
            return 0
        return launch


@pytest.fixture()
def recorder(monkeypatch):
    pkg.build()
    rec = _Recorder(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", rec)
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0))
    monkeypatch.setattr(ops, "_f16", lambda t, name: None)
    monkeypatch.setattr(torch.distributed, "all_reduce", lambda t, group=None, op=None: None)
    monkeypatch.setattr(torch.distributed, "all_gather", lambda parts, t, group=None: [p.copy_(t) for p in parts])
    return rec


@pytest.mark.parametrize("tp_rank,tp_world", [(0, 1), (1, 2)])
def test_launch_trace_every_expert_sliced_and_fp32_routes(recorder, tp_rank, tp_world):
    a = dict(sparse.TINY_SPARSE, max_seq_len=320)
    cfg = EngineConfig.from_model_args("mixtral_sparse", a, bits=4, tp_rank=tp_rank, tp_world=tp_world)
    eng = DecodeEngine(cfg, "cpu").load_random(seed=2)
    eng.use_graph = False
    E, D, fl = cfg.num_experts, cfg.dim, cfg.ffn_hidden // tp_world
    assert (eng.E_loc, eng.e_first, eng.F) == (E, 0, fl)
    for lw in eng.layers:
        assert len(lw.e_w13) == len(lw.e_w2) == E
        assert all((p.N, p.K) == (2 * fl, D) for p in lw.e_w13) and all((p.N, p.K) == (D, fl) for p in lw.e_w2)
    assert eng.prefill_tc_supported()
    toks = torch.randint(1, cfg.vocab_size, (1, 40), generator=torch.Generator().manual_seed(1))
    eng.forward_inference(toks[:, :37], 0)          # tensor-core prompt
    eng.forward_inference(toks[:, 37:38], 37)        # decode step
    eng.forward_inference(toks[:, :12].reshape(2, 6), 0)  # GEMV-chunk prompt, two sequences
    calls = recorder.calls
    routes = [a[0]._obj for n, a in calls if n == "b200_moe_route"]
    assert len(routes) == 3 * cfg.n_layers
    assert all(r.scores_f32 == 1 and r.E == E for r in routes)
    ffn = [a[0]._obj for n, a in calls if n == "b200_moe_expert_ffn"]
    assert len(ffn) == 2 * cfg.n_layers
    for f in ffn:
        assert (f.e_first, f.e_count, f.F) == (0, E, fl)
        assert all((f.w13[i].N, f.w13[i].K, f.w2[i].N, f.w2[i].K) == (2 * fl, D, D, fl) for i in range(E))
    grouped = [a for n, a in calls if n == "b200_prefill_moe_gemm_w4"]
    assert len(grouped) == 2 * cfg.n_layers
    assert all(g[1] == 0 and g[2] == E for g in grouped)
    comb = [a for n, a in calls if n == "b200_moe_combine"]
    assert all(c[3] == 0 and c[4] == E for c in comb)


# ----------------------------------------------------------------------------------------------- real library -------
no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box WITHOUT a GPU (the launches must not run)")
VALIDATED = ("b200_gemv", "b200_attn_decode", "b200_embed", "b200_prefill_gemm_w4", "b200_prefill_moe_gemm_w4",
             "b200_prefill_rmsnorm", "b200_prefill_rope_kv", "b200_prefill_silu_mul", "b200_moe_route",
             "b200_moe_expert_ffn", "b200_moe_combine", "b200_argmax", "b200_advance_pos")


class _Validator:
    def __init__(self, real):
        self.real, self.rejected, self.accepted = real, [], {}

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        if name not in VALIDATED:
            return fn

        def call(*args):
            rc = fn(*args)
            if rc < 0:
                self.rejected.append((name, rc, self.real.b200_last_error().decode()))
            else:
                self.accepted[name] = self.accepted.get(name, 0) + 1
            return 0
        return call


@no_gpu
@pytest.mark.parametrize("tp", [1, 2, 4, 8])
def test_c4_width_launches_pass_the_library_checks(monkeypatch, tp):
    """Mixtral-8x7B widths (D 4096, F 14336: F / TP = 14336, 7168, 3584, 1792, all multiples of 128), W4, bs 16, the last
    rank of each TP size: a 2-token prompt, two decode steps and a 40-token tensor-core prompt."""
    pkg.build()
    v = _Validator(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", v)
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0))
    monkeypatch.setattr(ops, "_f16", lambda t, name: None)
    monkeypatch.setattr(torch.distributed, "all_gather", lambda parts, t, group=None: [p.copy_(t) for p in parts])
    monkeypatch.setattr(torch.distributed, "all_reduce", lambda t, group=None, op=None: None)
    args = dict(MIX, n_layers=1, max_seq_len=96, max_batch_size=16)
    eng = DecodeEngine(EngineConfig.from_model_args("mixtral_sparse", args, bits=4, tp_rank=tp - 1, tp_world=tp), "cpu")
    eng.load_random(seed=0)
    eng.use_graph = False
    toks = torch.randint(1, 32000, (16, 4), generator=torch.Generator().manual_seed(1))
    eng.forward_inference(toks[:, :2], 0)
    for j in range(2):
        eng.forward_inference(toks[:, 2 + j:3 + j], 2 + j)
    eng.forward_inference(torch.randint(1, 32000, (1, 40)), 0)
    assert not v.rejected, v.rejected[:4]
    assert all(v.accepted.get(k, 0) > 0 for k in ("b200_moe_route", "b200_moe_expert_ffn", "b200_moe_combine",
                                                  "b200_prefill_moe_gemm_w4"))


def test_refuses_a_slice_that_is_not_whole_128_row_blocks():
    a = dict(sparse.TINY_SPARSE, hidden_dim=1024)
    check_kernel_limits(EngineConfig.from_model_args("mixtral_sparse", a, tp_world=8))
    with pytest.raises(ValueError, match="multiple of 128"):
        check_kernel_limits(EngineConfig.from_model_args("mixtral_sparse", a, tp_world=16))
    with pytest.raises(ValueError, match="multiple of 128"):
        check_kernel_limits(EngineConfig.from_model_args("mixtral_sparse", dict(a, hidden_dim=960), tp_world=1))
    check_kernel_limits(EngineConfig.from_model_args("mixtral", dict(a, hidden_dim=960), tp_world=1))  # base: padded


@no_gpu
def test_library_refuses_a_bad_score_rule():
    pkg.build()
    lib = _cabi.lib()
    r = _cabi.MoeRouteArgs()
    r.T, r.D, r.E, r.topk = 1, 64, 8, 2
    r.resid = r.gamma = r.gate_w = r.xn_out = r.slot_weight = r.slot_expert = 0x1000  # never dereferenced: refused first
    for bad in (2, -1):
        r.scores_f32 = bad
        assert lib.b200_moe_route(C.byref(r), None) < 0
        assert b"scores_f32" in lib.b200_last_error()
