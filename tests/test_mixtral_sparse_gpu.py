"""GPU: `mixtral_sparse` models on the H100 -- the fp32 router rule of moe_route_kernel at real widths, and the engine with
every expert sliced over the tensor-parallel ranks.

  * Router (D 4096, E 8, top-2, T up to 256).  A float64 logit farther than R from an fp16 rounding midpoint has one
    possible fp16 value, the others two (R: the running-error bound of the kernel's lane chains and warp tree,
    oracle.numerics.logit_window).  For some choice of those, scores_f32 = 1 must give the experts and weights of
    oracle.numerics.kernel_route_f32 (moe_route_kernel<true> line by line) bit for bit, or differ only inside the window
    the device expf allows: experts exchanged only where their fp32 scores lie that close, a weight's other fp16 rounding
    only where score / sum lies that close to a midpoint (route_check_f32).  With scores_f32 = 0 the same launch must
    satisfy the CPU model of the fp16 rule (route_check, as tests/test_gemv_batched_moe_gpu.py checks it).
  * The engine against the goldens of the unmodified module and against the port (oracle/sparse.py), with the parity rule
    of tests/test_model_parity_gpu.py: GEMV-chunk prompts, tensor-core prompts, a continuation prompt, decode eager and
    from a graph.  Against the port, the port takes the engine's routes (force_routes); every route that differs from the
    port's own is a near-tie of its fp32 scores.
  * Base against sliced at TP = 1: the two engines share every kernel, so with a router whose top-2 are exact ties in
    pairs (weights exactly 0.5 under both score rules) the logits are equal bit for bit.
  * Simulated TP 2 / 4: one DecodeEngine per rank in its own thread, in-process stand-ins for all_reduce / all_gather
    (the fp32 rank-order sum rounded once, as oracle/llama_port.py models NCCL), against the TP = 1 engine and the port.
  * build_engine_from_pretrained on a mixtral_sparse folder (fake-quantised W4, checkpoint TP 2) at TP 1 and simulated
    TP 2, and a packed-shard round trip.
"""
import json
import os
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import _cabi, checkpoint, ops  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig  # noqa: E402
from oracle import omniquant, sparse, weights  # noqa: E402
from oracle.numerics import route_check, route_check_f32  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RULE_FACTOR = 1.5  # tests/test_model_parity_gpu.py
# a routing flip against the port counts as a near-tie when the port's fp32 scores of the exchanged experts lie within this
# many fp16 ulps (the screen of tests/test_prefill_moe_gpu.py)
FLIP_ULPS = 4


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _ulp16(x):
    """Spacing of fp16 at |x| (float64 array)."""
    a = np.maximum(np.abs(x), 2.0 ** -14)
    return 2.0 ** (np.floor(np.log2(a)) - 10)


# --------------------------------------------------------------------------------------------------- router ---------
@pytest.mark.parametrize("T", [1, 16, 256])
def test_fp32_router_at_real_widths(T):
    D, E, k = 4096, 8, 2
    g = torch.Generator(device="cuda").manual_seed(T)
    f16 = dict(dtype=torch.float16, device="cuda")
    resid = torch.randn(T, D, generator=g, device="cuda").half()
    delta = (torch.randn(T, D, generator=g, device="cuda") * 0.5).half()
    gamma = (1 + 0.1 * torch.randn(D, generator=g, device="cuda")).half()
    gate = ((torch.rand(E, D, generator=g, device="cuda") * 2 - 1) * 4 / D ** 0.5).half()
    out = {}
    for rule in (1, 0):
        h_out, xn = torch.empty(T, D, **f16), torch.empty(T, D, **f16)
        sw, se = torch.empty(T * k, **f16), torch.empty(T * k, dtype=torch.int32, device="cuda")
        ops.moe_route(T=T, D=D, E=E, topk=k, resid=resid, delta=delta, h_out=h_out, gamma=gamma, eps=1e-5, gate_w=gate,
                      xn_out=xn, slot_weight=sw, slot_expert=se, scores_f32=rule)
        torch.cuda.synchronize()
        out[rule] = (xn.cpu(), sw.view(T, k).cpu(), se.view(T, k).cpu().long())
    xn = out[1][0]
    assert torch.equal(xn, out[0][0])
    _, sw32, se32 = out[1]
    m32, w32, s32 = route_check_f32(xn.cuda(), gate, sw32.cuda(), se32.cuda(), k)
    assert s32 == 0 and m32 + w32 == T and m32 >= 0.9 * T, (m32, w32, s32)
    # scores_f32 = 0: today's CPU model of the fp16 rule
    matched, window, skipped = route_check(xn.cuda(), gate, out[0][1].cuda(), out[0][2].cuda(), k)
    assert matched + window == T and skipped == 0
    print(f"\n[router T={T}] fp32 rule: {m32} bit for bit, {w32} in the expf window; fp16 rule: {matched} bit for bit, "
          f"{window} in the expf window")


# --------------------------------------------------------------------------------------------------- engine ---------
def _rule(got, ref16, ref32, what):
    e16, e32 = np.abs(got - ref16).max(), np.abs(got - ref32).max()
    floor = np.abs(ref16 - ref32).max()
    rms32 = float(np.sqrt(np.mean((got - ref32) ** 2)))
    rms_floor = float(np.sqrt(np.mean((ref16 - ref32) ** 2)))
    print(f"\n[{what}] |eng-ref16|={e16:.3e} |eng-ref32|={e32:.3e} |ref16-ref32|={floor:.3e}")
    assert np.isfinite(got).all()
    assert (e16 <= 1e-3 or e32 <= RULE_FACTOR * floor
            or (rms32 <= 1.02 * rms_floor and e32 <= 1.25 * floor)), (what, e16, e32, floor, rms32, rms_floor)
    top2 = np.sort(ref32, axis=-1)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 4 * floor
    assert (got.argmax(-1)[clear] == ref32.argmax(-1)[clear]).all(), what


def _engine(args, sd, recs, bits, tp_rank=0, tp_world=1, use_graph=False):
    cfg = EngineConfig.from_model_args("mixtral_sparse", args, bits=bits or 16, tp_rank=tp_rank, tp_world=tp_world)
    eng = DecodeEngine(cfg, "cuda")
    eng.use_graph = use_graph
    return eng.load_master_state_dict(sd, quant_records=recs if bits else None)


def _run(eng, toks, plen, ndec):
    toks = toks.cuda()
    outs = [eng.forward_inference(toks[:, :plen], 0).float().cpu().clone()]
    for j in range(ndec):
        outs.append(eng.forward_inference(toks[:, plen + j:plen + j + 1], plen + j).float().cpu().clone())
    return torch.stack(outs).numpy()


@pytest.mark.parametrize("name", list(sparse.CASES))
def test_engine_matches_the_golden_logits(name):
    """GEMV-chunk prompt (5 / 6 tokens) and decode steps, eager and from CUDA graphs."""
    args, sd, sd_ref, recs, toks = sparse.build_case(name)
    _, bits, _, _, plen, ndec = sparse.CASES[name]
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    eager = _run(_engine(args, sd, recs, bits), toks, plen, ndec)
    _rule(eager, g["logits_fp16"], g["logits_fp32"], name)
    graph = _run(_engine(args, sd, recs, bits, use_graph=True), toks, plen, ndec)
    assert np.array_equal(eager, graph)


@pytest.mark.parametrize("plen", [40, 300])
def test_engine_tensor_core_and_continuation_prompts_match_the_port(monkeypatch, plen):
    """A tensor-core prompt (40 tokens; 300 = two 256-token chunks), a 37-token continuation prompt at start_pos = plen
    (tensor cores again), two decode steps; bs 2, the W4 case's weights.  The port runs with the engine's routes; a route
    that differs from the port's own choice must be a near-tie."""
    args, sd, sd_ref, recs, _ = sparse.build_case("mixtral_sparse_w4")
    args = dict(args, max_seq_len=384)
    toks = weights.synthetic_tokens(2, plen + 39, args["vocab_size"], seed=plen)
    sched = [(0, plen), (plen, plen + 37), (plen + 37, plen + 38), (plen + 38, plen + 39)]
    eng = _engine(args, sd, recs, 4)
    assert eng.prefill_tc_supported()
    routes = _capture_routes(monkeypatch, [eng])
    tk = toks.cuda()
    got = np.stack([eng.forward_inference(tk[:, a:b], a).float().cpu().numpy() for a, b in sched])
    ref16, ref32, fl = _forced_port_pair(args, sd_ref, toks, sched, routes(eng))
    _rule(got, ref16, ref32, f"tensor-core prompt {plen} + continuation 37 + decode 2 ({fl} near-tie flips)")


def test_base_and_sliced_engines_agree_bit_for_bit_at_tp1():
    """Router rows equal in pairs (0 = 1, 2 = 3): every token's top-2 is an exact tie, weight 0.5 under both score rules, so
    the base engine (whole experts, fp16 rule) and the sliced one (fp32 rule) run the same kernels on the same data."""
    name = "mixtral_sparse_w4"
    args, sd, sd_ref, recs, toks = sparse.build_case(name)
    base = weights.mixtral_state_dict(args)
    E = args["moe"]["num_experts"]
    for i in range(args["n_layers"]):
        gk = f"layers.{i}.feed_forward.gate.weight"
        gw = base[gk].clone()
        gw[1], gw[3] = gw[0], gw[2]
        base[gk] = gw
    sp = sparse.to_sparse(base, E)
    args = dict(args, max_seq_len=128)
    toks = weights.synthetic_tokens(2, 50, args["vocab_size"], seed=5)
    sched = [(0, 40), (40, 46), (46, 47), (47, 48)]  # tensor-core prompt, GEMV-chunk continuation, decode
    res = []
    for kind, w in (("mixtral", base), ("mixtral_sparse", sp)):
        eng = DecodeEngine(EngineConfig.from_model_args(kind, args, bits=4), "cuda")
        eng.use_graph = False
        eng.load_master_state_dict(w, quant_records=recs)
        tk = toks.cuda()
        res.append(np.stack([eng.forward_inference(tk[:, a:b], a).float().cpu().numpy() for a, b in sched]))
    assert np.array_equal(res[0], res[1])


# ------------------------------------------------------------------------------------- simulated tensor parallel ----
class _Ranks:
    """tp engines on one device, each driven from its own thread.  Launches go through the library one at a time (a lock);
    all_reduce / all_gather exchange device tensors at a barrier, all_reduce being the fp32 rank-order sum rounded once."""

    def __init__(self, tp):
        self.tp, self.lock = tp, threading.Lock()
        self.bar = threading.Barrier(tp, timeout=300)
        self.local, self.slots = threading.local(), [None] * tp

    def _exchange(self, t):
        torch.cuda.synchronize()
        self.slots[self.local.rank] = t.detach().clone()
        torch.cuda.synchronize()
        self.bar.wait()
        vals = list(self.slots)
        self.bar.wait()
        return vals

    def all_gather(self, parts, t, group=None, **kw):
        for p, v in zip(parts, self._exchange(t)):
            p.copy_(v)

    def all_reduce(self, t, op=None, group=None, **kw):
        vals = self._exchange(t)
        acc = vals[0].float()
        for v in vals[1:]:
            acc = acc + v.float()
        t.copy_(acc.to(t.dtype))

    def run(self, fn):
        out, errs = [None] * self.tp, []

        def body(r):
            self.local.rank = r
            try:
                out[r] = fn(r)
            except BaseException as e:  # noqa: BLE001 -- re-raised below
                errs.append(e)
                self.bar.abort()
        ths = [threading.Thread(target=body, args=(r,)) for r in range(self.tp)]
        for t in ths:
            t.start()
        for t in ths:
            t.join(timeout=900)
        assert not any(t.is_alive() for t in ths)
        if errs:
            raise errs[0]
        return out


class _SerialLib:
    def __init__(self, real, lock):
        self.real, self.lock = real, lock

    def __getattr__(self, name):
        fn = getattr(self.real, name)

        def call(*args):
            with self.lock:
                return fn(*args)
        return call


@pytest.fixture()
def ranks(monkeypatch):
    import torch.distributed as dist

    def make(tp):
        rk = _Ranks(tp)
        monkeypatch.setattr(_cabi, "_lib", _SerialLib(_cabi.lib(), rk.lock))
        monkeypatch.setattr(dist, "all_gather", rk.all_gather)
        monkeypatch.setattr(dist, "all_reduce", rk.all_reduce)
        return rk
    return make


TP_ARGS = dict(sparse.TINY_SPARSE, n_kv_heads=4, max_seq_len=128)  # 4 kv heads: TP 4 keeps one per rank


def _tp_run(rk, engines, toks, sched):
    def one(r):
        tk = toks.cuda()
        return np.stack([engines[r].forward_inference(tk[:, a:b], a).float().cpu().numpy() for a, b in sched])
    return rk.run(one)


def _capture_routes(monkeypatch, engines):
    """Record every moe_route launch of `engines`: -> fn(engine) = {(start_pos, layer): slot_expert int64 [B * S, k]}, the
    keys and row order the port's force_routes takes (chunks of one call are concatenated in launch order)."""
    real = ops.moe_route
    got, sp = {id(e): {} for e in engines}, {}
    gates = {id(lw.gate): (e, i) for e in engines for i, lw in enumerate(e.layers)}

    def route(**kw):
        real(**kw)
        hit = gates.get(id(kw["gate_w"]))
        if hit is not None:
            e, i = hit
            T, k = kw["T"], kw["topk"]
            torch.cuda.synchronize()
            got[id(e)].setdefault((sp[id(e)], i), []).append(kw["slot_expert"][:T * k].view(T, k).cpu().long())
    monkeypatch.setattr(ops, "moe_route", route)
    for e in engines:
        def fwd(tokens, start_pos, _f=e.forward_inference, _e=e):
            sp[id(_e)] = start_pos
            return _f(tokens, start_pos)
        e.forward_inference = fwd
    return lambda e: {key: torch.cat(v) for key, v in got[id(e)].items()}


def _forced_port_pair(args, sd_ref, toks, sched, routes, tp=1):
    """The port in fp16 and fp32 with the engine's routes; every route that differs from the fp32 port's own choice must be
    a near-tie of its fp32 scores.  -> (ref16, ref32, number of flipped tokens)."""
    out, flips = {}, 0
    for dt in (torch.float16, torch.float32):
        m = sparse.SparsePortModel(args, sd_ref, dtype=dt, tp=tp)
        m.force_routes, m.record = routes, []
        out[dt] = np.stack([m.forward_inference(toks[:, a:b], a).float().numpy() for a, b in sched])
        if dt != torch.float32:
            continue
        for rec in m.record:
            for own, used, sc in zip(rec["own"], rec["routes"], rec["scores"]):
                k = own.shape[-1]
                own, used, sc = own.reshape(-1, k), used.reshape(-1, k), sc.reshape(own.numel() // k, -1).double()
                for t in range(own.shape[0]):
                    o, u = set(own[t].tolist()), set(used[t].tolist())
                    if o == u:
                        continue
                    so, su = max(float(sc[t, e]) for e in o - u), min(float(sc[t, e]) for e in u - o)
                    assert so - su <= FLIP_ULPS * _ulp16(np.array(so)), (rec["start_pos"], t, o, u, so, su)
                    flips += 1
    return out[torch.float16], out[torch.float32], flips


@pytest.mark.timeout(900)
@pytest.mark.parametrize("tp", [2, 4])
def test_simulated_tensor_parallel_matches_tp1_and_the_port(ranks, monkeypatch, tp):
    """Every rank returns the same logits; the TP = tp ranks and the TP = 1 engine each meet the port rule against the port
    (with the same expert slicing) forced to their own routes, where any route that differs from the port's own choice is
    a near-tie; where the two engines routed alike everywhere, their logits agree to 4e-3."""
    base = weights.mixtral_state_dict(TP_ARGS)
    base_ref, recs = omniquant.fake_quantize_state_dict(base, 4, 0)
    E = TP_ARGS["moe"]["num_experts"]
    sd, sd_ref = sparse.to_sparse(base, E), sparse.to_sparse(base_ref, E)
    toks = weights.synthetic_tokens(2, 48, TP_ARGS["vocab_size"], seed=11)
    sched = [(0, 6), (6, 46), (46, 47), (47, 48)]  # GEMV-chunk prompt, tensor-core continuation, decode
    rk = ranks(tp)
    one = _engine(TP_ARGS, sd, recs, 4)
    engines = [_engine(TP_ARGS, sd, recs, 4, tp_rank=r, tp_world=tp) for r in range(tp)]
    for e in engines:
        assert e.E_loc == E and e.e_first == 0 and e.F == TP_ARGS["hidden_dim"] // tp
    routes = _capture_routes(monkeypatch, [one] + engines)
    tk = toks.cuda()
    tp1 = np.stack([one.forward_inference(tk[:, a:b], a).float().cpu().numpy() for a, b in sched])
    got = _tp_run(rk, engines, toks, sched)
    assert all(np.array_equal(got[0], g) for g in got[1:])
    r1, rt = routes(one), routes(engines[0])
    assert all(torch.equal(rt[key], routes(e)[key]) for e in engines[1:] for key in rt)  # the ranks route alike
    ref16, ref32, fl = _forced_port_pair(TP_ARGS, sd_ref, toks, sched, rt, tp=tp)
    _rule(got[0], ref16, ref32, f"simulated TP {tp} vs port (TP {tp} slices, engine routes; {fl} near-tie flips)")
    ref16, ref32, fl1 = _forced_port_pair(TP_ARGS, sd_ref, toks, sched, r1)
    _rule(tp1, ref16, ref32, f"TP 1 vs port (engine routes; {fl1} near-tie flips)")
    same = r1.keys() == rt.keys() and all(torch.equal(r1[key], rt[key]) for key in r1)
    err = np.abs(got[0] - tp1).max()
    print(f"[simulated TP {tp}] |tp{tp} - tp1|max = {err:.3e}, routes {'equal' if same else 'differ at near-ties'}")
    if same:
        assert err <= 4e-3


@pytest.mark.timeout(900)
def test_build_engine_from_pretrained_sparse_folder_and_packed_round_trip(ranks, tmp_path):
    """A reference-format mixtral_sparse folder (checkpoint TP 2, OmniQuant fake-quantised W4): at TP 1 the recovered
    integers reproduce the engine loaded from the master weights and their records bit for bit; at simulated TP 2 every
    rank serves it and agrees with the TP = 1 engine; a packed shard written and read back gives the same logits."""
    args, sd, sd_ref, recs, toks = sparse.build_case("mixtral_sparse_w4")
    _, _, _, _, plen, ndec = sparse.CASES["mixtral_sparse_w4"]
    path = str(tmp_path / "ckpt")
    checkpoint.save_tensor_parallel_shards(sd_ref, path, 2)
    cfg = {k: v for k, v in args.items() if k not in ("max_seq_len", "max_batch_size")}
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(cfg, f)
    with open(os.path.join(path, "meta.json"), "w") as f:
        json.dump({"llama_type": "mixtral_sparse"}, f)
    kw = dict(bits=4, fake_quantised=True, max_seq_len=args["max_seq_len"], max_batch_size=args["max_batch_size"])
    eng, meta = checkpoint.build_engine_from_pretrained(path, **kw)
    assert meta["llama_type"] == "mixtral_sparse" and eng.cfg.sparse_moe
    eng.use_graph = False
    got = _run(eng, toks, plen, ndec)
    want = _run(_engine(args, sd, recs, 4), toks, plen, ndec)
    assert np.array_equal(got, want)
    g = np.load(os.path.join(GOLD, "mixtral_sparse_w4.npz"))
    _rule(got, g["logits_fp16"], g["logits_fp32"], "build_engine_from_pretrained, TP 1")
    checkpoint.save_packed(eng, str(tmp_path / "packed"))
    back = checkpoint.load_packed(DecodeEngine(eng.cfg, "cuda"), str(tmp_path / "packed"))
    back.use_graph = False
    assert np.array_equal(_run(back, toks, plen, ndec), got)
    rk = ranks(2)
    engines = []
    for r in range(2):
        e, _ = checkpoint.build_engine_from_pretrained(path, tp_rank=r, tp_world=2, **kw)
        e.use_graph = False
        engines.append(e)
    sched = [(0, plen)] + [(plen + j, plen + j + 1) for j in range(ndec)]
    tp2 = _tp_run(rk, engines, toks, sched)
    assert np.array_equal(tp2[0], tp2[1])
    err = np.abs(tp2[0] - got).max()
    print(f"\n[from_pretrained TP 2] |tp2 - tp1|max = {err:.3e}")
    assert err <= 4e-3
    _rule(tp2[0], g["logits_fp16"], g["logits_fp32"], "build_engine_from_pretrained, simulated TP 2")
