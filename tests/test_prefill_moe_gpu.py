"""GPU: the grouped MoE form of the wgmma W4A16 prompt GEMM (csrc/prefill.cu b200_prefill_moe_gemm_w4) and the Mixtral
prompt path built on it (engine._prefill_chunk_tc).

Grouped GEMM:
  - against the dense GEMM: every row the grouped launch writes must equal, bit for bit, b200_prefill_gemm_w4 on that
    expert over the same gathered rows in the same (slot) order; rows of slots routed elsewhere keep a NaN sentinel;
  - against float64 at Mixtral-8x7B widths (D 4096, F 14336, 8 experts, top-2): the elementwise bound and exact fraction
    of test_prefill_gpu (ulp16(ref) + 2^-18 |x| . |w_hat|^T);
  - repeated launches and a launch on a side stream give the same bits.
Engine: the CPU port (bit-pinned to the unmodified reference) in fp32 / fp16 with the asserted rule of
test_prefill_gpu (e16 <= 1e-3 or e32 <= 1.5 floor), prompts from position 0 and continuation prompts, tensor-core path
on and off.  No bitwise TC-vs-GEMV comparison: a routing tie between the two paths' fp16 router inputs can flip an expert.
"""
import contextlib
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import kvlayout, ops, quant  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig  # noqa: E402
from oracle import cases, omniquant, weights  # noqa: E402
from oracle.llama_port import PortModel  # noqa: E402
from oracle.numerics import route_check  # noqa: E402

DEV = "cuda"
C_ACC = 2.0 ** -18  # fp32 tensor-core accumulation allowance of test_prefill_gpu, relative to |x| . |w_hat|^T
# a routing flip against the fp32 port counts as a near-tie when the fp32 scores of the exchanged experts lie within this
# many fp16 ulps.  A heuristic, not a derived bound: it only screens out a flip at a clear margin.  The asserted evidence
# that a flip is legitimate is the forced-routing rule, route_check of the engine's own launch, and the residual leaving
# the fp16 / fp32 band first at a flipped token (test_mixtral_continuation_prompt_matches_port)
FLIP_ULPS = 4
# the engine's residual after a block leaves the port's band when it is further than this factor from the fp32 port than
# the fp16 port is (the port rule's factor), with differences below BAND_ABS (a few fp16 ulps of O(1) values) ignored
BAND_FACTOR, BAND_ABS = 1.5, 2.0 ** -9


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _nan16(*shape, pattern=0x7E5A):
    return torch.full(shape, pattern, dtype=torch.int16, device=DEV).view(torch.float16)


def _ulp16(a):
    e = torch.floor(torch.log2(a.double().abs().clamp_min(2.0 ** -24)))
    return torch.exp2(e.clamp_min(-14) - 10)


def _experts(E, N, K, seed):
    """E random per-channel W4 experts generated in packed form on the device."""
    return [quant.random_packed(4, N, K, 0, DEV, seed + i) for i in range(E)]


def _w_hat(pl):
    """fp16(fp16(q - z) * s) of a packed per-channel W4 linear, on the device."""
    q = quant.unpack_quantized(pl).to(DEV)
    sz = pl.scales.view(torch.float16).reshape(pl.N, 2)
    return quant.dequantize(q, sz[:, :1].contiguous(), sz[:, 1:].contiguous(), pl.K)


def _grouped(pls, x, slot_e, src_div, e_first):
    n = slot_e.numel()
    out = _nan16(n, pls[0].N)
    ops.prefill_moe_gemm_w4(pls, x, out, slot_expert=slot_e, n_slots=n, src_div=src_div, e_first=e_first)
    torch.cuda.synchronize()
    return out


def _check_against_dense(pls, x, slot_e, src_div, e_first):
    out = _grouped(pls, x, slot_e, src_div, e_first)
    se = slot_e.cpu()
    local = torch.zeros(se.numel(), dtype=torch.bool)
    for i, pl in enumerate(pls):
        sl = torch.nonzero(se == e_first + i).flatten()
        local[sl] = True
        if sl.numel() == 0:
            continue
        xg = x[(sl // src_div).to(DEV)].contiguous()
        ref = _nan16(sl.numel(), pl.N)
        ops.prefill_gemm_w4(pl, xg, ref, sl.numel())
        torch.cuda.synchronize()
        got = out[sl.to(DEV)]
        assert torch.equal(got.view(torch.int16), ref.view(torch.int16)), (i, sl.numel())
    rest = out[torch.nonzero(~local).flatten().to(DEV)]
    assert bool((rest.view(torch.int16) == 0x7E5A).all())  # rows of other experts are not written
    return out


def _topk_routing(T, E, k, g):
    return torch.rand(T, E, generator=g).topk(k, dim=1).indices.reshape(-1).int()


def _counts_routing(counts, g):
    ids = torch.cat([torch.full((c,), e, dtype=torch.int32) for e, c in enumerate(counts)])
    return ids[torch.randperm(ids.numel(), generator=g)]


ROUTINGS = {
    # name: (T tokens, E, top-k (= src_div), e_first, e_count, slot_expert builder)
    "uniform": (300, 8, 2, 0, 8, lambda g: _topk_routing(300, 8, 2, g)),
    "two_experts": (200, 8, 2, 0, 8, lambda g: torch.tensor([1, 5], dtype=torch.int32).repeat(200)),
    "empty_experts": (150, 8, 2, 0, 8, lambda g: _topk_routing(150, 3, 2, g)),
    "counts_1_31_32_33_255_256_512": (1120, 7, 1, 0, 7, lambda g: _counts_routing([1, 31, 32, 33, 255, 256, 512], g)),
    "T1": (1, 8, 2, 0, 8, lambda g: _topk_routing(1, 8, 2, g)),
    "T32": (32, 8, 2, 0, 8, lambda g: _topk_routing(32, 8, 2, g)),
    "T33": (33, 8, 2, 0, 8, lambda g: _topk_routing(33, 8, 2, g)),
    "T255": (255, 8, 2, 0, 8, lambda g: _topk_routing(255, 8, 2, g)),
    "T256": (256, 8, 2, 0, 8, lambda g: _topk_routing(256, 8, 2, g)),
    # rank 1 of TP = 4: local experts 2, 3; the slots of the other ranks' experts are left alone
    "tp4_rank1": (256, 8, 2, 2, 2, lambda g: _topk_routing(256, 8, 2, g)),
}


@pytest.mark.timeout(300)
@pytest.mark.parametrize("N,K", [(256, 512), (384, 1024)])
@pytest.mark.parametrize("name", list(ROUTINGS))
def test_grouped_gemm_rows_equal_the_dense_gemm_on_gathered_rows(name, N, K):
    T, E, k, e_first, e_count, route = ROUTINGS[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)) + N)
    slot_e = route(g).to(DEV)
    assert slot_e.numel() == T * k
    pls = _experts(e_count, N, K, seed=N + K)
    x = torch.randn(T, K, generator=torch.Generator(device=DEV).manual_seed(T), device=DEV).half()
    out = _check_against_dense(pls, x, slot_e, k, e_first)
    assert torch.isfinite(out[(slot_e >= e_first) & (slot_e < e_first + e_count)]).all()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("proj", ["w13", "w2"])
def test_grouped_gemm_matches_float64_at_mixtral_widths(proj):
    D, F, E, k, T = 4096, 14336, 8, 2, 256
    N, K, src_div = (2 * F, D, k) if proj == "w13" else (D, F, 1)
    g = torch.Generator().manual_seed(17)
    slot_e = _topk_routing(T, E, k, g).to(DEV)
    rows = T if proj == "w13" else T * k
    x = torch.randn(rows, K, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV).half()
    pls = _experts(E, N, K, seed=40 if proj == "w13" else 80)
    out = _grouped(pls, x, slot_e, src_div, 0)
    worst, c_seen, min_exact = 0.0, 0.0, 1.0
    se = slot_e.cpu()
    for i, pl in enumerate(pls):
        sl = torch.nonzero(se == i).flatten()
        if sl.numel() == 0:
            continue
        wd = _w_hat(pl).double()
        xd = x[(sl // src_div).to(DEV)].double()
        ref = xd @ wd.T
        mag = xd.abs() @ wd.abs().T
        got = out[sl.to(DEV)].double()
        err = (got - ref).abs()
        ulp = _ulp16(ref)
        worst = max(worst, float((err / (ulp + C_ACC * mag)).max()))
        c_seen = max(c_seen, float(((err - ulp).clamp_min(0) / mag.clamp_min(1e-30)).max()))
        exact = float(((got.half() + 0.0).view(torch.int16) == (ref.half() + 0.0).view(torch.int16)).double().mean())
        min_exact = min(min_exact, exact)
        assert torch.isfinite(got).all()
        del wd, ref, mag
    print(f"\n[grouped {proj} {N}x{K} E={E} top-{k} T={T}] max err/tol={worst:.3f} "
          f"implied C=2^{math.log2(max(c_seen, 1e-30)):.1f} min exact={min_exact:.4f}")
    assert worst <= 1.0, (worst, c_seen)
    assert min_exact >= 1.0 - 2.0 ** -10 * math.sqrt(K), min_exact


@pytest.mark.timeout(180)
def test_grouped_gemm_is_deterministic_across_launches_and_streams():
    N, K, E, k = 512, 1024, 8, 2
    pls = _experts(E, N, K, seed=5)
    g = torch.Generator().manual_seed(5)
    cases_ = [(T, _topk_routing(T, E, k, g).to(DEV)) for T in (33, 256, 7, 161)]
    xs = [torch.randn(T, K, generator=torch.Generator(device=DEV).manual_seed(T), device=DEV).half() for T, _ in cases_]
    base = [_grouped(pls, x, se, k, 0) for x, (T, se) in zip(xs, cases_)]
    again = [_grouped(pls, x, se, k, 0) for x, (T, se) in zip(xs, cases_)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        outs = [_nan16(se.numel(), N) for _, se in cases_]
        for x, o, (T, se) in zip(xs, outs, cases_):
            ops.prefill_moe_gemm_w4(pls, x, o, slot_expert=se, n_slots=se.numel(), src_div=k, e_first=0)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for a, b, c in zip(base, again, outs):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
        assert torch.equal(a.view(torch.int16), c.view(torch.int16))


@pytest.mark.timeout(180)
def test_grouped_gemm_op_checks_its_tensors():
    N, K, n = 256, 512, 64
    pls = _experts(2, N, K, seed=1)
    x, out = torch.zeros(n // 2, K, dtype=torch.float16, device=DEV), _nan16(n, N)
    se = torch.zeros(n, dtype=torch.int32, device=DEV)
    call = lambda **kw: ops.prefill_moe_gemm_w4(kw.get("pls", pls), kw.get("x", x), kw.get("out", out),  # noqa: E731
                                                slot_expert=kw.get("se", se), n_slots=n, src_div=2, e_first=0)
    bad = [lambda: call(x=x[:-1]), lambda: call(x=x.float()), lambda: call(x=x.cpu()), lambda: call(out=out[:-1]),
           lambda: call(se=se.long()), lambda: call(se=se[:-1]), lambda: call(se=se.cpu()), lambda: call(pls=[])]
    n0 = ops.launch_count
    for f in bad:
        with pytest.raises(ValueError):
            f()
    assert ops.launch_count == n0
    call()
    torch.cuda.synchronize()
    assert ops.launch_count == n0 + 1 and torch.isfinite(out).all()


# ------------------------------------------------------------------------------------------------- the engine ---------
def _tiny_mixtral(max_seq_len=640):
    args = dict(cases.TINY_MIXTRAL, max_seq_len=max_seq_len)
    sd = weights.mixtral_state_dict(args, seed=0)
    sd_ref, recs = omniquant.fake_quantize_state_dict(sd, 4, 0)
    return args, sd, sd_ref, recs


def _engine(args, sd, recs, tc, use_graph=True):
    eng = DecodeEngine(EngineConfig.from_model_args("mixtral", args, bits=4, group_size=0), DEV)
    eng.use_prefill_tc = tc
    eng.use_graph = use_graph
    eng.load_master_state_dict(sd, quant_records=recs)
    assert eng.prefill_tc_supported() == tc
    return eng


def _run(eng, toks, plen, ndec):
    """cases.run_schedule for the engine: a decode step's logits are a view of the captured graph's output buffer."""
    outs = [eng.forward_inference(toks[:, :plen], 0).float().cpu().clone()]
    for j in range(ndec):
        outs.append(eng.forward_inference(toks[:, plen + j:plen + j + 1], plen + j).float().cpu().clone())
    return torch.stack(outs).numpy()


def _rule(label, got, ref16, ref32, asserted=True):
    e32, e16 = np.abs(got - ref32).max(), np.abs(got - ref16).max()
    floor = np.abs(ref16 - ref32).max()
    print(f"\n[{label}] |eng-ref16|={e16:.3e} |eng-ref32|={e32:.3e} floor={floor:.3e}")
    from conftest import record_parity
    record_parity(label, e16=e16, e32=e32, floor=floor, strict_pass=bool(e16 <= 1e-3 or e32 <= floor),
                  rule_pass=bool(e16 <= 1e-3 or e32 <= 1.5 * floor), source="oracle port fp16 / fp32")
    assert np.isfinite(got).all()
    if asserted:
        assert e16 <= 1e-3 or e32 <= 1.5 * floor, (label, e16, e32, floor)
    return bool(e16 <= 1e-3 or e32 <= 1.5 * floor)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("plen", [33, 64, 255, 256, 257, 300, 513])
def test_mixtral_prompt_through_grouped_gemm_matches_port(plen):
    args, sd, sd_ref, recs = _tiny_mixtral()
    ndec = 3
    toks = weights.synthetic_tokens(2, plen + ndec, args["vocab_size"], seed=7)
    ref32 = cases.run_schedule(PortModel("mixtral", args, sd_ref, dtype=torch.float32), toks, plen, ndec).numpy()
    ref16 = cases.run_schedule(PortModel("mixtral", args, sd_ref, dtype=torch.float16), toks, plen, ndec).numpy()
    for tc in (True, False):
        got = _run(_engine(args, sd, recs, tc), toks.cuda(), plen, ndec)
        _rule(f"tiny_mixtral_w4_prefill{plen}_{'wgmma' if tc else 'gemv_chunks'}", got, ref16, ref32)


def _schedule(model, toks, p0, p1, ndec):
    """p0-token prompt, p1-token prompt continuing at p0, ndec decode steps -> (logits, canonical K/V per layer after the
    prompts)."""
    outs = [model.forward_inference(toks[:, :p0], 0).float().cpu().clone(),
            model.forward_inference(toks[:, p0:p0 + p1], p0).float().cpu().clone()]
    if isinstance(model, PortModel):
        kv = [(k.permute(0, 2, 1, 3).double(), v.permute(0, 2, 1, 3).double()) for k, v in zip(model.k_cache, model.v_cache)]
    else:
        kv = [(kvlayout.k_from_engine(model.kcache[i]).double().cpu(), kvlayout.v_from_engine(model.vtcache[i]).double().cpu())
              for i in range(model.kcache.shape[0])]
    for j in range(ndec):
        s = p0 + p1 + j
        outs.append(model.forward_inference(toks[:, s:s + 1], s).float().cpu().clone())
    return torch.stack(outs).numpy(), kv


def _locate_excess(label, calls, got, ref16, ref32, rr, port, n_layers):
    """Where an engine run that misses the port rule parts from the port: the rule's numbers per call (prompt,
    continuation, decode steps), then the first token, in the order the engine computes them (call, position, layer),
    whose residual after a block leaves the port's fp16 / fp32 band.  Asserts that the engine and the fp32 port chose
    different experts for that token at that layer."""
    for c, (sp, n) in enumerate(calls):
        e32, e16 = np.abs(got[c] - ref32[c]).max(), np.abs(got[c] - ref16[c]).max()
        print(f"[{label}] call start {sp} length {n}: |eng-ref32| {e32:.3e} |eng-ref16| {e16:.3e} "
              f"floor {np.abs(ref16[c] - ref32[c]).max():.3e}")
    rec32, rec16 = port[torch.float32].record, port[torch.float16].record
    first = None
    for c, (sp, n) in enumerate(calls):
        for o in range(n):
            for i in range(n_layers):
                for b in range(2):
                    h32, h16 = rec32[c]["h"][i][b, o].float(), rec16[c]["h"][i][b, o].float()
                    d_e = float((rr.hidden[(sp, i, b, o)] - h32).abs().max())
                    d_16 = float((h16 - h32).abs().max())
                    if first is None and d_e > BAND_FACTOR * max(d_16, BAND_ABS):
                        first = (c, sp + o, i, b, d_e, d_16)
    assert first is not None, "the logits miss the rule but every residual stays inside the band"
    c, pos, i, b, d_e, d_16 = first
    sp = calls[c][0]
    eng_set, port_set = rr.got[(sp, i, b, pos - sp)].tolist(), rec32[c]["own"][i][b, pos - sp].tolist()
    sc = rec32[c]["scores"][i][b, pos - sp].tolist()
    print(f"[{label}] the residual first leaves the band at call start {sp}, position {pos}, layer {i}, sequence {b}: "
          f"|eng-port32| {d_e:.3e} against |port16-port32| {d_16:.3e}; experts engine {eng_set}, fp32 port {port_set}, "
          f"fp32 port scores {[round(x, 5) for x in sc]}")
    assert set(eng_set) != set(port_set), "the residual leaves the band at a token the engine routed like the port"


class _RouteRecorder:
    """Every moe_route launch of an engine's GEMV-chunk path: the experts of each token, as the port's force_routes takes
    them ((start_pos, layer) -> int64 [bsz * seqlen, k]), and every token's residual after each block (the fp16 sum of
    moe_route's h_out and moe_combine's output, which the next RMSNorm prologue forms).  Each launch's routing is checked
    against the float64 logit window of its own xn_out (oracle.numerics.route_check: a kernel_route outcome of that
    window)."""

    def __init__(self, eng):
        self.eng, self.got, self.hidden, self.start_pos, self.step, self.layer = eng, {}, {}, 0, None, 0

    def __enter__(self):
        eng, real_route, real_step, real_fwd = self.eng, ops.moe_route, self.eng._step, self.eng.forward_inference
        real_combine = ops.moe_combine

        def fwd(tokens, start_pos):
            self.start_pos, self.shape = start_pos, tuple(tokens.shape)
            return real_fwd(tokens, start_pos)

        def step(T, tps, kv, row0=0, **kw):
            self.step, self.layer = (T, tps, row0), 0
            return real_step(T, tps, kv, row0=row0, **kw)

        def route(**kw):
            real_route(**kw)
            torch.cuda.synchronize()
            T, k = kw["T"], kw["topk"]
            se, sw = kw["slot_expert"][:T * k].view(T, k), kw["slot_weight"][:T * k].view(T, k)
            matched, window, skipped = route_check(kw["xn_out"][:T], kw["gate_w"], sw, se, k)
            assert matched + window == T and skipped == 0
            _, tps, row0 = self.step
            off = eng.pos[:T].cpu().long() - self.start_pos
            self.keys = [(self.start_pos, self.layer, row0 + t // tps, int(off[t])) for t in range(T)]
            for t in range(T):
                self.got[self.keys[t]] = se[t].cpu().long()
            self.h_attn = kw["h_out"]
            self.layer += 1

        def combine(y_slot, slot_weight, slot_expert, out, **kw):
            real_combine(y_slot, slot_weight, slot_expert, out, **kw)
            after = (self.h_attn[:kw["T"]] + out[:kw["T"]]).float().cpu()
            for t, key in enumerate(self.keys):
                self.hidden[key] = after[t]
        ops.moe_route, ops.moe_combine, eng._step, eng.forward_inference = route, combine, step, fwd
        self._restore = lambda: (setattr(ops, "moe_route", real_route), setattr(ops, "moe_combine", real_combine),
                                 delattr(eng, "_step"), delattr(eng, "forward_inference"))
        return self

    def __exit__(self, *exc):
        self._restore()

    def routes(self, calls, bsz, n_layers):
        out = {}
        for sp, n in calls:
            for i in range(n_layers):
                out[(sp, i)] = torch.stack([self.got[(sp, i, b, o)] for b in range(bsz) for o in range(n)])
        return out


@pytest.mark.timeout(300)
@pytest.mark.parametrize("p0,p1", [(5, 40), (100, 200), (40, 300), (250, 33)])
def test_mixtral_continuation_prompt_matches_port(p0, p1):
    """A second prompt at start_pos = p0 > 0, then decode; both paths' logits (and the tensor-core path's KV cache) meet
    the port rule.

    The GEMV-chunk path at (40, 300) does not meet the plain rule: e32 = 2.2e-2 against a floor of 2.6e-3 (8.6x) on an
    H100.  Diagnosis: every launch of the schedule meets its float64 bound and writes nothing else, and every routing
    decision is the float64 route of the engine's own router input (test_engine_launch_audit_gpu.py).  This test prints
    the rest when the plain rule fails (_locate_excess, the port's per-layer record and forced routing).  The first prompt meets the rule (e32 2.6e-3, floor 2.1e-3); the excess starts in the
    continuation (1.4e-2) and carries into the decode steps (up to 2.2e-2).  The engine's residual stays inside the
    port's fp16 / fp32 band up to layer 0 of sequence 1 at position 107, where it leaves it by 600x (0.19 against 3.1e-4):
    there the fp32 port routes to experts (0, 3) and the engine to (0, 2), whose fp32 scores 0.28764 and 0.28701 differ
    by 2.6 fp16 ulps.  A second near-tie flips at layer 1, sequence 0, position 189 (0.3 ulp).  With the engine's routing
    forced into the port, e32 = 2.6e-3 against a floor of 2.6e-3: the rule holds.  So the excess is a routing flip at
    near-ties, not a kernel or glue error.
    Asserted: the plain rule, or all of: the rule against the port run with the engine's routing; every engine route a
    kernel_route outcome of its own float64 logit window; the first residual to leave the band sits at a token the
    engine and the fp32 port routed differently; and every flip (the engine's expert set differing from the fp32 port's
    own top-k on the same routed history) a near-tie within FLIP_ULPS fp16 ulps (a heuristic screen, not a bound)."""
    args, sd, sd_ref, recs = _tiny_mixtral()
    ndec, P = 3, p0 + p1
    toks = weights.synthetic_tokens(2, P + ndec, args["vocab_size"], seed=11)
    port = {}
    for dt in (torch.float32, torch.float16):
        port[dt] = PortModel("mixtral", args, sd_ref, dtype=dt)
        port[dt].record = []
    ref32 = _schedule(port[torch.float32], toks, p0, p1, ndec)
    ref16 = _schedule(port[torch.float16], toks, p0, p1, ndec)
    calls = [(0, p0), (p0, p1)] + [(P + j, 1) for j in range(ndec)]
    for tc in (True, False):
        label = f"tiny_mixtral_w4_continue{p0}+{p1}_{'wgmma' if tc else 'gemv_chunks'}"
        eng = _engine(args, sd, recs, tc, use_graph=tc)  # the GEMV-chunk path runs eager: its router launches are recorded
        with contextlib.nullcontext() if tc else _RouteRecorder(eng) as rr:
            got = _schedule(eng, toks.cuda(), p0, p1, ndec)
        if not tc:
            if _rule(label, got[0], ref16[0], ref32[0], asserted=False):
                continue
            _locate_excess(label, calls, got[0], ref16[0], ref32[0], rr, port, args["n_layers"])
            routes = rr.routes(calls, 2, args["n_layers"])
            forced = {}
            for dt in (torch.float32, torch.float16):
                m = PortModel("mixtral", args, sd_ref, dtype=dt)
                m.force_routes, m.record = routes, []
                forced[dt] = (_schedule(m, toks, p0, p1, ndec)[0], m.record)
            _rule(label + "_engine_routing", got[0], forced[torch.float16][0], forced[torch.float32][0])
            flips = []
            for rec in forced[torch.float32][1]:
                for i in range(args["n_layers"]):
                    used, own, sc = rec["routes"][i], rec["own"][i], rec["scores"][i]
                    for b in range(used.shape[0]):
                        for o in range(used.shape[1]):
                            a_, b_ = set(used[b, o].tolist()), set(own[b, o].tolist())
                            if a_ != b_:
                                s = sc[b, o].double()
                                lo, hi = s[sorted(a_ - b_)].min(), s[sorted(b_ - a_)].max()
                                n_ulp = float((hi - lo) / _ulp16(hi))
                                flips.append((rec["start_pos"] + o, i, b, n_ulp))
            print(f"\n[{label}] routing flips against the fp32 port (position, layer, sequence, fp16 ulps): {flips}")
            assert flips and all(f[3] <= FLIP_ULPS for f in flips), flips
            continue
        _rule(label, got[0], ref16[0], ref32[0])
        for i in range(args["n_layers"]):
            for j, name in enumerate("KV"):
                e = got[1][i][j][:, :, :P]
                r16, r32 = ref16[1][i][j][:, :, :P], ref32[1][i][j][:, :, :P]
                assert bool((got[1][i][j][:, :, P:] == 0).all()), (tc, i, name)  # nothing written past the prompts
                k16, k32, kf = float((e - r16).abs().max()), float((e - r32).abs().max()), float((r16 - r32).abs().max())
                assert k16 <= 1e-3 or k32 <= 1.5 * kf, (tc, i, name, k16, k32, kf)


@pytest.mark.timeout(300)
def test_graph_decode_after_a_tensor_core_prompt_equals_eager():
    """max_seq_len = 128: the eager step sizes attention for (pos + 128) // 128 * 128 cached rows, the captured step for
    the whole cache, and only where the two agree do both take the same KV split (and so the same summation order)."""
    args, sd, sd_ref, recs = _tiny_mixtral(max_seq_len=128)
    plen, ndec = 70, 4
    toks = weights.synthetic_tokens(2, plen + ndec, args["vocab_size"], seed=13).cuda()
    eager = _run(_engine(args, sd, recs, True, use_graph=False), toks, plen, ndec)
    graph = _run(_engine(args, sd, recs, True, use_graph=True), toks, plen, ndec)
    assert np.array_equal(eager, graph)


@pytest.mark.timeout(300)
def test_mixtral_golden_through_the_bit_exact_w_hat_instance():
    """force_tc: every forward_inference call of the mixtral_w4 golden case (prompt and decode steps) through the tensor-core
    GEMMs, whose dequant rebuilds the reference's w_hat bit for bit.  The asserted rule is the port rule; strict_pass is
    recorded, not asserted (a routing tie can flip an expert)."""
    import os
    name = "mixtral_w4"
    kind, args, bits, gs, bsz, plen, ndec = cases.CASES[name]
    kind, args, sd, sd_ref, recs, toks = cases.build_case(name)
    eng = DecodeEngine(EngineConfig.from_model_args(kind, args, bits=bits, group_size=gs), DEV)
    eng.load_master_state_dict(sd, quant_records=recs)
    eng.force_tc = True
    assert eng.prefill_tc_supported()
    got = _run(eng, toks.cuda(), plen, ndec)
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"{name}.npz"))
    _rule(name + "_exact_what_wgmma", got, g["logits_fp16"], g["logits_fp32"])


MIXTRAL_WIDTH = dict(dim=4096, hidden_dim=14336, n_layers=1, n_heads=32, n_kv_heads=8, norm_eps=1e-5, rope_theta=1e6,
                     vocab_size=2048, max_seq_len=320, max_batch_size=1, moe=dict(num_experts=8, num_experts_per_tok=2))


@pytest.mark.timeout(600)
def test_mixtral_width_prompt_matches_port():
    """One block at Mixtral-8x7B width (D 4096, F 14336, 8 experts, top-2), a 300-token prompt (256 + 44-token chunks)
    + decode, against the port run on the GPU in fp32 and fp16 on the same fake-quantised weights."""
    args = MIXTRAL_WIDTH
    torch.cuda.empty_cache()
    sd = {k: v.to(DEV) for k, v in weights.mixtral_state_dict(args, seed=21).items()}
    sd_ref, recs = omniquant.fake_quantize_state_dict(sd, 4, 0)
    plen, ndec = 300, 2
    toks = weights.synthetic_tokens(1, plen + ndec, args["vocab_size"], seed=23)
    with torch.inference_mode():
        ref32 = cases.run_schedule(PortModel("mixtral", args, sd_ref, dtype=torch.float32), toks.cuda(), plen, ndec).cpu().numpy()
        torch.cuda.empty_cache()
        ref16 = cases.run_schedule(PortModel("mixtral", args, sd_ref, dtype=torch.float16), toks.cuda(), plen, ndec).cpu().numpy()
    torch.cuda.empty_cache()
    eng = _engine(args, sd, recs, True)
    got = _run(eng, toks.cuda(), plen, ndec)
    _rule("mixtral_width_w4_prefill300_wgmma", got, ref16, ref32)
