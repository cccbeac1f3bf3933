"""GPU, one device: the fused tensor-parallel all-reduce of the bs = 1 decode step (ll.cuh, DESIGN.md section 5), every rank
simulated in one process with plain local buffers standing in for the peer-mapped ones.

The exchange.  A row-parallel GEMV (wo / w2, F16 epilogue) called with ar_out_peers pushes its fp16 partial sums as 8-byte
units {half2, seq} into slot `rank` of every rank's buffer ([tp][N / 2] units; unit j = rows 2j (low half) and 2j + 1).  The
next GEMV's RMSNorm prologue (ar_in) polls the tp slots of its own buffer until every unit carries the expected sequence
number seq = (step * period + id + 1) mod 2^32, adds the slots in rank order in fp32 and rounds once to fp16 (delta), then
does the residual add h = fp16(resid + delta).  The CPU model of all this lives in oracle/numerics.py (ll_*).

Rank-sum bound.  Write s for the exact sum of the partials p_r and s32 for the rank-order fp32 sum.  Each of the tp - 1
fp32 additions rounds to nearest, off by at most 2^-24 times a partial sum, and every partial sum is at most sum_r |p_r|
(up to its own rounding, the factor 1 + 2^-20); the final fp16 rounding is half an fp16 spacing at |s32|:
    |delta - s| <= 1/2 ulp16(s32) + (tp - 1) 2^-24 sum_r |p_r|
Partials whose exponents span at most 11 binades sum exactly in fp32 at tp <= 8 (every partial sum is a multiple of the
finest fp16 spacing among them and below 2^24 times it), so there delta must equal fp16 of the exact sum.

Safety: no launch here ever waits on a poll.  Before every launch with ar_in the host reads the polled buffer and fails the
test, without launching, unless every unit carries the sequence number that launch expects; after every launch the error
word must still be 0 (or still 1 where a test sets it on purpose).  Ranks never run concurrently: producers run one after
the other and their consumers only afterwards.  A single device cannot test NVLink store visibility, concurrent polling or
CUDA IPC mapping; tests/test_tp_gpu.py on two GPUs remains the only check of those.
"""
import contextlib
import ctypes as C
import math
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import kvlayout, ops, quant  # noqa: E402
from llama2_accessory_b200.engine import EngineConfig, _interleave_w13, rope_table  # noqa: E402
from oracle.numerics import LL_SENT, SENT, gemv_check, ll_decode, ll_encode, ll_rank_sum  # noqa: E402
from oracle.numerics import ll_rank_sum_bound, ll_seq, nan16, tuned  # noqa: E402

DEV = "cuda"
EPS = 1e-5
SLOT = 16384             # bytes of one weight-ring stage
STATS = {"units": 0, "elements": 0, "gemv_ratio": 0.0, "sum_ratio": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()
    yield
    print(f"\n[tp all-reduce] units checked bit for bit {STATS['units']}, consumer elements {STATS['elements']}; worst "
          f"producer GEMV err/tol {STATS['gemv_ratio']:.3f}, worst rank-sum err/tol {STATS['sum_ratio']:.3f}")


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _sync(x):
    torch.cuda.synchronize()
    return x


# ------------------------------------------------------------------------------------------------- exchange helpers --
def _ll_buf(tp, N):
    """An LL buffer [tp, N / 2, 2] int32 filled with the sentinel word."""
    return torch.full((tp, N // 2, 2), LL_SENT, dtype=torch.int32, device=DEV)


def _ctr(step, err=0):
    """The engine's counter block: [0] decode-step counter (uint32 in an int32 word), [1] poll time-out word."""
    c = torch.zeros(4, dtype=torch.int32, device=DEV)
    c[0] = int(np.uint32(step % (1 << 32)).view(np.int32))
    c[1] = err
    return c


def _ar(ctr, world, rank, period, **kw):
    return dict(world=world, rank=rank, step=ctr.data_ptr(), period=period, err=ctr.data_ptr() + 4, **kw)


def _peers(bufs):
    return (C.c_void_p * len(bufs))(*[b.data_ptr() for b in bufs])


def _precheck(buf, seq, label):
    """The host read before a consumer launch: every unit of every slot carries `seq`, else fail without launching."""
    _, s = ll_decode(_sync(buf).cpu().numpy())
    bad = int((s != np.uint32(seq)).sum())
    assert bad == 0, f"{label}: {bad} of {s.size} polled units do not carry sequence number {seq}; consumer not launched"


def _err_word(ctr):
    return int(_sync(ctr)[1].item())


# ------------------------------------------------------------------------------------------------------- weights ------
def _linear(bits, gs, N, K, seed, w13=False):
    """Random codes / scales / zero points -> (PackedLinear, float64 w_hat, float64 A with M = A . |x|), as
    tests/test_gemv_batched_moe_gpu.py.  w13: rows interleaved as the engine's w13."""
    g = _gen(seed)
    if bits == 16:
        w = ((torch.rand(N, K, generator=g, device=DEV) * 2 - 1) / math.sqrt(K)).half()
        return quant.pack_fp16(w, DEV), w.double(), w.double().abs()
    G = 1 if gs == 0 else K // gs
    qmax = 2 ** bits - 1

    def one(n):
        q = torch.randint(0, qmax + 1, (n, K), generator=g, device=DEV, dtype=torch.uint8)
        s = ((0.75 + 0.5 * torch.rand(n, G, generator=g, device=DEV)) * 2.0 / (qmax * math.sqrt(K))).half()
        return q, s, torch.randint(0, qmax + 1, (n, G), generator=g, device=DEV).half()
    if w13:
        (q1, s1, z1), (q3, s3, z3) = one(N // 2), one(N // 2)
        q, s, z = _interleave_w13(q1, q3), _interleave_w13(s1, s3), _interleave_w13(z1, z3)
    else:
        q, s, z = one(N)
    pl = quant.pack_quantized(q, s, z, bits, gs, DEV)
    sd = s.double().repeat_interleave(K // G, dim=1)
    zd = z.double().repeat_interleave(K // G, dim=1)
    return pl, (q.double() - zd) * sd, sd * (q.double() + zd.abs())


ARCH = {"7b": dict(dim=4096, n_heads=32, vocab_size=32000, multiple_of=256),
        "13b": dict(dim=5120, n_heads=40, vocab_size=32000, multiple_of=256),
        "70b": dict(dim=8192, n_heads=64, n_kv_heads=8, vocab_size=32000, multiple_of=4096, ffn_dim_multiplier=1.3)}


def _widths(arch, tp):
    """(dim, local FFN width padded to 128 as DecodeEngine does, local q heads, local kv heads) of one rank."""
    c = EngineConfig.from_model_args("llama", dict(ARCH[arch], n_layers=1), bits=4, group_size=0, tp_rank=0, tp_world=tp)
    F = (c.ffn_hidden // tp + 127) // 128 * 128
    return c.dim, F, c.n_heads // tp, c.kv_heads // tp


# ---------------------------------------------------------------------------------------------- 1. producer side ----
PRODUCER_SHAPES = [(a, tp, lin) for a, tps in (("7b", (2, 4, 8)), ("13b", (2, 4)), ("70b", (2, 8))) for tp in tps
                   for lin in ("wo", "w2")]
#            label              bits  gs   tune knob
CODECS = [("w4_pc",             4,    0, None),
          ("w4_g128",           4,  128, None),
          ("w4_g64",            4,   64, None),
          ("w4_pc_generic",     4,    0, ("B200_GEMV1", 0)),
          ("w4_g128_generic",   4,  128, ("B200_GEMV1_GROUPED", 0)),
          ("w3_pc",             3,    0, None),
          ("w2_g128",           2,  128, None),
          ("f16",              16,    0, None)]


def _knob(k):
    return tuned(*k) if k is not None else contextlib.nullcontext()


def _push(pl, x, tp, rank, step, period, ident, **kw):
    """One producer launch into tp fresh sentinel buffers -> (buffers, out, counter)."""
    bufs = [_ll_buf(tp, pl.N) for _ in range(tp)]
    ctr = _ctr(step)
    out = nan16(1, pl.N, device=DEV)
    ops.gemv(pl, 1, xin=x, out=out, ar=_ar(ctr, tp, rank, period, out_peers=_peers(bufs), out_id=ident), **kw)
    _sync(out)
    assert _err_word(ctr) == 0
    return [b.cpu().numpy() for b in bufs], out, ctr


def _check_push(bufs, rank, ref16, seq, label):
    """Slot `rank` of every buffer: identical bytes, payload == ref16 bit for bit, every seq == seq; all else sentinel."""
    tp = len(bufs)
    first = bufs[0][rank]
    pay, s = ll_decode(first[None])
    missing = int((first.view(np.uint32) == np.uint32(LL_SENT)).all(-1).sum())
    assert missing == 0, f"{label}: {missing} of {first.shape[0]} units of slot {rank} never written"
    assert (s == np.uint32(seq)).all(), (label, "sequence number", int(s.min()), int(s.max()), seq)
    assert np.array_equal(pay[0].view(np.uint16), ref16.view(np.uint16)), (label, "payload")
    for r, b in enumerate(bufs):
        assert np.array_equal(b[rank], first), (label, "buffer", r, "differs in slot", rank)
        others = np.delete(b, rank, axis=0)
        assert (others.view(np.uint32) == np.uint32(LL_SENT)).all(), (label, "buffer", r, "written outside slot", rank)
    STATS["units"] += tp * first.shape[0]


def _wrap_steps(period, ident):
    """Counter values whose sequence numbers straddle the unsigned wrap for this period and id."""
    s0 = ((1 << 32) - ident - 1) // period
    return [s0 - 1, s0, s0 + 1]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("label,bits,gs,knob", CODECS, ids=[c[0] for c in CODECS])
@pytest.mark.parametrize("arch,tp,lin", PRODUCER_SHAPES, ids=[f"{a}_tp{t}_{n}" for a, t, n in PRODUCER_SHAPES])
def test_producer_pushes_every_row_to_every_rank(arch, tp, lin, label, bits, gs, knob):
    """The wo / w2 shard of one rank: the units equal the launch's own fp16 output (itself within the float64 GEMV bound),
    in slot `rank` of every buffer only, with the formula's sequence number for every counter value; `out` untouched;
    PDL, prefetches and ring depths leave the units bit-identical."""
    D, F, _, _ = _widths(arch, tp)
    N, K = D, (D // tp if lin == "wo" else F)
    rank = tp - 1 if tp > 2 else 1
    seed = N + K + bits + gs + tp
    pl, W, A = _linear(bits, gs, N, K, seed)
    x = torch.randn(1, K, generator=_gen(seed), device=DEV).half()
    tag = f"{arch}/tp{tp}/{lin}/{label}"
    L, ident = 32, 2 * 5 + (lin == "w2")
    with _knob(knob):
        plain = nan16(1, N, device=DEV)
        ops.gemv(pl, 1, xin=x, out=plain)
        ratio, _, _ = gemv_check(_sync(plain), (W @ x.double().reshape(-1)).reshape(1, -1),
                                 (A @ x.double().abs().reshape(-1)).reshape(1, -1), tag)
        STATS["gemv_ratio"] = max(STATS["gemv_ratio"], ratio)
        ref16 = plain.reshape(-1).cpu().numpy()
        base = None
        steps = [(1, 2 * L + 2), (2, 2 * L + 2), (40_000_000, 2 * L + 2)]
        steps += [(s, 2 * l + 2) for l in (32, 80) for s in _wrap_steps(2 * l + 2, ident)]
        for step, period in steps:
            bufs, out, _ = _push(pl, x, tp, rank, step, period, ident)
            seq = ll_seq(step, period, ident)
            assert seq != np.uint32(LL_SENT)
            _check_push(bufs, rank, ref16, seq, f"{tag} step={step} period={period}")
            assert bool((out.view(torch.int16) == SENT).all()), (tag, "out written by a pushing launch")
            if base is None:
                base = bufs
        nxt = quant.random_packed(4, 1024, 512, 0, DEV, 9)
        gamma = torch.ones(4096, dtype=torch.float16, device=DEV)
        variants = [dict(use_pdl=True), dict(prefetch=(nxt.qweight, nxt.qweight.numel(), nxt.N // 16)),
                    dict(prefetch_const=gamma)] + [dict(ring_bytes=n * SLOT) for n in (2, 3, 8, 24)]
        for kw in variants:
            bufs, _, _ = _push(pl, x, tp, rank, steps[0][0], steps[0][1], ident, **kw)
            assert all(np.array_equal(a, b) for a, b in zip(bufs, base)), (tag, list(kw))
    print(f"\n[{tag}] GEMV err/tol {ratio:.3f}; {len(steps) + len(variants)} pushes x {tp} buffers x {N // 2} units exact")


# ---------------------------------------------------------------------------------------------- 3. consumer side ----
def _families(tp, K, seed):
    """name -> fp16 partials [tp, K] (numpy).  Every pattern is tiled over K with rank placements varied per element."""
    rng = np.random.default_rng(seed)
    e = np.arange(K)
    fam = {}
    # 1. exact sums: exponents within 11 binades ([-4, 6]), mixed signs
    ex = rng.integers(-4, 7, (tp, K))
    fam["exact"] = (rng.choice([-1.0, 1.0], (tp, K)) * 2.0 ** ex * (1 + rng.integers(0, 1024, (tp, K)) / 1024)).astype(np.float16)
    # 2. position-coded integers: a swapped half, a misaddressed unit or a slot read twice changes an exact sum
    fam["position"] = ((e[None] % 61) + 32 * np.arange(tp)[:, None]).astype(np.float16)
    if tp >= 4:
        # 3. order: 2^15, 16 and two 3 * 2^-11: in rank order both small ones vanish (0.375 fp32 ulp each) and the sum
        #    ties to 2^15 in fp16; added first they survive and push the sum above the fp16 midpoint.  Placements and
        #    scales are drawn at random and kept where the CPU model confirms that reversing the rank order changes delta.
        sc = 2.0 ** -rng.integers(0, 8, K * 4) * rng.choice([-1.0, 1.0], K * 4)
        cand = np.zeros((tp, K * 4))
        slots = np.argsort(rng.random((tp, K * 4)), 0)[:4]
        slots = np.sort(slots, 0)
        for i, v in enumerate((32768.0, 16.0, 3 * 2.0 ** -11, 3 * 2.0 ** -11)):
            cand[slots[i], np.arange(K * 4)] = v * sc
        cand = cand.astype(np.float16)
        keep = ll_rank_sum(cand).view(np.uint16) != ll_rank_sum(cand, list(range(tp))[::-1]).view(np.uint16)
        assert int(keep.sum()) >= K, int(keep.sum())
        fam["order"] = cand[:, keep][:, :K]
    if tp >= 3:
        # 4. fp32 accumulation: a small value, then +-big cancelling pair: an fp16 running sum loses the small value
        big = (32 * rng.integers(1024, 2047, K)).astype(np.float64)
        small = rng.integers(1, 255, K) * 2.0 ** -8
        p = np.zeros((tp, K))
        p[0], p[1], p[2] = small, big, -big
        fam["fp32_acc"] = p.astype(np.float16)
        run16 = np.zeros(K, np.float16)
        for r in range(tp):
            run16 = (run16 + fam["fp32_acc"][r]).astype(np.float16)
        assert (run16.view(np.uint16) != ll_rank_sum(fam["fp32_acc"]).view(np.uint16)).all()
    # 5. edges: -0.0, subnormals, +-65504 with a finite sum
    edge = np.zeros((tp, K), np.float16)
    kind = e % 4
    edge[:, kind == 0] = np.float16(-0.0)
    sub = rng.integers(1, 1023, (tp, K)) * rng.choice([-1, 1], (tp, K))
    edge[:, kind == 1] = (sub[:, kind == 1] * 2.0 ** -24).astype(np.float16)
    alt = np.where(np.arange(tp) % 2 == 0, 65504.0, -65504.0)       # running sums 65504, 0, 65504, ...
    deep = np.array([-1, -1, 1, 1, -1, 1, -1, 1][:tp]) * 65504.0 if tp >= 3 else -alt  # -65504, -131008 (fp32 only), ...
    edge[:, kind == 2] = alt[:, None]
    edge[:, kind == 3] = deep[:, None]
    fam["edge"] = edge
    for name, p in fam.items():
        assert np.isfinite(ll_rank_sum(p).astype(np.float32)).all(), name
    return fam


def _consumer_case(tp, epi):
    """(PackedLinear, aux) of one consumer launch at the 7B width: aux is the SiLU output width F, the QKV launch's heads
    per kind (q = k = v) or the lm_head's vocabulary shard N."""
    D = 4096
    if epi in ("silu", "silu_generic"):
        F = (11008 // tp + 127) // 128 * 128
        return _linear(4, 0, 2 * F, D, 100 + tp, w13=True)[0], F
    if epi == "qkv":
        H = max(1, 32 // tp)
        return _linear(4, 0, 3 * H * 128, D, 200 + tp)[0], H
    N = (32000 // tp) // 16 * 16
    return _linear(16, 0, N, D, 300 + tp)[0], N


def _consume_qkv(pl, Hq, Hkv, resid, gamma, **kw):
    """One QKV launch at position 40 into sentinel caches -> (h_out, q, K cache, V cache)."""
    S, ps = 64, 40
    kc = kvlayout.k_to_engine(nan16(1, Hkv, S, 128, device=DEV))
    vt = nan16(1, Hkv, S // 32, 128, 32, device=DEV)
    rope = rope_table(128, 2 * S, 10000.0, None).to(DEV)
    q, h_out = nan16(1, Hq * 128, device=DEV), nan16(1, pl.K, device=DEV)
    qkv = dict(n_q_rows=Hq * 128, n_kv_rows=Hkv * 128, rope=rope, pos=torch.tensor([ps], dtype=torch.int32, device=DEV),
               tokens_per_seq=1, kcache=kc, vtcache=vt, cache_seq=S)
    ops.gemv(pl, 1, resid=resid, h_out=h_out, gamma=gamma, eps=EPS, epilogue=ops.B200_EPI_QKV, out=q, qkv=qkv, **kw)
    return _sync(h_out), q, kc, vt


def _consume(pl, epi, aux, resid, gamma, **kw):
    """One RMSNorm-prologue launch -> tuple of its outputs (h_out first)."""
    h_out = nan16(1, pl.K, device=DEV)
    if epi in ("silu", "silu_generic"):
        out = nan16(1, aux, device=DEV)
        ops.gemv(pl, 1, resid=resid, h_out=h_out, gamma=gamma, eps=EPS, epilogue=ops.B200_EPI_SILU, out=out, **kw)
        return _sync(h_out), out
    if epi == "qkv":
        return _consume_qkv(pl, aux, aux, resid, gamma, **kw)
    out = torch.full((1, aux), float("nan"), device=DEV)
    ops.gemv(pl, 1, resid=resid, h_out=h_out, gamma=gamma, eps=EPS, epilogue=ops.B200_EPI_F32, out=out, **kw)
    return _sync(h_out), out


def _same(a, b):
    dt = torch.int16 if a.element_size() == 2 else torch.int32
    return torch.equal(a.contiguous().view(dt), b.contiguous().view(dt))


CONSUMER_EPIS = ["silu", "qkv", "lm_head", "silu_generic"]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("epi", CONSUMER_EPIS)
@pytest.mark.parametrize("tp", [2, 3, 4, 5, 8])
def test_consumer_rank_sum_matches_the_model(tp, epi):
    """A buffer pre-filled with valid units from crafted partials: h_out == fp16(resid + model delta) and every output equals
    the same launch given delta = model delta as a plain fp16 vector (covered against float64 by test_decode_path_gpu.py)."""
    K = 4096
    pl, aux = _consumer_case(tp, epi)
    g = _gen(tp * 10 + len(epi))
    resid = torch.randn(1, K, generator=g, device=DEV).half()
    gamma = (1 + 0.2 * torch.randn(K, generator=g, device=DEV)).half()
    period, ident, step = 2 * 32 + 2, 2 * 7 + 1, 12345
    seq = ll_seq(step, period, ident)
    knob = ("B200_GEMV1", 0) if epi == "silu_generic" else None
    worst = 0.0
    with _knob(knob):
        for name, parts in _families(tp, K, seed=tp).items():
            model = ll_rank_sum(parts)
            r_in = resid
            if name == "edge":
                # -0 residual in the -0.0 and subnormal columns: h = fp16(-0 + delta) is delta itself, sign of zero included
                zc = torch.from_numpy(np.arange(K) % 4 < 2).to(DEV)
                r_in = torch.where(zc, torch.tensor(-0.0, dtype=torch.float16, device=DEV), resid)
            s, bound = ll_rank_sum_bound(parts)
            r = float((np.abs(model.astype(np.float64) - s) / bound).max())
            assert r <= 1.0, (name, r)
            worst = max(worst, r)
            if name in ("exact", "position"):
                assert np.array_equal(model.view(np.uint16), s.astype(np.float16).view(np.uint16)), name
            buf = torch.from_numpy(ll_encode(parts, seq)).to(DEV)
            ctr = _ctr(step)
            _precheck(buf, seq, f"tp{tp}/{epi}/{name}")
            got = _consume(pl, epi, aux, r_in, gamma, ar=_ar(ctr, tp, 0, period, in_buf=buf.data_ptr(), in_id=ident))
            assert _err_word(ctr) == 0, (tp, epi, name)
            dl = torch.from_numpy(model).to(DEV).reshape(1, K)
            want = _consume(pl, epi, aux, r_in, gamma, delta=dl)
            assert _same(want[0], r_in + dl), (tp, epi, name, "plain-delta h_out")
            if name == "edge":
                assert _same(got[0][0, zc], dl[0, zc]), (tp, epi, "-0.0 / subnormal deltas not carried into h_out")
            for i, (a, b) in enumerate(zip(got, want)):
                assert _same(a, b), (tp, epi, name, "output", i, int((a.view(torch.int16) != b.view(torch.int16)).sum())
                                     if a.element_size() == 2 else -1)
            STATS["elements"] += K
    STATS["sum_ratio"] = max(STATS["sum_ratio"], worst)
    print(f"\n[tp{tp}/{epi}] families bit-exact; worst rank-sum err/tol {worst:.3f}")


@pytest.mark.timeout(120)
def test_error_word_already_set_changes_nothing_when_units_are_valid():
    """The capped-poll branch (error word 1 from an earlier time-out): with every unit valid the outputs are those of a
    clean launch, and the word stays 1."""
    tp, K = 4, 4096
    pl, aux = _consumer_case(tp, "silu")
    g = _gen(5)
    resid = torch.randn(1, K, generator=g, device=DEV).half()
    gamma = (1 + 0.2 * torch.randn(K, generator=g, device=DEV)).half()
    parts = _families(tp, K, seed=1)["exact"]
    seq = ll_seq(7, 66, 3)
    buf = torch.from_numpy(ll_encode(parts, seq)).to(DEV)
    outs = []
    for err in (0, 1):
        ctr = _ctr(7, err)
        _precheck(buf, seq, f"error word {err}")
        outs.append(_consume(pl, "silu", aux, resid, gamma, ar=_ar(ctr, tp, 0, 66, in_buf=buf.data_ptr(), in_id=3)))
        assert _err_word(ctr) == err
    assert all(_same(a, b) for a, b in zip(*outs))


# ---------------------------------------------------------------------------------------- 4. chain at real widths ----
CHAIN = [("7b", 2), ("7b", 4), ("7b", 8), ("70b", 8)]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("arch,tp", CHAIN, ids=[f"{a}_tp{t}" for a, t in CHAIN])
def test_chain_wo_w13_w2_wqkv_over_two_steps(arch, tp):
    """All ranks' wo shards push, every rank's w13 consumes; all w2 push, every rank's next-layer wqkv consumes, over two
    counter steps with step n - 1's units still in the buffers.  Every rank's h_out is bit-identical, equals the CPU
    model, and every rank's outputs equal its launch with the plain model delta."""
    D, F, H, Hkv = _widths(arch, tp)
    L, period = 2, 2 * 2 + 2
    ranks = []
    for r in range(tp):
        s = 1000 * tp + 10 * r
        ranks.append(dict(wo=_linear(4, 0, D, H * 128, s)[0], w13=_linear(4, 0, 2 * F, D, s + 1, w13=True)[0],
                          w2=_linear(4, 0, D, F, s + 2)[0], wqkv=_linear(4, 0, (H + 2 * Hkv) * 128, D, s + 3)[0]))
    g = _gen(tp)
    gamma = (1 + 0.2 * torch.randn(D, generator=g, device=DEV)).half()
    buf_o = [_ll_buf(tp, D) for _ in range(tp)]
    buf_f = [_ll_buf(tp, D) for _ in range(tp)]
    ctr = [_ctr(0) for _ in range(tp)]
    for step in (5, 6):
        for c in ctr:
            c[0] = step
        resid = torch.randn(1, D, generator=g, device=DEV).half()     # every rank holds the same residual stream
        attn = [(0.5 * torch.randn(1, H * 128, generator=g, device=DEV)).half() for _ in range(tp)]
        for stage, (prod, cons, peers, pid) in enumerate((("wo", "w13", buf_o, 0), ("w2", "wqkv", buf_f, 1))):
            parts = []
            for r in range(tp):
                x = attn[r] if prod == "wo" else acts[r]
                plain = nan16(1, D, device=DEV)
                ops.gemv(ranks[r][prod], 1, xin=x, out=plain)
                parts.append(_sync(plain).reshape(-1).cpu().numpy())
                ops.gemv(ranks[r][prod], 1, xin=x, out=nan16(1, D, device=DEV),
                         ar=_ar(ctr[r], tp, r, period, out_peers=_peers(peers), out_id=pid))
            parts = np.stack(parts)
            seq = ll_seq(step, period, pid)
            for r in range(tp):
                _precheck(peers[r], seq, f"{arch}/tp{tp} step {step} {prod} -> rank {r}")
                pay, _ = ll_decode(peers[r].cpu().numpy())
                assert np.array_equal(pay.view(np.uint16), parts.view(np.uint16)), (arch, tp, step, prod, r)
            model = torch.from_numpy(ll_rank_sum(parts)).to(DEV).reshape(1, D)
            hs, acts_next = [], []
            for r in range(tp):
                aux = F if cons == "w13" else Hkv
                epi = "silu" if cons == "w13" else "qkv"
                pl = ranks[r][cons]
                if epi == "qkv":
                    got = _consume_qkv(pl, H, Hkv, resid, gamma, ar=_ar(ctr[r], tp, r, period, in_buf=peers[r].data_ptr(),
                                                                         in_id=pid))
                    want = _consume_qkv(pl, H, Hkv, resid, gamma, delta=model)
                else:
                    got = _consume(pl, epi, aux, resid, gamma, ar=_ar(ctr[r], tp, r, period, in_buf=peers[r].data_ptr(),
                                                                      in_id=pid))
                    want = _consume(pl, epi, aux, resid, gamma, delta=model)
                assert _err_word(ctr[r]) == 0, (arch, tp, step, cons, r)
                assert all(_same(a, b) for a, b in zip(got, want)), (arch, tp, step, cons, r)
                hs.append(got[0])
                acts_next.append(got[1])
            assert all(_same(h, resid + model) for h in hs), (arch, tp, step, cons)
            STATS["elements"] += tp * D
            if cons == "w13":
                acts = acts_next
                resid = hs[0]
    print(f"\n[chain {arch} tp{tp}] two steps: {tp} ranks bit-identical, equal to the rank-sum model")


# ------------------------------------------------------------- 5. the engine's TP decode step, all ranks in lockstep ----
LAUNCHES = {"b200_gemv", "b200_attn_decode", "b200_embed", "b200_advance_pos", "b200_argmax", "b200_prefill_gemm_w4",
            "b200_prefill_moe_gemm_w4", "b200_prefill_rmsnorm", "b200_prefill_rope_kv", "b200_prefill_silu_mul",
            "b200_moe_route", "b200_moe_expert_ffn", "b200_moe_combine", "b200_sample_top_p", "b200_generate_update"}


class _Lockstep:
    """tp DecodeEngines driven from tp threads on one device.

    Stands in for the library: every launch runs under one lock and is synchronised, then all ranks meet at a barrier, so
    launch k of every rank has completed before any rank's launch k + 1 starts (the ranks issue the same launches in the
    same order); a b200_gemv with ar_in is preceded by the host pre-check of its buffer.  Stands in for torch.distributed:
    all_gather / all_reduce / barrier exchange device tensors at the same barrier, and all_reduce of fp16 is the fp32
    rank-order sum rounded once (the semantics of the fused path).  DecodeEngine._peer_buffers hands every rank the same
    tp zeroed local buffers."""

    def __init__(self, real, tp):
        self.real, self.tp = real, tp
        self.lock = threading.Lock()
        self.bar = threading.Barrier(tp, timeout=120)
        self.local = threading.local()
        self.engines = [None] * tp
        self.peer = {}
        self.slots = [None] * tp
        self.prechecked = 0

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        if name not in LAUNCHES:
            return fn

        def call(*args):
            rank = getattr(self.local, "rank", None)
            if rank is None:
                return fn(*args)
            with self.lock:
                if name == "b200_gemv":
                    self._precheck(rank, args[0]._obj)
                rc = fn(*args)
                torch.cuda.synchronize()
            self.wait()
            return rc
        return call

    def wait(self):
        try:
            self.bar.wait()
        except threading.BrokenBarrierError:
            raise RuntimeError("another rank failed") from None

    def _precheck(self, rank, a):
        if a.ar_world <= 1 or not a.ar_in:
            return
        torch.cuda.synchronize()
        step = int(self.engines[rank]._ar["step"][0].item()) & 0xFFFFFFFF
        n = a.ar_world * a.lin.K * 4
        for bufs in self.peer.values():
            t = bufs[rank]
            off = a.ar_in - t.data_ptr()
            if 0 <= off and off + n <= t.numel():
                units = t[off:off + n].view(torch.int32).reshape(a.ar_world, a.lin.K // 2, 2)
                _precheck(units, ll_seq(step, a.ar_period, a.ar_in_id), f"rank {rank} in_id {a.ar_in_id}")
                self.prechecked += 1
                return
        raise AssertionError(f"rank {rank}: ar_in is not one of the exchange buffers")

    def peer_buffers(self, eng, nbytes):
        with self.lock:
            bufs = self.peer.setdefault(nbytes, [torch.zeros(nbytes, dtype=torch.uint8, device=DEV) for _ in range(self.tp)])
        return bufs[eng.cfg.tp_rank].data_ptr(), [b.data_ptr() for b in bufs]

    def _exchange(self, t):
        r = self.local.rank
        torch.cuda.synchronize()
        self.slots[r] = t.detach().clone()
        self.wait()
        vals = list(self.slots)
        self.wait()
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

    def barrier(self, group=None, **kw):
        self.wait()

    def run(self, fn):
        """fn(rank) in tp threads -> [its result per rank]; any failure aborts the barrier and is raised here."""
        out, errs = [None] * self.tp, []

        def body(r):
            self.local.rank = r
            try:
                out[r] = fn(r)
            except BaseException as e:  # noqa: BLE001 -- re-raised in the calling thread
                errs.append(e)
                self.bar.abort()
        ths = [threading.Thread(target=body, args=(r,)) for r in range(self.tp)]
        for t in ths:
            t.start()
        for t in ths:
            t.join(timeout=900)
        assert not any(t.is_alive() for t in ths), "a rank thread did not finish"
        if errs:
            raise next((e for e in errs if not isinstance(e, RuntimeError) or "another rank" not in str(e)), errs[0])
        self.bar.reset()
        return out


@pytest.fixture()
def lockstep(monkeypatch):
    import torch.distributed as dist
    from llama2_accessory_b200 import _cabi
    from llama2_accessory_b200.engine import DecodeEngine

    def make(tp):
        ls = _Lockstep(_cabi.lib(), tp)
        monkeypatch.setattr(_cabi, "_lib", ls)
        monkeypatch.setattr(DecodeEngine, "_peer_buffers", lambda self, nbytes: ls.peer_buffers(self, nbytes))
        monkeypatch.setattr(dist, "all_gather", ls.all_gather)
        monkeypatch.setattr(dist, "all_reduce", ls.all_reduce)
        monkeypatch.setattr(dist, "barrier", ls.barrier)
        return ls
    return make


def _engines(ls, arch, tp, n_layers, sd=None, recs=None):
    """tp engines (rank r = tp_rank r) on the one device, graphs off.  sd: master weights (quantised, then sharded);
    otherwise load_random with every rank's linears and lm_head shard drawn from rank-specific seeds (the embedding and
    norms, which every rank holds whole, from one seed)."""
    from llama2_accessory_b200.engine import DecodeEngine
    args = dict(ARCH[arch], n_layers=n_layers, max_seq_len=2112, max_batch_size=1)
    for r in range(tp):
        cfg = EngineConfig.from_model_args("llama", args, bits=4, group_size=0, tp_rank=r, tp_world=tp)
        eng = DecodeEngine(cfg, DEV)
        eng.use_graph = False
        if sd is not None:
            eng.load_master_state_dict(sd, quant_records=recs)
        else:
            eng.load_random(seed=0)
            s, D = 1000 + 100 * r, cfg.dim
            eng.lm_head = quant.random_packed(16, eng.V_loc, D, 0, DEV, s)
            for i, lw in enumerate(eng.layers):
                lw.wqkv = quant.random_packed(4, (eng.Hq + 2 * eng.Hkv) * 128, D, 0, DEV, s + 4 * i + 1)
                lw.wo = quant.random_packed(4, D, eng.Hq * 128, 0, DEV, s + 4 * i + 2)
                lw.w13 = quant.random_packed(4, 2 * eng.F, D, 0, DEV, s + 4 * i + 3)
                lw.w2 = quant.random_packed(4, D, eng.F, 0, DEV, s + 4 * i + 4)
        ls.engines[r] = eng
    return args


def _schedule(ls, toks, plen, positions, noise):
    """Every rank: the prompt, then (noise: the KV cache refilled with noise) one decode step per position.
    -> per rank ([logits after the prompt and after every step], [h rows after every step])."""
    def one(r):
        eng = ls.engines[r]
        outs, hs = [eng.forward_inference(toks[:, :plen], 0).float().clone()], []
        if noise:
            with torch.inference_mode():  # the cache was allocated by forward_inference, under inference mode
                eng.fill_kv_cache_noise(std=0.5, seed=r)
        for j, ps in enumerate(positions):
            outs.append(eng.forward_inference(toks[:, plen + j:plen + j + 1], ps).float().clone())
            hs.append(torch.stack([eng.h[0][0], eng.h[1][0]]).clone())
        return outs, hs
    return ls.run(one)


ENGINE_CASES = [("7b", 2, 2, False), ("7b", 4, 2, False), ("7b", 8, 2, False), ("70b", 8, 2, False), ("70b", 2, 1, False),
                ("7b", 2, 2, True), ("70b", 8, 1, True)]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("arch,tp,n_layers,generic", ENGINE_CASES,
                         ids=[f"{a}_tp{t}_L{n}" + ("_gemv1_off" if g else "") for a, t, n, g in ENGINE_CASES])
def test_engine_tp_step_fused_matches_unfused(lockstep, arch, tp, n_layers, generic):
    """The engine's own TP decode step, every rank an engine in its own thread: the fused exchange (LL push in wo / w2,
    rank-ordered sum in w13 / the next wqkv / lm_head) against the same engines on the (stand-in) NCCL all-reduce of the
    same semantics gives identical logits and identical h on every rank after every step, bit for bit; the step counter
    counts the decode steps and no poll timed out.  Positions cross attention tile edges around 1024 and 2048 of a cache
    pre-filled with noise.  generic: B200_GEMV1 = 0, both ends of the exchange through the generic HMMA kernel."""
    ls = lockstep(tp)
    args = _engines(ls, arch, tp, n_layers)
    positions = [1022, 1023, 1024, 1025, 2047, 2048]
    toks = torch.randint(1, args["vocab_size"], (1, 5 + len(positions)), generator=torch.Generator().manual_seed(tp))
    with _knob(("B200_GEMV1", 0) if generic else None):
        for eng in ls.engines:
            eng.use_ar_fused = True
        fused = _schedule(ls, toks, 5, positions, noise=True)
        n_pre = ls.prechecked
        for eng in ls.engines:
            assert eng._ar is not None
            st = eng._ar["step"].cpu()
            assert int(st[0]) == len(positions) and int(st[1]) == 0, st.tolist()
            eng.use_ar_fused = False
        plain = _schedule(ls, toks, 5, positions, noise=True)
    # every consumer of a fused step was pre-checked: L w13, L - 1 wqkv (layer 0's has no delta) and the lm_head per rank
    assert n_pre == tp * len(positions) * 2 * n_layers, (n_pre, tp, len(positions), n_layers)
    assert ls.prechecked == n_pre, "the unfused run polled an exchange buffer"
    for r in range(tp):
        (lf, hf), (lp, hp) = fused[r], plain[r]
        for j, (a, b) in enumerate(zip(lf, lp)):
            assert _same(a, b), (arch, tp, "rank", r, "logits of step", j)
        for j, (a, b) in enumerate(zip(hf, hp)):
            assert _same(a, b), (arch, tp, "rank", r, "h after step", j)
        for j in range(len(lf)):
            assert _same(lf[j], fused[0][0][j]), (arch, tp, "rank", r, "disagrees with rank 0 on logits", j)
        for j in range(len(hf)):
            assert _same(hf[j], fused[0][1][j]), (arch, tp, "rank", r, "disagrees with rank 0 on h", j)
    assert all(bool(torch.isfinite(x).all()) for x in fused[0][0])
    print(f"\n[engine {arch} tp{tp} L{n_layers}{' gemv1 off' if generic else ''}] prompt + {len(positions)} steps: fused == "
          f"unfused on every rank, {n_pre} consumer launches pre-checked")


@pytest.fixture(scope="module")
def port_7b():
    """7B widths, 2 layers: master weights, their fake-quantised W4 form and the port's fp32 / fp16 logits (on the GPU)."""
    from oracle import omniquant, weights
    from oracle.llama_port import PortModel
    args = dict(ARCH["7b"], n_layers=2, max_seq_len=2112, max_batch_size=1)
    sd = weights.llama_state_dict(args, seed=0)
    sd_ref, recs = omniquant.fake_quantize_state_dict(sd, 4, 0)
    toks = weights.synthetic_tokens(1, 9, args["vocab_size"])
    refs = {}
    with torch.inference_mode():
        for dt in (torch.float32, torch.float16):
            port = PortModel("llama", args, {k: v.to(DEV) for k, v in sd_ref.items()}, dtype=dt)
            outs = [port.forward_inference(toks[:, :5].to(DEV), 0)]
            for j in range(4):
                outs.append(port.forward_inference(toks[:, 5 + j:6 + j].to(DEV), 5 + j))
            refs[dt] = torch.stack([o.float() for o in outs]).cpu().numpy()
            del port
    return sd, recs, toks, refs[torch.float32], refs[torch.float16]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("tp", [2, 4, 8])
def test_engine_tp_step_matches_the_port(lockstep, port_7b, tp):
    """Gathered logits of the fused TP engine (7B widths, 2 layers, master weights quantised then sharded) against the port
    in fp32 / fp16 on the same fake-quantised weights, with the rule of tests/test_tp_gpu.py, or the absolute allowance of
    two fp16 steps at the largest logit that tests/test_zzz_parity_widths_gpu.py grants these two-block 7B-width models."""
    sd, recs, toks, ref32, ref16 = port_7b
    ls = lockstep(tp)
    _engines(ls, "7b", tp, 2, sd=sd, recs=recs)
    out = _schedule(ls, toks, 5, [5, 6, 7, 8], noise=False)
    for r in range(1, tp):
        assert all(_same(a, b) for a, b in zip(out[r][0], out[0][0])), ("rank", r)
    assert all(int(e._ar["step"][0]) == 4 and int(e._ar["step"][1]) == 0 for e in ls.engines)
    got = torch.stack(out[0][0]).cpu().numpy()
    floor = float(np.abs(ref16 - ref32).max())
    e32, e16 = float(np.abs(got - ref32).max()), float(np.abs(got - ref16).max())
    ulp = 2.0 ** (math.floor(math.log2(max(float(np.abs(ref32).max()), 1e-3))) - 10)
    print(f"\n[engine 7b tp{tp} vs port] |eng-ref16|={e16:.3e} |eng-ref32|={e32:.3e} floor={floor:.3e} ulp={ulp:.3e}")
    assert np.isfinite(got).all() and (e16 <= 1e-3 or e32 <= 1.5 * floor + 5e-4 or e32 <= 2.05 * ulp)
