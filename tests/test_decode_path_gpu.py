"""GPU: the bs = 1 decode path kernel by kernel, at the widths of LLaMA-2 7B, 13B and one rank of 70B at TP = 8, with the
launch arguments the engine passes.

References run in float64 on the device.
  - gemv1 (csrc/gemv1.cu): the integer dot product is exact, so y = sum_g s_g (sum q x - z_g sum x) in float64 is the
    reference; the kernel may differ by fp16 rounding of the output plus fp32 noise of its plane recombination
    (2^-20 of the largest output per channel, 2^-17 with group scales: the bounds of test_gemv1_gpu.py).
  - RMSNorm prologue: x = fp16(fp16(h * rstd) * gamma) with the kernel's fp32 rstd = 1 / sqrtf(ssq / K + eps).  ssq sums
    K non-negative squares: each lane chains <= 16 fmaf (gemv1: two 8-element pieces; the fp16 HMMA kernel of the
    lm_head: <= 32), then a 5-level warp tree, then the 16 warp partials in order.  The depth is <= 37 (53), so ssq is
    within 37u (53u) of sum h^2, u = 2^-24.  The division by K and the eps add round once each (2u), sqrtf halves the
    relative error and rounds (0.5u), the reciprocal rounds (0.5u): rstd lies within 21u (30u) of rstd64, and h * rstd
    rounds once more: 21.5u (30.5u).  Hence
      * an index k is AMBIGUOUS when h_k * rstd64 lies within 2^-18 = 64u (relative) of an fp16 midpoint: only there can
        fp16(h * rstd) differ from the float64 rounding, by one fp16 step;
      * the kernel's rstd is one of the fp32 values within RSTD_ULPS = 32 ulps of rstd64 (31 ulps: 30.5u plus the rounding
        of rstd64 to fp32), so its x is one of at most 65 vectors, each computed here exactly.  The epilogue checks run
        against every such candidate and pass when one candidate explains every output.
  - Epilogues: the F16 launch on the same inputs computes the same fp32 y and rounds it the same way; it is held to the
    F16 bound above (and most of its outputs to fp16 of float64 y exactly), and every downstream value of the SiLU / QKV
    launch (RoPE in fp32 without FMA, SiLU in fp32 then fp16, the K / V cache slots) must follow from that fp16 y bit for bit.
  - PDL, L2 prefetches and ring depths change nothing the kernels compute: those cases demand bit identity.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import kvlayout, ops, quant  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig, _interleave_w13, rope_table  # noqa: E402
from oracle.numerics import SENT, fp16_sides as _fp16_sides, nan16, rstd64, tuned as _tuned  # noqa: E402
from oracle.numerics import x_candidates as _x_candidates  # noqa: E402

DEV = "cuda"
EPS = 1e-5
AMB_X = 2.0 ** -18       # relative distance from an fp16 midpoint below which fp16(h * rstd) is ambiguous (see above)
SILU_REL = 2.0 ** -20    # fp32 a / (1 + expf(-a)): expf <= 2 ulp, the add and the division 0.5 ulp each -> <= 3.5u << 16u
C_ACC16 = 2.0 ** -18     # fp32 tensor-core accumulation of the fp16 HMMA GEMV, relative to |x| . |w|^T (test_prefill_gpu)
# least fraction of an epilogue launch's fp16 y equal to fp16 of float64 y (best rstd candidate), per channel / grouped.
# Measured on an H100 80GB HBM3 (400 W limit) over every shape here: 0.998 to 1.0 per channel, 0.977 to 1.0 grouped.
MIN_EXACT = {False: 0.97, True: 0.9}
SLOT = 16384             # bytes of one weight-ring stage


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _nan16(*shape):
    return nan16(*shape, device=DEV)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _acc(y, G):
    """fp32 noise allowance of the integer-path GEMV output before its fp16 rounding (test_gemv1_gpu.py)."""
    return float(y.abs().max()) * (2.0 ** -20 if G == 1 else 2.0 ** -17) + 1e-7


def _f16_ratio(out, ref, G, extra=None):
    """largest |out - ref| / tol, tol = half an fp16 ulp of ref + the fp32 allowance (+ the prologue's ambiguity term)."""
    tol = ref.abs() * 2.0 ** -11 + _acc(ref, G)
    if extra is not None:
        tol = tol + extra * (1 + 2.0 ** -10)
    assert torch.isfinite(out).all()
    return float(((out.double().reshape(-1) - ref).abs() / tol).max())


def _weights(N, K, gs, seed, w13=False):
    """Random W4 codes, scales ~ 2 / (15 sqrt(K)) and zero points 0..15 -> (PackedLinear, float64 w_hat [N, K], groups).
    w13: the rows are the engine's interleaving of two halves (engine._interleave_w13)."""
    g = _gen(seed)
    G = 1 if gs == 0 else K // gs

    def one(n):
        q = torch.randint(0, 16, (n, K), generator=g, device=DEV, dtype=torch.uint8)
        s = ((0.75 + 0.5 * torch.rand(n, G, generator=g, device=DEV)) * 2.0 / (15 * math.sqrt(K))).half()
        return q, s, torch.randint(0, 16, (n, G), generator=g, device=DEV).half()
    if w13:
        (q1, s1, z1), (q3, s3, z3) = one(N // 2), one(N // 2)
        q, s, z = _interleave_w13(q1, q3), _interleave_w13(s1, s3), _interleave_w13(z1, z3)
    else:
        q, s, z = one(N)
    pl = quant.pack_quantized(q, s, z, 4, gs, DEV)
    w = ((q.double().reshape(N, G, -1) - z.double().reshape(N, G, 1)) * s.double().reshape(N, G, 1)).reshape(N, K)
    return pl, w, G


def _norm_inputs(K, seed):
    g = _gen(seed)
    resid = torch.randn(1, K, generator=g, device=DEV).half()
    delta = (0.3 * torch.randn(1, K, generator=g, device=DEV)).half()
    gamma = (1 + 0.2 * torch.randn(K, generator=g, device=DEV)).half()
    return resid, delta, gamma


def _x_ref(h, gamma, eps):
    """-> (x from float64 rstd, x with the other rounding of fp16(h * rstd), ambiguous mask)."""
    v = h.double().reshape(-1) * rstd64(h, eps)[0]
    near, alt, dist = _fp16_sides(v)
    g = gamma.double().reshape(-1)
    return (near * g).half(), (alt * g).half(), dist <= AMB_X * v.abs()


def _gemv(pl, out, **kw):
    ops.gemv(pl, 1, out=out, **kw)
    torch.cuda.synchronize()
    return out


# ------------------------------------------------------------------------------------------- epilogue checkers --------
def _f16_y(pl, W, G, resid, delta, gamma, label):
    """The F16 launch on an epilogue launch's inputs.  It computes the same fp32 y and rounds it the same way, so its output
    is the fp16 y that the SiLU / QKV epilogue starts from.  It must meet the F16 bound for one fp32 rstd of the derived
    window.  -> (fp16 y [N], fraction of y equal to fp16 of that candidate's float64 value)."""
    y16 = _gemv(pl, _nan16(1, pl.N), resid=resid, delta=delta, gamma=gamma, eps=EPS).reshape(-1)
    Y = W @ _x_candidates(resid + delta if delta is not None else resid, gamma, EPS).double().T
    r = [_f16_ratio(y16, Y[:, c], G) for c in range(Y.shape[1])]
    c = min(range(len(r)), key=r.__getitem__)
    assert r[c] <= 1.0, (label, r[c])
    return y16, float((y16.double() == _fp16_sides(Y[:, c])[0]).double().mean())


def _silu_mismatches(act, y16):
    """act [F] against the fp16 y [2F] of the w13 launch (rows r, r + 8 of every 16-row tile as w1 / w3): fp16(silu(a)) in
    fp32 then times b in fp16 (gemv1_core.cuh), either rounding of silu(a) where expf may tip it.  -> (mismatches, tipped)."""
    F = act.numel()
    t = y16.reshape(F // 8, 2, 8)
    a, b = t[:, 0].reshape(-1).double(), t[:, 1].reshape(-1).double()
    sl = a / (1 + torch.exp(-a))
    sn, sa, sd = _fp16_sides(sl)
    amb = sd <= SILU_REL * sl.abs()
    got = act.double().reshape(-1)
    ok = (got == (sn * b).half().double()) | (amb & (got == (sa * b).half().double()))
    return int((~ok).sum()), int(amb.sum())


def _rot(y16, cs):
    """fp32 RoPE on the CPU as separate multiplies and adds (llama.py:59-77): y16 [rows] fp16 values of whole heads."""
    p = y16.float().cpu().reshape(-1, 64, 2)
    e, o = p[..., 0], p[..., 1]
    c, s = cs[:, 0], cs[:, 1]
    return torch.stack([e * c - o * s, e * s + o * c], dim=-1).reshape(-1).half()


def _qkv_launch(pl, nq, nkv, S, ps, rope, resid, delta, gamma, kc=None, vt=None, **kw):
    Hkv = nkv // 128
    kc = kvlayout.k_to_engine(_nan16(1, Hkv, S, 128)) if kc is None else kc
    vt = _nan16(1, Hkv, S // 32, 128, 32) if vt is None else vt
    q_out = _nan16(1, nq)
    h_out = _nan16(1, pl.K)
    pos = torch.tensor([ps], dtype=torch.int32, device=DEV)
    qkv = dict(n_q_rows=nq, n_kv_rows=nkv, rope=rope, pos=pos, tokens_per_seq=1, kcache=kc, vtcache=vt, cache_seq=S,
               prefetch_kv=kw.pop("prefetch_kv", False))
    _gemv(pl, q_out, resid=resid, delta=delta, h_out=h_out, gamma=gamma, eps=EPS, epilogue=ops.B200_EPI_QKV, qkv=qkv, **kw)
    return q_out, h_out, kc, vt


def _check_qkv(pl, W, G, nq, nkv, S, ps, rope, resid, delta, gamma, label):
    """One QKV launch at position ps into a sentinel cache: q out and K are the fp32 RoPE of the fp16 y bit for bit, V is
    fp16 y, K / V land at exactly (head, ps) and nothing else in either cache changes.  -> exact fraction of y."""
    Hkv, nr = nkv // 128, nq + nkv
    q_out, _, kc, vt = _qkv_launch(pl, nq, nkv, S, ps, rope, resid, delta, gamma)
    assert int((kc.view(torch.int16) != SENT).sum()) == Hkv * 128, label
    assert int((vt.view(torch.int16) != SENT).sum()) == Hkv * 128, label
    k_can, v_can = kvlayout.k_from_engine(kc), kvlayout.v_from_engine(vt)
    y16, exact = _f16_y(pl, W, G, resid, delta, gamma, label)
    got_rot = torch.cat([q_out.reshape(-1), k_can[0, :, ps].reshape(-1)]).float().cpu()
    bad = int((got_rot != _rot(y16[:nr], rope[ps].cpu()).float()).sum())
    bad += int((v_can[0, :, ps].reshape(-1).view(torch.int16) != y16[nr:].view(torch.int16)).sum())
    assert bad == 0, (label, bad)
    return exact


# ------------------------------------------------------------------------------------- 1. gemv1 vs float64 ----------
#          name             N      K     launch   Hq  Hkv
SHAPES = [("7b_wqkv",     12288,  4096, "qkv",   32, 32),
          ("7b_wo",        4096,  4096, "f16",    0,  0),
          ("7b_w13",      22016,  4096, "silu",   0,  0),
          ("7b_w2",        4096, 11008, "f16",    0,  0),
          ("13b_wqkv",    15360,  5120, "qkv",   40, 40),
          ("13b_w13",     27648,  5120, "silu",   0,  0),
          ("13b_w2",       5120, 13824, "f16",    0,  0),
          ("70b_tp8_wqkv", 1280,  8192, "qkv",    8,  1),
          ("70b_tp8_w13",  7168,  8192, "silu",   0,  0),
          ("70b_tp8_w2",   8192,  3584, "f16",    0,  0)]


@pytest.mark.timeout(120)
@pytest.mark.parametrize("gs", [0, 128, 64], ids=["pc", "g128", "g64"])
@pytest.mark.parametrize("name,N,K,form,Hq,Hkv", SHAPES, ids=[s[0] for s in SHAPES])
def test_gemv1_engine_launch_matches_float64(name, N, K, form, Hq, Hkv, gs):
    seed = N + K + gs
    pl, W, G = _weights(N, K, gs, seed, w13=form == "silu")
    label = f"{name}/{gs or 'pc'}"
    if form == "f16":
        x = torch.randn(1, K, generator=_gen(seed), device=DEV).half()
        r = _f16_ratio(_gemv(pl, _nan16(1, N), xin=x), W @ x.double().reshape(-1), G)
        print(f"\n[{label}] F16 worst err/tol {r:.3f}")
        assert r <= 1.0, (label, r)
        return
    resid, delta, gamma = _norm_inputs(K, seed)
    # RMSNorm prologue, F16 epilogue: h_out is the fp16 residual add bit for bit, x meets both bounds
    rs = []
    for dl in (delta, None):
        h_out = _nan16(1, K)
        out = _gemv(pl, _nan16(1, N), resid=resid, delta=dl, h_out=h_out, gamma=gamma, eps=EPS)
        h = resid + dl if dl is not None else resid
        assert torch.equal(h_out.view(torch.int16), h.view(torch.int16)), label
        xr, xa, amb = _x_ref(h, gamma, EPS)
        ref = W @ xr.double().reshape(-1)
        A = W.abs() @ ((xa.double() - xr.double()).abs() * amb).reshape(-1)
        r_amb = _f16_ratio(out, ref, G, A)
        Y = W @ _x_candidates(h, gamma, EPS).double().T
        r_cand = min(_f16_ratio(out, Y[:, c], G) for c in range(Y.shape[1]))
        assert r_amb <= 1.0 and r_cand <= 1.0, (label, dl is None, r_amb, r_cand)
        rs.append((r_amb, r_cand, int(amb.sum())))
    # exact-norm probe: eps = 0 and |h| = 2^-2 everywhere make rstd exact and x = +-gamma
    sign = torch.where(torch.rand(K, generator=_gen(seed + 1), device=DEV) < 0.5, -1.0, 1.0)
    r_probe = 0.0
    for with_delta in (True, False):
        rp = (sign * (0.1875 if with_delta else 0.25)).half().reshape(1, K)
        dp = (sign * 0.0625).half().reshape(1, K) if with_delta else None
        out = _gemv(pl, _nan16(1, N), resid=rp, delta=dp, gamma=gamma, eps=0.0)
        r_probe = max(r_probe, _f16_ratio(out, W @ (sign.double() * gamma.double()), G))
    assert r_probe <= 1.0, (label, r_probe)
    # the launch's own epilogue
    if form == "silu":
        act = _gemv(pl, _nan16(1, N // 2), resid=resid, delta=delta, gamma=gamma, eps=EPS, epilogue=ops.B200_EPI_SILU)
        y16, best = _f16_y(pl, W, G, resid, delta, gamma, label)
        bad, tipped = _silu_mismatches(act, y16)
        assert bad == 0, (label, bad)
        epi = f"SiLU: y exact {best:.4f}, silu rounding tipped at {tipped}/{N // 2}"
    else:
        S = 2048
        rope = rope_table(128, 2 * S, 10000.0, None).to(DEV)
        best = _check_qkv(pl, W, G, Hq * 128, Hkv * 128, S, 1023, rope, resid, delta, gamma, label)
        epi = f"QKV: y exact {best:.4f}"
    print(f"\n[{label}] F16 worst err/tol: ambiguity bound {max(r[0] for r in rs):.3f}, best rstd "
          f"{max(r[1] for r in rs):.3f}, exact-norm probe {r_probe:.3f}; ambiguous k {rs[0][2]}/{K}; {epi}")
    assert best >= MIN_EXACT[G > 1], (label, best)


@pytest.mark.timeout(120)
@pytest.mark.parametrize("Hq,Hkv", [(8, 1), (32, 8), (32, 32)])
def test_gemv1_qkv_epilogue_at_cache_edges(Hq, Hkv):
    """K lands at (head, pos) through the odd / even chunk swizzle, V at row pos & 31 of tile pos >> 5, q gets the RoPE of
    row pos; the rest of both caches is byte-unchanged."""
    S, K = 2048, 4096
    nq, nkv = Hq * 128, Hkv * 128
    pl, W, G = _weights(nq + 2 * nkv, K, 0, seed=Hq * 100 + Hkv)
    rope = rope_table(128, 2 * S, 10000.0, None).to(DEV)
    resid, delta, gamma = _norm_inputs(K, seed=Hkv)
    fr = []
    for ps in (0, 1, 31, 32, 33, 1023, S - 1):
        fr.append(_check_qkv(pl, W, G, nq, nkv, S, ps, rope, resid, delta, gamma, f"Hkv={Hkv} pos={ps}"))
    print(f"\n[qkv Hq={Hq} Hkv={Hkv}] exact fraction per position {[round(f, 4) for f in fr]}")
    assert min(fr) >= MIN_EXACT[False]


@pytest.mark.timeout(120)
@pytest.mark.parametrize("gs", [0, 128], ids=["pc", "g128"])
def test_gemv1_epilogue_beyond_the_staged_tiles(gs):
    """More than kMaxLocal = 16 tiles per CTA: the epilogue reads scales and RoPE values straight from global memory."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    K, S = 256, 64

    def most_tiles(N):
        n_tiles = N // 16
        return -(-n_tiles // min(n_tiles, sms))
    N = 16 * (16 * sms + 37)
    assert most_tiles(N) > 16
    pl, W, G = _weights(N, K, gs, seed=N + gs)
    x = torch.randn(1, K, generator=_gen(gs), device=DEV).half()
    r = _f16_ratio(_gemv(pl, _nan16(1, N), xin=x), W @ x.double().reshape(-1), G)
    assert r <= 1.0, r
    Hkv, Hq = 8, 2 * sms + 8  # the q rows alone exceed 16 tiles per CTA
    nq, nkv = Hq * 128, Hkv * 128
    assert (nq // 16) > 16 * sms and most_tiles(nq + 2 * nkv) > 16
    pl, W, G = _weights(nq + 2 * nkv, K, gs, seed=nq + gs)
    rope = rope_table(128, 2 * S, 10000.0, None).to(DEV)
    resid, delta, gamma = _norm_inputs(K, seed=gs + 3)
    fr = [_check_qkv(pl, W, G, nq, nkv, S, ps, rope, resid, delta, gamma, f"non-staged pos={ps}") for ps in (33, S - 1)]
    print(f"\n[non-staged {gs or 'pc'}] {most_tiles(nq + 2 * nkv)} tiles per CTA; F16 worst err/tol {r:.3f}; "
          f"QKV exact {[round(f, 4) for f in fr]}")
    assert min(fr) >= MIN_EXACT[G > 1]


# ------------------------------------------------------------------ 2. launch arguments that must not change results --
def _ndiff(a, b):
    n = 0
    for x, y in zip(a, b):
        if x is None:
            continue
        dt = torch.int16 if x.element_size() == 2 else torch.int32
        n += int((x.view(dt) != y.view(dt)).sum())
    return n


@pytest.mark.timeout(180)
def test_prefetch_pdl_and_ring_depth_leave_every_launch_bit_identical():
    D, F, S, H = 4096, 11008, 2048, 32
    lins = {"wqkv": quant.random_packed(4, 3 * H * 128, D, 0, DEV, 1), "wo": quant.random_packed(4, D, D, 0, DEV, 2),
            "w13": quant.random_packed(4, 2 * F, D, 0, DEV, 3), "w2": quant.random_packed(4, D, F, 0, DEV, 4)}
    nxt = {"wqkv": "wo", "wo": "w13", "w13": "w2", "w2": "wqkv"}
    small = quant.random_packed(4, 64, 256, 0, DEV, 5)  # 8 KB: shorter than one prefetch window
    g = _gen(7)
    resid, delta, gamma = _norm_inputs(D, 8)
    gamma_next = (1 + 0.2 * torch.randn(D, generator=g, device=DEV)).half()
    xa = torch.randn(1, D, generator=g, device=DEV).half()
    xf = (0.1 * torch.randn(1, F, generator=g, device=DEV)).half()
    kc0 = (0.5 * torch.randn(1, H, S, 128, generator=g, device=DEV)).half()
    vt0 = (0.5 * torch.randn(1, H, S // 32, 128, 32, generator=g, device=DEV)).half()
    rope = rope_table(128, 2 * S, 10000.0, None).to(DEV)

    def run(name, ps, **kw):
        pl = lins[name]
        kc, vt = kc0.clone(), vt0.clone()
        if name == "wqkv":
            q_out, h_out, _, _ = _qkv_launch(pl, H * 128, H * 128, S, ps, rope, resid, delta, gamma, kc=kc, vt=vt, **kw)
            return q_out, h_out, kc, vt
        if name == "w13":
            h_out = _nan16(1, D)
            out = _gemv(pl, _nan16(1, F), resid=resid, delta=delta, h_out=h_out, gamma=gamma, eps=EPS,
                        epilogue=ops.B200_EPI_SILU, **kw)
            return out, h_out, kc, vt
        return _gemv(pl, _nan16(1, pl.N), xin=xa if name == "wo" else xf, **kw), None, kc, vt

    def head(pl):
        return (pl.qweight, pl.qweight.numel(), pl.N // 16)
    report = []
    for name, pl in lins.items():
        for ps in ((33, S - 1) if name == "wqkv" else (0,)):
            base = run(name, ps)
            nx = head(lins[nxt[name]])
            variants = [("prefetch", dict(prefetch=nx)), ("prefetch<window", dict(prefetch=head(small))),
                        ("prefetch_const", dict(prefetch_const=gamma_next)), ("use_pdl", dict(use_pdl=True))]
            variants += [(f"ring{n}", dict(ring_bytes=n * SLOT)) for n in (2, 3, 8, 24)]
            every = dict(prefetch=nx, prefetch_const=gamma_next, use_pdl=True)
            if name == "wqkv":
                variants.append(("prefetch_kv", dict(prefetch_kv=True)))
                every["prefetch_kv"] = True
            variants.append(("all", every))
            n = 0
            for lab, kw in variants:
                d = _ndiff(run(name, ps, **kw), base)
                assert d == 0, (name, ps, lab, d)
                n += 1
            for knob, val in (("B200_PF_EARLY", 1), ("B200_SELF_PF_KB", 64), ("B200_STREAM_EF", 0),
                              ("B200_QKV_RING_KB", 48)):
                with _tuned(knob, val):
                    d = _ndiff(run(name, ps, **every), base)
                assert d == 0, (name, ps, knob, d)
                n += 1
            report.append(f"{name}@{ps}: {n} variants, 0 differing elements")
    # attention with the wo prefetch, with and without PDL and the early-prefetch knob
    q = torch.randn(1, H * 128, generator=g, device=DEV).half()
    for ps in (33, S - 1):
        pos = torch.tensor([ps], dtype=torch.int32, device=DEV)

        def attn(**kw):
            ns = ops.attn_split(1, H, S)
            ws = torch.zeros(ops.attn_workspace_bytes(1, H, ns), dtype=torch.uint8, device=DEV)
            cnt = torch.zeros(H, dtype=torch.int32, device=DEV)
            out = _nan16(1, H * 128)
            ops.attn_decode(q, kc0, vt0, pos, out, T=1, Hq=H, Hkv=H, cache_seq=S, tokens_per_seq=1, max_kv_len=S, ws=ws,
                            counters=cnt, n_split=ns, **kw)
            torch.cuda.synchronize()
            return (out,)
        base = attn()
        for kw in (dict(prefetch=head(lins["wo"])), dict(prefetch=head(small)), dict(use_pdl=True, prefetch=head(lins["wo"]))):
            assert _ndiff(attn(**kw), base) == 0, (ps, list(kw))
        with _tuned("B200_PF_EARLY", 1):
            assert _ndiff(attn(use_pdl=True, prefetch=head(lins["wo"])), base) == 0, ps
        report.append(f"attn@{ps}: 4 variants, 0 differing elements")
    print("\n" + "\n".join(report))


# ------------------------------------------------------------------------------------------------ 3. lm_head --------
@pytest.mark.timeout(120)
@pytest.mark.parametrize("N,K", [(32000, 4096), (32000, 5120), (32000, 8192), (4000, 8192)])
def test_lm_head_rmsnorm_f32_matches_float64(N, K):
    """The fp16 HMMA GEMV (gemv.cu, bits = 16) at T = 1 with the RMSNorm prologue and the F32 epilogue: the final norm and
    the vocabulary projection of a decode step (N = 4000: one TP = 8 shard of a 32000 vocabulary)."""
    g = _gen(N + K)
    w = ((torch.rand(N, K, generator=g, device=DEV) * 2 - 1) / math.sqrt(K)).half()
    pl = quant.pack_fp16(w, DEV)
    resid, delta, gamma = _norm_inputs(K, N + K)
    out = torch.full((1, N), float("nan"), device=DEV)
    _gemv(pl, out, resid=resid, delta=delta, gamma=gamma, eps=EPS, epilogue=ops.B200_EPI_F32)
    got = out.double().reshape(-1)
    assert torch.isfinite(out).all()
    assert torch.equal(out, out.half().float())  # the logits are fp16 values (the reference's fp16 head)
    h = resid + delta
    wd = w.double()
    xr, xa, amb = _x_ref(h, gamma, EPS)
    ref = wd @ xr.double().reshape(-1)
    A = wd.abs() @ ((xa.double() - xr.double()).abs() * amb).reshape(-1)
    tol = ref.abs() * 2.0 ** -11 + C_ACC16 * (wd.abs() @ xr.double().abs().reshape(-1)) + A * (1 + 2.0 ** -10) + 1e-7
    ratio = float(((got - ref).abs() / tol).max())
    X = _x_candidates(h, gamma, EPS).double()
    Y, M = wd @ X.T, wd.abs() @ X.abs().T
    r_cand = float(((got[:, None] - Y).abs() / (Y.abs() * 2.0 ** -11 + C_ACC16 * M + 1e-7)).amax(0).min())
    top = ref.topk(2)
    margin = float(top.values[0] - top.values[1])
    need = float(tol[top.indices[0]] + tol[top.indices[1]])
    print(f"\n[lm_head N={N} K={K}] worst err/tol: ambiguity bound {ratio:.3f}, best rstd {r_cand:.3f}; ambiguous k "
          f"{int(amb.sum())}/{K}; top-2 margin {margin:.3e} vs bound {need:.3e}")
    assert ratio <= 1.0 and r_cand <= 1.0, (ratio, r_cand)
    if margin > need:
        assert int(got.argmax()) == int(top.indices[0])


# ------------------------------------------------------------------------------------ 4. the decode chain -------------
LLAMA7B = dict(dim=4096, n_heads=32, ffn_hidden=11008)
LLAMA70B_TP8 = dict(dim=8192, n_heads=64, n_kv_heads=8, ffn_hidden=28672, tp_world=8, tp_rank=0)
STEPS = 3


@pytest.mark.timeout(180)
@pytest.mark.parametrize("gs", [0, 128], ids=["w4", "w4g128"])
@pytest.mark.parametrize("arch", [LLAMA7B, LLAMA70B_TP8], ids=["7b", "70b_tp8_rank"])
def test_decode_chain_bit_identical_under_pdl_prefetch_and_graphs(arch, gs):
    """PDL off with no prefetch is plain stream order: every other way of running the same steps (PDL, L2 prefetches, the
    captured decode graph, the captured greedy loop) must give the same logits and the same whole KV cache, bit for bit."""
    cfg = EngineConfig(kind="llama", n_layers=2, vocab_size=32000, max_seq_len=2048, bits=4, group_size=gs, **arch)
    eng = DecodeEngine(cfg, DEV)
    eng.shard_only = cfg.tp_world > 1  # one rank's kernels, without the collectives
    eng.load_random(seed=11)
    eng.allocate_kv_cache(1)
    eng.fill_kv_cache_noise(seed=12)
    k0, v0 = eng.kcache.clone(), eng.vtcache.clone()
    S = eng.cache_seq
    toks = torch.randint(0, cfg.vocab_size, (STEPS,), generator=_gen(13), device=DEV)

    def reset(tok, ps, pdl=True, pf=1):
        eng.use_pdl, eng.prefetch_bytes = pdl, pf
        eng.kcache.copy_(k0)
        eng.vtcache.copy_(v0)
        eng.tokens[:1].copy_(tok.reshape(1))
        eng.pos[:1].fill_(ps)

    def state(logits):
        torch.cuda.synchronize()
        return [torch.stack(logits), eng.kcache.clone(), eng.vtcache.clone()]

    def eager(start, pdl, pf):
        reset(toks[0], start, pdl, pf)
        lg = []
        for j in range(STEPS):
            eng.tokens[:1].copy_(toks[j:j + 1])
            eng.pos[:1].fill_(start + j)
            lg.append(eng._step(1, 1, S).clone())
        return state(lg)

    def greedy_eager(start):
        reset(toks[0], start)
        lg = []
        for _ in range(4):
            logits = eng._step(1, 1, S)
            ops.argmax(logits.contiguous(), eng.tokens, 1, logits.shape[-1])
            ops.advance_pos(eng.pos, 1, 1)
            lg.append(torch.cat([logits.reshape(-1), eng.tokens[:1].float()]))
        return state(lg)

    eng.use_pdl, eng.prefetch_bytes = True, 1
    greedy, _ = eng.capture_greedy_loop(1)
    report = []
    for start in (31, 32, 1023, 2047 - STEPS):
        ref = eager(start, False, 0)
        for pdl, pf in ((False, 1), (True, 0), (True, 1)):
            d = _ndiff(eager(start, pdl, pf), ref)
            assert d == 0, (start, pdl, pf, d)
        pdl_run = eager(start, True, 1)
        reset(toks[0], start)
        lg = [eng.decode_step(toks[j:j + 1], start + j).clone() for j in range(STEPS)]
        d_graph = _ndiff(state(lg), pdl_run)
        assert d_graph == 0, (start, "graph", d_graph)
        ge = greedy_eager(start)
        reset(toks[0], start)
        lg = []
        for _ in range(4):
            greedy.replay()
            lg.append(torch.cat([eng.greedy_logits.reshape(-1), eng.tokens[:1].float()]))
        d_greedy = _ndiff(state(lg), ge)
        assert d_greedy == 0, (start, "greedy", d_greedy)
        report.append(start)
    print(f"\n[chain {cfg.dim} gs={gs}] starts {report}: PDL x prefetch, graph and greedy-loop replays: 0 differing elements")
