"""GPU: the wgmma W4A16 prefill GEMM (csrc/prefill.cu) and the prompt path built on it, through the C-ABI.

GEMM checker: ref = x . w_hat^T in float64, with w_hat = fp16(fp16(q - z) * s16) -- the reference's fake-quantised
weight, which the kernel rebuilds bit for bit before the tensor cores multiply it.
  - sparse probes (one or two power-of-two nonzeros per token) make the fp32 accumulation exact, so every output must
    equal fp16(ref) bit for bit: they pin the dequant, the k order inside a 64-block, the stage ring and the epilogue map;
  - random inputs get an elementwise bound |out - ref| <= ulp16(ref) + C_ACC * (|x| . |w_hat|^T) and a minimum fraction of
    outputs equal to fp16(ref).
Elementwise prompt kernels: torch at the reference's rounding points, bit for bit.
Prompt checker: the CPU port (bit-pinned to the unmodified reference) in fp32 / fp16, prompts from position 0 and
continuation prompts at start_pos > 0.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import kvlayout, ops, quant  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig, _interleave_w13, rope_table  # noqa: E402
from oracle import cases, omniquant, weights  # noqa: E402
from oracle.llama_port import PortModel  # noqa: E402

DEV = "cuda"
# fp32 tensor-core accumulation allowance, relative to |x| . |w_hat|^T.  Measured on an H100 80GB HBM3 (700 W limit)
# over every shape below: at most 2^-20.7 (K = 28672), so 2^-18 leaves a margin of 6.5x.
C_ACC = 2.0 ** -18


def _min_exact(K):
    """Least fraction of random-input outputs equal to fp16(ref): fp32 accumulation noise grows like sqrt(K).  Measured
    misses (same H100): 1.2% at K = 512, 1.7% at 4096, 4.9% at 13824, 9.0% at 28672, about half of 2^-10 sqrt(K)."""
    return 1.0 - 2.0 ** -10 * math.sqrt(K)


# zero points across the packed format's whole range, [-1024, 1024]
ZEROS = [-1024, -1023, -517, -16, -1, 0, 1, 7, 8, 15, 16, 255, 1000, 1024]


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _bits(t):
    """fp16 bit pattern with -0 folded into +0 (the GEMM's accumulators start at +0)."""
    return (t + 0.0).view(torch.int16)


def _ulp16(a):
    """fp16 spacing at |a| (subnormal spacing 2^-24 below 2^-14)."""
    e = torch.floor(torch.log2(a.double().abs().clamp_min(2.0 ** -24)))
    return torch.exp2(e.clamp_min(-14) - 10)


def _nan16(*shape, pattern=0x7E5A):
    """fp16 tensor holding one NaN bit pattern: a sentinel no kernel writes."""
    return torch.full(shape, pattern, dtype=torch.int16, device=DEV).view(torch.float16)


def _uniform_qsz(N, K, seed, G=1):
    """Random codes, zero point 8, scales ~ 2 / (15 sqrt(K)): weights ~ U(-1/sqrt(K), 1/sqrt(K))."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randint(0, 16, (N, K), generator=g, dtype=torch.uint8)
    s = ((0.75 + 0.5 * torch.rand(N, G, generator=g)) * 2.0 / (15 * math.sqrt(K))).half()
    return q, s, torch.full((N, G), 8.0).half()


def _extreme_qsz(N, K, seed, G=1):
    """Every zero point of ZEROS meets each kind of scale: fp16(1e-5) (subnormal), 2^-14 (smallest normal), 1e-3 and
    random ones up to 0.05, so |w_hat| <= 1039 * 0.05 stays finite."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randint(0, 16, (N, K), generator=g, dtype=torch.uint8)
    r = torch.arange(N * G).reshape(N, G)
    z = torch.tensor(ZEROS, dtype=torch.float32)[r % len(ZEROS)]
    fixed = torch.tensor([float(torch.tensor(1e-5).half()), 2.0 ** -14, 1e-3])
    kind = (r // len(ZEROS)) % 4
    s = torch.where(kind < 3, fixed[kind.clamp_max(2)], 1e-4 + 0.05 * torch.rand(N, G, generator=g))
    return q, s.half(), z.half()


QSZ = {"uniform": _uniform_qsz, "extreme": _extreme_qsz}


def _linear(q, s, z):
    """-> (PackedLinear on the GPU, w_hat fp16 [N, K] on the GPU) for one W4 linear, per-channel when s has one column."""
    N, K = q.shape
    gs = K // s.shape[1]
    pl = quant.pack_quantized(q, s, z, 4, 0 if gs == K else gs, DEV)
    return pl, quant.dequantize(q.to(DEV), s.to(DEV), z.to(DEV), gs)


def _gemm(pl, x, T):
    out = _nan16(T, pl.N)
    ops.prefill_gemm_w4(pl, x, out, T)
    torch.cuda.synchronize()
    return out


def _check_random(pl, w_hat, x, T, label):
    """Elementwise bound and exact fraction for one launch; returns (largest err / tol, implied C, exact fraction)."""
    out = _gemm(pl, x, T)
    xd, wd = x[:T].double(), w_hat.double()
    ref = xd @ wd.T
    mag = xd.abs() @ wd.abs().T
    err = (out.double() - ref).abs()
    ulp = _ulp16(ref)
    ratio = float((err / (ulp + C_ACC * mag)).max())
    c_seen = float(((err - ulp).clamp_min(0) / mag.clamp_min(1e-30)).max())
    exact = float((_bits(out) == _bits(ref.half())).double().mean())
    assert torch.isfinite(out).all(), label
    assert float(err.max()) <= 2.0 ** -10 * float(ref.abs().max()) + 1e-4, label  # one fp16 ulp of the largest output
    assert ratio <= 1.0, (label, ratio, c_seen)
    assert exact >= _min_exact(pl.K), (label, exact)
    return ratio, c_seen, exact


# ---------------------------------------------------------------------------------------------------- the GEMM --------
@pytest.mark.timeout(300)
@pytest.mark.parametrize("N,K,T,wts", [
    # the product quantiser on symmetric uniform weights (zero points 7 or 8)
    *[pytest.param(N, K, T, "quantised", id=f"{N}-{K}-{T}") for N, K, T in
      [(128, 64, 1), (128, 256, 16), (256, 512, 77), (4096, 4096, 256), (1024, 11008, 300), (384, 1536, 513)]],
    (256, 512, 1, "extreme"), (384, 1024, 300, "extreme"), (256, 4096, 256, "extreme"),
    # real LLaMA-2 widths (7B wqkv / w2, 13B wqkv / w2, 70B w2); N / 128 > 132 CTAs is more than one wave
    (22016, 4096, 200, "uniform"), (22016, 4096, 256, "uniform"), (4096, 11008, 200, "uniform"),
    (4096, 11008, 256, "uniform"), (15360, 5120, 200, "uniform"), (15360, 5120, 256, "uniform"),
    (5120, 13824, 200, "uniform"), (5120, 13824, 256, "uniform"), (8192, 28672, 200, "uniform"),
    (8192, 28672, 256, "uniform")])
def test_prefill_gemm_w4_matches_fake_quantised_linear(N, K, T, wts):
    if wts == "quantised":
        g = torch.Generator().manual_seed(N + K + T)
        w = ((torch.rand(N, K, generator=g) * 2 - 1) / math.sqrt(K)).half()
        q, s, z, _ = quant.quantize_weight(w, 4, 0)
        pl, w_hat = _linear(q, s, z)
        x = torch.randn(T, K, generator=g).half().to(DEV)
    else:
        pl, w_hat = _linear(*QSZ[wts](N, K, seed=N + K + T))
        x = torch.randn(T, K, generator=torch.Generator(device=DEV).manual_seed(N + T), device=DEV).half()
    ratio, c_seen, exact = _check_random(pl, w_hat, x, T, (N, K, T, wts))
    print(f"\n[gemm {N}x{K} T={T} {wts}] max err/tol={ratio:.3f} implied C=2^{math.log2(max(c_seen, 1e-30)):.1f} "
          f"exact={exact:.4f}")


@pytest.mark.timeout(300)
def test_prefill_gemm_w4_every_chunk_count_and_residue():
    """Every NC = 1..8 instance and every token residue inside a 32-token chunk, then multi-launch prompts."""
    N, K = 256, 512
    pl, w_hat = _linear(*_uniform_qsz(N, K, seed=1))
    g = torch.Generator(device=DEV).manual_seed(1)
    worst = (0.0, 0.0, 1.0)
    for T in list(range(1, 257)) + [257, 288, 511, 512, 513, 769]:
        x = torch.randn(T, K, generator=g, device=DEV).half()
        r = _check_random(pl, w_hat, x, T, T)
        worst = (max(worst[0], r[0]), max(worst[1], r[1]), min(worst[2], r[2]))
    print(f"\n[gemm chunk sweep 256x512] max err/tol={worst[0]:.3f} implied C=2^{math.log2(max(worst[1], 1e-30)):.1f} "
          f"min exact={worst[2]:.4f}")


@pytest.mark.timeout(180)
@pytest.mark.parametrize("probe,K,T,wts", [("one", 256, 256, "uniform"), ("one", 4096, 4096, "uniform"),
                                           ("two", 1024, 256, "uniform"), ("two", 4096, 300, "uniform"),
                                           ("one", 256, 256, "extreme"), ("one", 1024, 300, "extreme")])
def test_prefill_gemm_w4_sparse_probe_is_exact(probe, K, T, wts):
    """one: x[t] = +-2^e_t . e_{k_t}  ->  out[t, :] = fp16(+-2^e_t . w_hat[:, k_t]), bit for bit.  With K = T = 256 every
    position of every 64-block is probed; otherwise k_t is drawn from a random permutation of K.
    two: nonzeros at k-blocks 1..5 apart, so the sum crosses the 4-stage ring; terms are powers of two times w_hat with
    |w_hat| in [s, 8 s], within 2^12 of each other, so the fp32 sum is exact and out = fp16(a + b)."""
    N = 384  # three CTAs, each with both consumer warpgroups
    pl, w_hat = _linear(*QSZ[wts](N, K, seed=K + T))
    g = torch.Generator().manual_seed(K * 7 + T)
    t = torch.arange(T)
    x = torch.zeros(T, K, dtype=torch.float64)
    sign = lambda: torch.randint(0, 2, (T,), generator=g).double() * 2 - 1  # noqa: E731
    if probe == "one":
        kt = t if K == T else torch.randperm(K, generator=g)[:T]
        x[t, kt] = sign() * torch.exp2((t % 7 - 3).double())
    else:
        KB, d = K // 64, 1 + t % 5
        kb1 = (torch.rand(T, generator=g) * (KB - d)).long()
        k1 = kb1 * 64 + torch.randint(0, 64, (T,), generator=g)
        k2 = (kb1 + d) * 64 + torch.randint(0, 64, (T,), generator=g)
        x[t, k1] = sign() * torch.exp2((t % 5 - 2).double())
        x[t, k2] = sign() * torch.exp2(((t // 5) % 5 - 2).double())
    x = x.half().to(DEV)
    out = _gemm(pl, x, T)
    ref = (x.double() @ w_hat.double().T).half()
    bad = _bits(out) != _bits(ref)
    if bad.any():
        tb, nb = [int(v) for v in torch.nonzero(bad)[0]]
        raise AssertionError(f"{int(bad.sum())} of {bad.numel()} outputs differ; first at token {tb}, row {nb}: "
                             f"{float(out[tb, nb])} != {float(ref[tb, nb])}")


@pytest.mark.timeout(180)
@pytest.mark.parametrize("T", [1, 77, 256, 300])
def test_prefill_gemm_w4_touches_only_its_rows(T):
    """Rows >= T of out keep their bit pattern, and x rows >= T (NaN here) do not reach any output."""
    N, K = 256, 512
    pl, _ = _linear(*_uniform_qsz(N, K, seed=T))
    g = torch.Generator(device=DEV).manual_seed(T)
    x = torch.randn(T, K, generator=g, device=DEV).half()
    x_guard = torch.cat([x, _nan16(64, K)])
    out_guard = _nan16(T + 64, N, pattern=0x7D3C)
    ops.prefill_gemm_w4(pl, x_guard, out_guard, T)
    clean = _gemm(pl, x, T)
    assert torch.equal(out_guard[T:].view(torch.int16), _nan16(64, N, pattern=0x7D3C).view(torch.int16))
    assert torch.equal(out_guard[:T].view(torch.int16), clean.view(torch.int16))


@pytest.mark.timeout(180)
def test_prefill_gemm_w4_streams_and_determinism():
    """Back-to-back launches of different NC on a side stream equal the default-stream results bit for bit; so do two
    identical runs."""
    N, K = 512, 1024
    pl, _ = _linear(*_uniform_qsz(N, K, seed=5))
    g = torch.Generator(device=DEV).manual_seed(5)
    Ts = [33, 256, 7, 300, 161, 64]
    xs = [torch.randn(T, K, generator=g, device=DEV).half() for T in Ts]
    base = [_gemm(pl, x, T) for x, T in zip(xs, Ts)]
    again = [_gemm(pl, x, T) for x, T in zip(xs, Ts)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        outs = [_nan16(T, N) for T in Ts]
        for x, o, T in zip(xs, outs, Ts):
            ops.prefill_gemm_w4(pl, x, o, T)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for T, a, b, c in zip(Ts, base, again, outs):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), T
        assert torch.equal(a.view(torch.int16), c.view(torch.int16)), T


@pytest.mark.timeout(180)
@pytest.mark.parametrize("gs", [0, 128])
@pytest.mark.parametrize("T", [1, 8])
def test_decode_gemv_on_extreme_zero_points(gs, T):
    """The decode GEMV on the same far-from-8 zero points and subnormal scales (its zero-point term grows with |z|)."""
    N, K = 256, 1024
    q, s, z = _extreme_qsz(N, K, seed=9, G=1 if gs == 0 else K // gs)
    pl = quant.pack_quantized(q, s, z, 4, gs, DEV)
    G = s.shape[1]
    w = ((q.reshape(N, G, -1).float() - z.reshape(N, G, 1).float()) * s.reshape(N, G, 1).float()).reshape(N, K).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(T)
    x = torch.randn(T, K, generator=g, device=DEV).half()
    out = _nan16(T, N)
    ops.gemv(pl, T, xin=x, out=out, epilogue=ops.B200_EPI_F16)
    torch.cuda.synchronize()
    ref = F.linear(x.float(), w)
    tol = 3.0 * float(ref.abs().max()) * 2 ** -11 + 1e-6  # test_kernels_gpu._tol
    assert torch.isfinite(out).all()
    assert (out.float() - ref).abs().max() <= tol, (out.float() - ref).abs().max()


# ---------------------------------------------------------------------------------------- elementwise kernels ---------
def _neighbour16(a, d):
    """fp16 one ulp from a: d = +1 away from zero, -1 toward zero."""
    b = a.view(torch.int16).int()
    sgn, mag = b & 0x8000, (b & 0x7FFF) + d
    mag = mag.clamp(0, 0x7BFF)
    return torch.where(sgn != 0, mag - 0x8000, mag).to(torch.int16).view(torch.float16)


@pytest.mark.timeout(180)
@pytest.mark.parametrize("D", [512, 4096, 5120, 8192])
@pytest.mark.parametrize("T", [1, 33, 256])
def test_prefill_rmsnorm_matches_reference_rounding(D, T):
    """h = resid (+ delta); x = fp16(h * rsqrt(mean(h^2) + eps)) * gamma (components.py:41-53).  Row 0 has |h| near 6e4,
    row 1 is all zero (only eps keeps rstd finite), row 2 is near-constant."""
    eps = 1e-5
    g = torch.Generator(device=DEV).manual_seed(D + T)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)  # noqa: E731
    gamma = (1 + 0.3 * rn(D)).half()
    one_ulp = total = 0
    for with_delta in (False, True):
        for with_hout in (False, True):
            resid, delta = (2 * rn(T, D)).half(), (2 * rn(T, D)).half() if with_delta else None
            sign = torch.sign(rn(D)).half()
            if with_delta:
                resid[0] = sign * (30000 + 1000 * rn(D).abs().clamp_max(2)).half()
                delta[0] = sign * (25000 + 1000 * rn(D).abs().clamp_max(2)).half()
            else:
                resid[0] = sign * (58000 + 2000 * rn(D).abs().clamp_max(3)).half()
            if T > 1:
                resid[1] = 0
                if with_delta:
                    delta[1] = 0
            if T > 2:
                resid[2] = (3.0 + 1e-3 * rn(D)).half()
            h_out = _nan16(T, D) if with_hout else None
            x = _nan16(T, D)
            ops.prefill_rmsnorm(resid, delta, h_out, gamma, eps, x, T, D)
            torch.cuda.synchronize()
            h = resid + delta if with_delta else resid
            if with_hout:
                assert torch.equal(h_out.view(torch.int16), h.view(torch.int16))
            hf = h.float()
            a = (hf * torch.rsqrt(hf.pow(2).mean(-1, keepdim=True) + eps)).half()
            ref = a * gamma
            exact = x.view(torch.int16) == ref.view(torch.int16)
            near = exact.clone()
            for d in (1, -1):  # rsqrt / the sum of squares rounding one fp32 ulp apart moves a by one fp16 ulp
                near |= x.view(torch.int16) == (_neighbour16(a, d) * gamma).view(torch.int16)
            assert torch.isfinite(x).all()
            assert bool(near.all()), (with_delta, with_hout, int((~near).sum()))
            one_ulp += int((~exact).sum())
            total += exact.numel()
    print(f"\n[rmsnorm D={D} T={T}] one ulp off at the rounding point: {one_ulp} of {total} ({one_ulp / total:.2e})")
    assert one_ulp <= 1e-3 * total  # at most 6.7e-5 measured on an H100 80GB HBM3 (700 W limit)


@pytest.mark.timeout(180)
@pytest.mark.parametrize("Hq,Hkv", [(4, 4), (32, 8), (64, 8), (8, 1)])
@pytest.mark.parametrize("nseq", [1, 2])
@pytest.mark.parametrize("start", ["zero", "37", "table_end"])
def test_prefill_rope_kv_matches_unfused_rope(Hq, Hkv, nseq, start):
    """q, k = fp16 of fp32 (x_e c - x_o s, x_e s + x_o c) as separate multiplies (llama.py:59-77), V copied; K / V land at
    (sequence, position) of the cache and nothing else in the cache changes."""
    R = 8192  # rope table rows; the cache is as long, so a prompt can end at the table's last row
    tps = 45
    T = nseq * tps
    p0 = {"zero": 0, "37": 37, "table_end": R - tps}[start]
    nq, nkv = Hq * 128, Hkv * 128
    rope = rope_table(128, R, 10000.0, None).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(Hq * 10 + Hkv + nseq)
    qkv = (4 * torch.randn(T, nq + 2 * nkv, generator=g, device=DEV)).half()
    pos = (p0 + torch.arange(T, device=DEV) % tps).int()
    kc = _nan16(nseq, Hkv, R, 128)
    vt = _nan16(nseq, Hkv, R // 32, 128, 32)
    q_out = _nan16(T, nq)
    ops.prefill_rope_kv(qkv, q_out, kc, vt, rope, pos, T, nq, nkv, tps, R)
    torch.cuda.synchronize()

    def rot(a, H):
        a = a.float().reshape(T, H, 64, 2)
        cs = rope[pos.long()]
        c, s = cs[:, None, :, 0], cs[:, None, :, 1]
        e, o = a[..., 0], a[..., 1]
        return torch.stack([e * c - o * s, e * s + o * c], dim=-1).reshape(T, H, 128).half()

    assert torch.equal(q_out.view(torch.int16), rot(qkv[:, :nq], Hq).reshape(T, nq).view(torch.int16))
    k_exp, v_exp = _nan16(nseq, Hkv, R, 128), _nan16(nseq, Hkv, R, 128)
    b = torch.arange(T, device=DEV) // tps
    k_exp[b, :, pos.long()] = rot(qkv[:, nq:nq + nkv], Hkv)
    v_exp[b, :, pos.long()] = qkv[:, nq + nkv:].reshape(T, Hkv, 128)
    assert torch.equal(kvlayout.k_from_engine(kc).view(torch.int16), k_exp.view(torch.int16))
    assert torch.equal(kvlayout.v_from_engine(vt).view(torch.int16), v_exp.view(torch.int16))


@pytest.mark.timeout(180)
@pytest.mark.parametrize("Fw", [64, 11008, 13824, 28672])
@pytest.mark.parametrize("T", [1, 256])
def test_prefill_silu_mul_matches_torch(Fw, T):
    """act = fp16(silu(a)) * b (llama.py:252-256) on gu with w1 / w3 rows interleaved 8 + 8 (the engine's w13 layout);
    torch's fp16 F.silu on the same GPU rounds at the same points, so the match is bitwise."""
    g = torch.Generator(device=DEV).manual_seed(Fw + T)
    a = (4 * torch.randn(T, Fw, generator=g, device=DEV)).half()
    b = (2 * torch.randn(T, Fw, generator=g, device=DEV)).half()
    special = torch.tensor([0.0, -0.0, -20.0, -100.0, 6e-8, -6e-8, 3e-6, -3e-6, 2.0 ** -14, 11.0, 30000.0, 65504.0,
                            -65504.0, 17.5], device=DEV).half()
    a[:, :special.numel()] = special
    a[:, -special.numel():] = special.flip(0)
    gu = _interleave_w13(a.T, b.T).T.contiguous()
    act = _nan16(T, Fw)
    ops.prefill_silu_mul(gu, act, T, Fw)
    torch.cuda.synchronize()
    ref = F.silu(a) * b
    diff = act.view(torch.int16) != ref.view(torch.int16)
    assert not bool(diff.any()), (int(diff.sum()), a[diff][:4].tolist(), act[diff][:4].tolist(), ref[diff][:4].tolist())


@pytest.mark.timeout(180)
def test_prefill_ops_check_their_tensors():
    """Wrong dtype, device, layout or a short buffer raises ValueError before anything launches."""
    T, N, K, D, Fw, H = 4, 128, 64, 256, 64, 128
    pl, _ = _linear(*_uniform_qsz(N, K, seed=3))
    z = lambda *s, dt=torch.float16: torch.zeros(*s, dtype=dt, device=DEV)  # noqa: E731
    x, out = z(T, K), _nan16(T, N)
    r, gm, xo = z(T, D), z(D), _nan16(T, D)
    qkv, qo, kc, vt = z(T, 3 * H), _nan16(T, H), _nan16(1, 1, 64, 128), _nan16(1, 1, 2, 128, 32)
    rope, pos = rope_table(128, 64, 10000.0, None).to(DEV), z(T, dt=torch.int32)
    gu, act = z(T, 2 * Fw), _nan16(T, Fw)
    gemm = lambda **kw: ops.prefill_gemm_w4(pl, kw.get("x", x), kw.get("out", out), T)  # noqa: E731
    norm = lambda **kw: ops.prefill_rmsnorm(kw.get("r", r), kw.get("d"), kw.get("h"), kw.get("gm", gm), 1e-5,  # noqa: E731
                                            kw.get("xo", xo), T, D)
    rkv = lambda **kw: ops.prefill_rope_kv(kw.get("qkv", qkv), kw.get("qo", qo), kw.get("kc", kc), kw.get("vt", vt),  # noqa: E731
                                           kw.get("rope", rope), kw.get("pos", pos), T, H, H, kw.get("tps", T), 64)
    silu = lambda **kw: ops.prefill_silu_mul(kw.get("gu", gu), kw.get("act", act), T, Fw)  # noqa: E731
    bad = [
        lambda: gemm(x=x.float()), lambda: gemm(x=x.cpu()), lambda: gemm(x=z(K, T).T), lambda: gemm(x=x[:T - 1]),
        lambda: gemm(out=out[:T - 1]), lambda: gemm(out=out.float()), lambda: gemm(x=None),
        lambda: norm(r=r.float()), lambda: norm(r=r[:T - 1]), lambda: norm(d=z(T, D - 2)), lambda: norm(h=z(T, D)[:, ::2]),
        lambda: norm(gm=gm[:D - 2]), lambda: norm(xo=xo[:T - 1]), lambda: norm(xo=None),
        lambda: rkv(qkv=qkv[:, :2 * H]), lambda: rkv(qo=qo.cpu()), lambda: rkv(kc=kc[..., :64]),
        lambda: rkv(vt=vt.float()), lambda: rkv(tps=1), lambda: rkv(rope=rope.half()),
        lambda: rkv(pos=pos.long()), lambda: rkv(pos=pos[:T - 1]),
        lambda: silu(gu=gu[:, :Fw]), lambda: silu(gu=gu.float()), lambda: silu(act=z(Fw, T).T),
    ]
    torch.cuda.synchronize()
    n0 = ops.launch_count
    for i, f in enumerate(bad):
        with pytest.raises(ValueError):
            f()
    torch.cuda.synchronize()
    assert ops.launch_count == n0
    for t in (out, xo, qo, kc, vt, act):  # the outputs still hold their sentinel
        assert bool((t.view(torch.int16) == 0x7E5A).all())
    gemm(), norm(), rkv(), silu()  # and the same calls with good tensors go through
    torch.cuda.synchronize()
    assert ops.launch_count == n0 + 4


# ------------------------------------------------------------------------------------------------- the engine ---------
def _tiny_w4():
    args = dict(cases.TINY_LLAMA, max_seq_len=640)
    sd = weights.llama_state_dict(args, seed=0)
    sd_ref, recs = omniquant.fake_quantize_state_dict(sd, 4, 0)
    return args, sd, sd_ref, recs


def _engine(args, sd, recs, tc):
    eng = DecodeEngine(EngineConfig.from_model_args("llama", args, bits=4, group_size=0), DEV)
    eng.use_prefill_tc = tc
    eng.load_master_state_dict(sd, quant_records=recs)
    assert eng.prefill_tc_supported() == tc
    return eng


@pytest.mark.timeout(300)
@pytest.mark.parametrize("plen", [33, 128, 255, 256, 257, 300, 513])
def test_long_prompt_through_tensor_core_prefill_matches_port(plen):
    args, sd, sd_ref, recs = _tiny_w4()
    ndec = 3
    toks = weights.synthetic_tokens(2, plen + ndec, args["vocab_size"], seed=7)
    ref32 = cases.run_schedule(PortModel("llama", args, sd_ref, dtype=torch.float32), toks, plen, ndec).numpy()
    ref16 = cases.run_schedule(PortModel("llama", args, sd_ref, dtype=torch.float16), toks, plen, ndec).numpy()
    floor = np.abs(ref16 - ref32).max()
    got = {}
    for tc in (True, False):
        eng = _engine(args, sd, recs, tc)
        tk = toks.cuda()
        outs = [eng.forward_inference(tk[:, :plen], 0).float().cpu().clone()]
        for j in range(ndec):
            outs.append(eng.forward_inference(tk[:, plen + j:plen + j + 1], plen + j).float().cpu().clone())
        got[tc] = torch.stack(outs).numpy()
        e32, e16 = np.abs(got[tc] - ref32).max(), np.abs(got[tc] - ref16).max()
        print(f"\\n[prefill {plen} tc={tc}] |eng-ref16|={e16:.3e} |eng-ref32|={e32:.3e} floor={floor:.3e}")
        from conftest import record_parity
        record_parity(f"tiny_llama_w4_prefill{plen}_{'wgmma' if tc else 'gemv_chunks'}", e16=e16, e32=e32, floor=floor,
                      strict_pass=bool(e16 <= 1e-3 or e32 <= floor), source="oracle port fp16 / fp32 on the CPU")
        assert np.isfinite(got[tc]).all()
        assert e16 <= 1e-3 or e32 <= 1.5 * floor, (e16, e32, floor)
    assert np.abs(got[True] - got[False]).max() <= 4e-3


def _schedule(model, toks, p0, p1, ndec):
    """A p0-token prompt at position 0, a p1-token prompt continuing at p0, then ndec teacher-forced decode steps (a
    two-segment cases.run_schedule).  -> (fp32 logits [2 + ndec, B, V], [(K, V) canonical [B, Hkv, S, 128] float64 per
    layer] as the prompts left the cache)."""
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


@pytest.mark.timeout(300)
@pytest.mark.parametrize("p0,p1", [(5, 40), (100, 200), (40, 300), (250, 33)])
@pytest.mark.parametrize("tc", [True, False])
def test_continuation_prompt_matches_port(p0, p1, tc):
    """A second prompt at start_pos = p0 > 0 (the port's right-aligned causal mask, llama.py:220-224), then decode; the KV
    cache after the prompts matches the port's by the fp16-vs-fp32 floor rule, layer 0 (embed -> rmsnorm -> GEMM -> RoPE)
    to about one fp16 ulp where the wgmma GEMM wrote it, and positions >= p0 + p1 are untouched.  The GEMV-chunk path
    once read stale K / V here: with programmatic dependent launch, attention waited for the QKV kernel only before the
    tile holding pos[tok], though a chunk crossing a 32-row tile also appends to the tile before it."""
    args, sd, sd_ref, recs = _tiny_w4()
    ndec, L = 3, args["n_layers"]
    toks = weights.synthetic_tokens(2, p0 + p1 + ndec, args["vocab_size"], seed=11)
    ref32 = _schedule(PortModel("llama", args, sd_ref, dtype=torch.float32), toks, p0, p1, ndec)
    ref16 = _schedule(PortModel("llama", args, sd_ref, dtype=torch.float16), toks, p0, p1, ndec)
    got = _schedule(_engine(args, sd, recs, tc), toks.cuda(), p0, p1, ndec)
    e32, e16 = np.abs(got[0] - ref32[0]).max(), np.abs(got[0] - ref16[0]).max()
    floor = np.abs(ref16[0] - ref32[0]).max()
    print(f"\n[continuation {p0}+{p1} tc={tc}] |eng-ref16|={e16:.3e} |eng-ref32|={e32:.3e} floor={floor:.3e}")
    from conftest import record_parity
    record_parity(f"tiny_llama_w4_continue{p0}+{p1}_{'wgmma' if tc else 'gemv_chunks'}", e16=e16, e32=e32, floor=floor,
                  strict_pass=bool(e16 <= 1e-3 or e32 <= floor), source="oracle port fp16 / fp32 on the CPU")
    assert np.isfinite(got[0]).all()
    assert e16 <= 1e-3 or e32 <= 1.5 * floor, (e16, e32, floor)

    P = p0 + p1
    # positions whose layer-0 K / V came from the wgmma GEMM (prompts longer than one 32-token chunk), which rebuilds
    # w_hat bit for bit; the decode GEMV applies (q - z) * s unrounded, so its rows get the floor rule only
    wg = torch.zeros(P, dtype=torch.bool)
    if tc:
        wg[:p0] = p0 > 32
        wg[p0:] = p1 > 32
    for i in range(L):
        for j, name in enumerate("KV"):
            e = got[1][i][j][:, :, :P]
            r16, r32 = ref16[1][i][j][:, :, :P], ref32[1][i][j][:, :, :P]
            assert bool((got[1][i][j][:, :, P:] == 0).all()), (i, name)  # nothing written past the prompts
            k16, k32, kf = float((e - r16).abs().max()), float((e - r32).abs().max()), float((r16 - r32).abs().max())
            print(f"  layer {i} {name}: |eng-ref16|={k16:.3e} |eng-ref32|={k32:.3e} floor={kf:.3e}")
            assert k16 <= 1e-3 or k32 <= 1.5 * kf, (i, name, k16, k32, kf)
            if i == 0 and bool(wg.any()):
                # one ulp of the value; K is rotated from two GEMM outputs, so one ulp of the pair's norm each; plus 1/8
                # ulp of the head's largest value for fp32 accumulation order where the GEMM output cancels
                ref_scale = r16 if name == "V" else r16.reshape(*r16.shape[:-1], 64, 2).norm(dim=-1).repeat_interleave(2, -1)
                tol = (1 if name == "V" else 2) * _ulp16(ref_scale) + _ulp16(r16.abs().amax(-1, keepdim=True)) / 8
                worst = float(((e - r16).abs() / tol)[:, :, wg].max())
                print(f"  layer 0 {name} (wgmma rows): max |eng - ref16| / tol = {worst:.3f}")
                assert worst <= 1.0, (name, worst)
