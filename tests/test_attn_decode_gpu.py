"""GPU: decode attention (attn_decode_kernel, csrc/attn.cu) against float64 at real widths, exact probes, both split
schedules, and the multi-token launch shapes that forward_inference makes.

References run in float64 on the device, from the fp16 q, K and V the kernel reads.  All inputs are built in canonical
[B, Hkv, S, 128] form and converted with kvlayout.  Notation: t_i = (q . k_i) log2(e) / sqrt(128) is key i's score in
log2 units, w_i = 2^(t_i - max t) its weight (the largest is 1), out = sum w V / sum w, u = 2^-24.

  A. The float64 bound.  The kernel's output is a convex combination of V rows: P is rounded to fp16 BEFORE it enters both
     the row sum l and the PV MMA, and every later factor (corr, the in-CTA and cross-split 2^(m - M)) multiplies l and O
     alike.  So each key carries one effective weight  w^_i = lambda w_i (1 + e_i), lambda common to all keys, and
       |out^ - out| = |sum (w^_i - w_i)(V_i - out)| / sum w^  <=  2 sum w_i e_i |V_i - out| / (sum w - sum w_i e_i).
     e_i is a sum of first-order terms; the factor 2 covers the products of the (1 + e) factors they come from.
       * score: the fp32 HMMA accumulation of q . k_i is within C_ACC sum_d |q_d k_id| (C_ACC = 2^-18: the accumulation
         constant of the project's fp16 HMMA kernels, measured at most 2^-20.7 on an H100 over K up to 28672 in
         test_prefill_gpu.py; a score sums 128 products).  scale_log2 = fp32(fp32(1/sqrt 128) * fp32(log2 e)) is within 3u
         of log2(e)/sqrt(128) and the product s * scale_log2 rounds once (4u |t_i| in all).  The exponent differences
         t_i - m and the chain m -> m' -> M of corr / merge factors round once per step; the steps telescope, so together
         they are within 2u (|t_i| + |M|).  With margin: 16u max(|t_i|, |max t|) in log2 units on top of the HMMA term,
         2^(that) - 1 relative.
       * exp2f: 2 ulp = 2^-22 relative (CUDA C Programming Guide, single-precision functions), once for p and once per
         factor on key i's way to the output: at most tiles-per-warp corrections, the in-CTA and the cross-split factor.
       * fp16 rounding of P: 2^-11 relative, or 2^-25 absolute where p is below the fp16 normal range.  p is taken
         against a running maximum <= the final one, so only keys with w_i < 2^-13 can be subnormal; each adds 2^-25
         |V_i - out| to the numerator and 2^-25 to what the denominator may lose.
     Then the fp32 sums that are not weights:
       * O: the PV HMMA chain of a warp (C_ACC again, relative to sum w |V|), one rounding per corr rescale (tiles per warp),
         the in-CTA merge (4) and the cross-split fmaf chain (n_split), the division: (C_ACC + (tpw + n_split + 8) u)
         sum w |V| / sum w.
       * l: a sequential fp32 sum of positive terms (4 adds and 1 pair add per tile, one rescale per tile), 2 shuffles, the
         in-CTA merge, the cross-split sum (a 5-level tree of per-lane sums of n_split / 32 terms): depth <= 5 tpw + n_split
         / 32 + 20, each rounding at most u of L, so (5 tpw + n_split / 32 + 20) u |out|.
       * the output rounds to fp16: half an ulp of the fp32 value, <= 2^-11 (|out| + its error) + 2^-25.
     V = 1 + 0.5 randn, so outputs are O(1) and the bound is relative in effect.  Regimes: natural (q, k ~ N(0, 1)),
     peaked (q x 6), flat (q = 0), the maximum in the last split (a key ramp of +0.032 per position), the maximum in the
     first split with a decay of 2 log2 per position (later splits' 2^(m - M) underflows to 0), large (q, k x 40: |t| in
     the thousands; the output must stay finite).
  B. Exact probes (bit for bit).
       * Selection: query head h is q = 16 e_d, and in column d of its kv head only key j holds a non-zero (32).  Every other
         key scores exactly 0, key j scores G = 16 * 32 log2(e) / sqrt(128) = 65.3 log2 units.  In j's tile the other P are
         fp16(2^-65.3) = 0; every other tile, warp and split contributes its O and l times 2^-65.3 (or 0), at most
         2^-65.3 * 32768 * 2 < 2^-49 against V_j >= 1, far below half an fp32 ulp; so out[h] = V_j exactly.  64 of the 128
         dims are probed per (sequence, kv head): 4 in each 16-byte chunk, at offsets the chunk c ^ 4 (the K swizzle's other
         row parity) does not probe, whose columns hold N(0, 1) noise.  A swizzle or V-transpose slip reads noise or moves
         V_j's columns.  Every head of a group probes its own (j, d), pinning the head-to-MMA-row map (rows g, g + 8).
         Targets: rows 0, 1, 31, 32, 33, pos, and the first two and last two keys of every split of the schedule launched.
       * Mean: q = 0 and V holds integers in [-64, 64]: every score is 0, every p is 1, every sum is an integer below 2^24,
         so out = fp16(fp32(sum V[0 .. pos]) / fp32(pos + 1)) exactly (no fast-math: the division is correctly rounded).
       * Mask and causality: the rows after a token's position up to the end of its last tile hold decoys (k = 8, the top
         score by far; V = +-65504), every later tile and every cache row outside the launch's sequences the NaN sentinel.
         In a multi-token launch the decoys are the later tokens' own rows.  Each token's output must equal, bit for bit,
         the T = 1 launch (same n_split, max_kv_len) on a cache whose rows past its position are zero.
       Contract: V rows past pos inside the last tile read must be FINITE.  Their p is 0, but 0 x NaN in the PV MMA is NaN
       (a K row there may hold anything: its score is replaced by -inf before use).  The reference's masked SDPA has the
       same property inside a chunk; the engine's caches are zero-filled and only ever hold finite rows.
  C. Schedules: B200_ATTN_EVEN 0 and 1, n_split 1, 2, 16, 17, the host's choice, one split per tile, more splits than the
     context has tiles (a grid sized for max_kv_len = cache_seq with a short pos, as a captured graph is), and a raised
     B200_ATTN_MAX_SPLIT that makes the host choose the staged merge of more than 16 splits.  B200_KV_EF (an L2 hint) must
     not change a bit.
  D. The engine's launch shapes (forward_inference): decode batches, tensor-core prompt sub-chunks of 32 with a short last
     one, GEMV chunks nb x ci for LLaMA (t_max 32) and Mixtral (t_max 16), and every launch of the tiny-Mixtral (40, 300)
     continuation of test_prefill_moe_gpu.py.
  E. Bit identities: batch invariance, repeats, a side stream, one workspace and counter buffer shared by launches of
     different T, no write outside out[:T, :Hq * 128], and K / V caches byte-unchanged.
  The kernel is also compared with oracle.numerics.attn_kernel_model on a few cases.  The model sums in another order and
  torch's exp2 is not exp2f, so no sharp bound between the two follows from the above: the difference is reported in fp16
  ulps, not asserted.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import _cabi, kvlayout, ops  # noqa: E402
from oracle.numerics import SENT, attn_choose_split, attn_host_split, attn_kernel_model, attn_split_ranges  # noqa: E402
from oracle.numerics import nan16, tuned  # noqa: E402
# the float64 reference and bound of section A live in oracle/numerics.py, shared with test_engine_launch_audit_gpu.py
from oracle.numerics import AttnRef as _Ref  # noqa: E402

DEV = "cuda"
PROBE_Q, PROBE_K = 16.0, 32.0   # selection probe: gap 65.3 log2 units
PAD = 512                       # NaN margin on each side of the output
S4K = 4096
POSS = [0, 1, 31, 32, 33, 127, 128, 2047, 4095]
SHAPES = [("7B", 32, 32), ("13B", 40, 40), ("70B_tp1", 64, 8), ("70B_tp2", 32, 4), ("70B_tp4", 16, 2),
          ("70B_tp8", 8, 1), ("mixtral", 32, 8), ("group16", 16, 1)]
REGIMES = ["natural", "peaked", "flat", "last_split", "first_split", "large"]


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _engine(k, v):
    return kvlayout.k_to_engine(k.half()).contiguous(), kvlayout.v_to_engine(v.half()).contiguous()


def _pos(p):
    return torch.tensor(p, dtype=torch.int32, device=DEV)


def _grid(T, Hkv, mkv, ns):
    """(n_split launched, chunk) for a request of ns splits (0: the host's choice)."""
    return attn_host_split(mkv, ns if ns > 0 else ops.attn_split(T, Hkv, mkv))


def _attn(q, kc, vt, pos, *, Hkv, tps, mkv, ns=0, ws=None, cnt=None):
    """One launch into a NaN-sentinel output framed by a NaN margin -> (out [T, Hq, 128], n_split, chunk).  The margin
    must survive and the counters must be back at zero."""
    T, Hq = q.shape[0], q.shape[1]
    n_split, chunk = _grid(T, Hkv, mkv, ns)
    if ws is None:
        ws = torch.zeros(ops.attn_workspace_bytes(T, Hq, n_split), dtype=torch.uint8, device=DEV)
    if cnt is None:
        cnt = torch.zeros(T * Hkv, dtype=torch.int32, device=DEV)
    n = T * Hq * 128
    buf = nan16(n + 2 * PAD, device=DEV)
    out = buf[PAD:PAD + n].view(T, Hq * 128)
    ops.attn_decode(q.contiguous(), kc, vt, pos, out, T=T, Hq=Hq, Hkv=Hkv, cache_seq=kc.shape[2], tokens_per_seq=tps,
                    max_kv_len=mkv, ws=ws, counters=cnt, n_split=ns)
    torch.cuda.synchronize()
    m = buf.view(torch.int16)
    assert bool((m[:PAD] == SENT).all()) and bool((m[PAD + n:] == SENT).all()), "write outside out[:T, :Hq * 128]"
    assert int(cnt.abs().sum()) == 0, "counters not reset"
    return out.view(T, Hq, 128), n_split, chunk


def _cdiv(a, b):
    return -(-a // b)


def _bits(x):
    return x.contiguous().view(torch.int16)


def _regime(name, q0, k0):
    """Score regimes (module docstring, A) from N(0, 1) q0 [T, Hq, 128] and k0 [B, Hkv, S, 128] (fp32)."""
    if name == "natural":
        return q0, k0
    if name == "peaked":
        return 6 * q0, k0
    if name == "flat":
        return 0 * q0, k0
    if name == "large":
        return 40 * q0, 40 * k0
    ramp = torch.arange(k0.shape[2], device=DEV, dtype=torch.float32)
    q, k = q0.clone(), k0.clone()
    q[..., 0] = 16.0
    k[..., 0] = ramp / 64 if name == "last_split" else -ramp
    return q, k


def _schedules(T, Hkv, S, p):
    """(even, n_split request, max_kv_len) for a context ending at p: eager and graph-sized grids, host's choice, 1, 2, 16,
    17 and one split per tile; one entry per distinct grid."""
    seen, out = set(), []
    for mkv in (min(S, (p + 128) // 128 * 128), S):
        for ns in (0, 1, 2, 16, 17, mkv // 32):
            for even in (0, 1):
                key = (even,) + _grid(T, Hkv, mkv, ns)
                if key not in seen:
                    seen.add(key)
                    out.append((even, ns, mkv))
    return out


def _bound_case(q, k, v, kc, vt, pos, tps, scheds, Hkv):
    """Every schedule of scheds against one reference -> worst err / tol."""
    ref = _Ref(q, k, v, pos, tps)
    worst = 0.0
    for even, ns, mkv in scheds:
        with tuned("B200_ATTN_EVEN", even):
            out, n_split, chunk = _attn(q, kc, vt, _pos(pos), Hkv=Hkv, tps=tps, mkv=mkv, ns=ns)
        r = ref.ratio(out, n_split, chunk, even)
        assert r <= 1.0, (even, ns, mkv, n_split, r)
        worst = max(worst, r)
    return worst


# ------------------------------------------------------------------------------------------- exact probes --------
def _probe_dims(b, g):
    """64 probed dims of (sequence b, kv head g): 4 per 16-byte chunk c, at offsets that chunk c ^ 4 does not probe."""
    return [8 * c + (c + j + b + g) % 8 for c in range(16) for j in range(4)]


def _targets(p, n_split, chunk, even):
    """rows a selection probe aims at for a token at position p."""
    t = {0, 1, 31, 32, 33, p}
    for b, e in attn_split_ranges(p + 1, n_split, chunk, even):
        if e > b:
            t |= {b, b + 1, e - 1, e - 2}
    return sorted(x for x in t if 0 <= x <= p)


def _selection(Hq, Hkv, S, B, pos, tps, targets, seed, rot):
    """-> (q [T, Hq, 128], k, v canonical fp16, expected fp16 [T, Hq, 128], probed rows).  Tokens are served in position
    order, so every hot key already placed lies at or before the current token's position (tokens of one sequence)."""
    T, r = len(pos), Hq // Hkv
    g = _gen(seed)
    k = torch.randn(B, Hkv, S, 128, generator=g, device=DEV)
    v = (1 + 0.5 * torch.rand(B, Hkv, S, 128, generator=g, device=DEV)).half()
    q = torch.zeros(T, Hq, 128, device=DEV)
    hot, sel = {}, [[0] * Hq for _ in range(T)]
    for t in sorted(range(T), key=lambda t: pos[t]):
        b = t // tps
        for gg in range(Hkv):
            dims, H, used = _probe_dims(b, gg), hot.setdefault((b, gg), {}), set()
            for h in range(r):
                tg = targets[t]
                want = tg[(gg * r + h + rot) % len(tg)]
                same = [d for d in H if H[d] == want and d not in used]
                free = [d for d in dims if d not in H]
                if same:
                    d = same[0]
                elif free:
                    d = free[(5 * gg + 3 * h + 7 * rot) % len(free)]
                    H[d] = want
                else:
                    old = [d for d in H if d not in used and H[d] <= pos[t]]
                    d = old[(h + rot) % len(old)]
                used.add(d)
                q[t, gg * r + h, d] = PROBE_Q
                sel[t][gg * r + h] = H[d]
    bi, gi, di, ji = [], [], [], []
    for (b, gg), H in hot.items():
        for d, j in H.items():
            bi.append(b), gi.append(gg), di.append(d), ji.append(j)
    bi, gi, di, ji = (torch.tensor(x, device=DEV) for x in (bi, gi, di, ji))
    k[bi, gi, :, di] = 0.0
    k[bi, gi, ji, di] = PROBE_K
    exp = torch.stack([torch.stack([v[t // tps, h // r, sel[t][h]] for h in range(Hq)]) for t in range(T)])
    return q.half(), k.half(), v, exp, {j for row in sel for j in row}


def _mean(Hq, Hkv, S, B, pos, tps, seed):
    T, r = len(pos), Hq // Hkv
    g = _gen(seed)
    k = torch.randn(B, Hkv, S, 128, generator=g, device=DEV).half()
    v = torch.randint(-64, 65, (B, Hkv, S, 128), generator=g, device=DEV).half()
    q = torch.zeros(T, Hq, 128, dtype=torch.float16, device=DEV)
    exp = []
    for t in range(T):
        n = pos[t] + 1
        s = v[t // tps, :, :n].double().sum(1).float().cpu()                     # exact integers
        exp.append((s / torch.tensor(float(n), dtype=torch.float32)).half().repeat_interleave(r, 0))
    return q, k, v, torch.stack(exp).to(DEV)


def _exact_probes(Hq, Hkv, S, B, pos, tps, scheds, seed):
    """Selection and mean probes under every schedule -> (probes checked, distinct rows hit)."""
    n_probe, rows = 0, set()
    for even, ns, mkv in scheds:
        with tuned("B200_ATTN_EVEN", even):
            n_split, chunk = _grid(len(pos), Hkv, mkv, ns)
            targets = [_targets(p, n_split, chunk, even) for p in pos]
            need = max(_cdiv(len(tg), Hq) for tg in targets)
            for rot in range(0, need * Hq, Hq):
                q, k, v, exp, hit = _selection(Hq, Hkv, S, B, pos, tps, targets, seed + rot, rot)
                kc, vt = _engine(k, v)
                out, _, _ = _attn(q, kc, vt, _pos(pos), Hkv=Hkv, tps=tps, mkv=mkv, ns=ns)
                bad = (_bits(out) != _bits(exp)).any(-1)
                assert not bool(bad.any()), ("selection", even, ns, mkv, rot, bad.nonzero()[:4].tolist())
                n_probe, rows = n_probe + out.shape[0] * Hq, rows | hit
            q, k, v, exp = _mean(Hq, Hkv, S, B, pos, tps, seed + 1)
            kc, vt = _engine(k, v)
            out, _, _ = _attn(q, kc, vt, _pos(pos), Hkv=Hkv, tps=tps, mkv=mkv, ns=ns)
            assert torch.equal(_bits(out), _bits(exp)), ("mean", even, ns, mkv)
            n_probe += out.shape[0] * Hq
    return n_probe, rows


def _mask_probe(Hq, Hkv, S, B, pos, tps, mkv, ns, seed):
    """Decoys after each token's position, NaN beyond the last tile and in the row outside the launch (row offset 1):
    every token's output equals its T = 1 launch on a cache zeroed past its position.  -> tokens checked."""
    T = len(pos)
    g = _gen(seed)
    q = (0.5 + 0.5 * torch.randn(T, Hq, 128, generator=g, device=DEV).abs()).half()
    k = torch.randn(B + 1, Hkv, S, 128, generator=g, device=DEV)
    v = 1 + 0.5 * torch.randn(B + 1, Hkv, S, 128, generator=g, device=DEV)
    nan = float("nan")
    sign = torch.where(torch.arange(128, device=DEV) % 2 == 0, 65504.0, -65504.0)
    k[0], v[0] = nan, nan
    for b in range(B):
        ps = [pos[t] for t in range(T) if t // tps == b]
        end = (max(ps) // 32 + 1) * 32
        k[b + 1, :, min(ps) + 1:end], v[b + 1, :, min(ps) + 1:end] = 8.0, sign
        k[b + 1, :, end:], v[b + 1, :, end:] = nan, nan
    kc, vt = _engine(k, v)
    out, n_split, _ = _attn(q, kc[1:], vt[1:], _pos(pos), Hkv=Hkv, tps=tps, mkv=mkv, ns=ns)
    assert bool(torch.isfinite(out).all())
    for t in range(T):
        b, p = t // tps, pos[t]
        end = (p // 32 + 1) * 32
        kk, vv = k[b + 1:b + 2].clone(), v[b + 1:b + 2].clone()
        kk[:, :, p + 1:end], vv[:, :, p + 1:end] = 0.0, 0.0
        kk[:, :, end:], vv[:, :, end:] = nan, nan
        kc1, vt1 = _engine(kk, vv)
        one, _, _ = _attn(q[t:t + 1], kc1, vt1, _pos([p]), Hkv=Hkv, tps=1, mkv=mkv, ns=n_split)
        assert torch.equal(_bits(one[0]), _bits(out[t])), ("mask", t, p, mkv, n_split)
    return T


# ------------------------------------------------------------------------------------------------ C. host --------
def test_host_split_choice_matches_the_restatement():
    """b200_attn_choose_split against attn_choose_split over token counts, kv heads, contexts and two caps."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 0
    for cap in (16, 64):
        with tuned("B200_ATTN_MAX_SPLIT", cap):
            for T in (1, 2, 3, 4, 7, 8, 16, 32):
                for Hkv in (1, 2, 4, 8, 32, 40):
                    for mkv in (1, 31, 32, 33, 128, 640, 2400, 4096, 32768):
                        assert ops.attn_split(T, Hkv, mkv) == attn_choose_split(T, Hkv, mkv, sms, cap), (cap, T, Hkv, mkv)
                        n += 1
    print(f"\n[host split] {n} (T, Hkv, max_kv_len, cap) cases agree ({sms} SMs)")


def test_host_refuses_a_merge_too_large_for_shared_memory():
    """16 heads per group and 512 splits: 16 (512 * 12 + 4) bytes of staged (m, l, f, L) exceed the 96 KB ring."""
    Hq, Hkv, S = 16, 1, 16384
    q = torch.zeros(1, Hq, 128, dtype=torch.float16, device=DEV)
    kc = torch.zeros(1, Hkv, S, 128, dtype=torch.float16, device=DEV)
    vt = torch.zeros(1, Hkv, S // 32, 128, 32, dtype=torch.float16, device=DEV)
    assert attn_host_split(S, 512) == (512, 32)
    ws = torch.zeros(ops.attn_workspace_bytes(1, Hq, 512), dtype=torch.uint8, device=DEV)
    cnt = torch.zeros(Hkv, dtype=torch.int32, device=DEV)
    out = nan16(1, Hq * 128, device=DEV)
    with pytest.raises(_cabi.B200Error) as e:
        ops.attn_decode(q, kc, vt, _pos([S - 1]), out, T=1, Hq=Hq, Hkv=Hkv, cache_seq=S, tokens_per_seq=1, max_kv_len=S,
                        ws=ws, counters=cnt, n_split=512)
    assert "rc=-1" in str(e.value) and "attn: too many splits" in str(e.value), str(e.value)
    torch.cuda.synchronize()
    assert bool((_bits(out) == SENT).all())


# --------------------------------------------------------------------------- A, B at the real head layouts --------
def _shape_inputs(Hq, Hkv, S, T, seed):
    g = _gen(seed)
    q0 = torch.randn(T, Hq, 128, generator=g, device=DEV)
    k0 = torch.randn(1, Hkv, S, 128, generator=g, device=DEV)
    v = (1 + 0.5 * torch.randn(1, Hkv, S, 128, generator=g, device=DEV)).half()
    return q0, k0, v


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name,Hq,Hkv", SHAPES, ids=[s[0] for s in SHAPES])
def test_float64_bound_at_real_widths(name, Hq, Hkv):
    """T = 1 at cache_seq 4096, every position of POSS, every regime, every schedule of _schedules."""
    q0, k0, v = _shape_inputs(Hq, Hkv, S4K, len(POSS), seed=Hq * 100 + Hkv)
    rep, n_launch = [], 0
    for reg in REGIMES:
        q, k = _regime(reg, q0, k0)
        q, k = q.half(), k.half()
        kc, vt = _engine(k, v)
        worst = 0.0
        for i, p in enumerate(POSS):
            sc = _schedules(1, Hkv, S4K, p)
            worst = max(worst, _bound_case(q[i:i + 1], k, v, kc, vt, [p], 1, sc, Hkv))
            n_launch += len(sc)
        rep.append(f"{reg} {worst:.3f}")
    print(f"\n[bound {name} {Hq}/{Hkv}] {n_launch} launches, worst err/tol: " + ", ".join(rep))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name,Hq,Hkv", SHAPES, ids=[s[0] for s in SHAPES])
def test_exact_probes_at_real_widths(name, Hq, Hkv):
    """Selection and mean probes at every position and schedule; the mask probe with the host's grid, one split, and one
    split per tile of a graph-sized grid, under both schedules."""
    n_probe, rows, n_mask = 0, set(), 0
    for i, p in enumerate(POSS):
        sc = _schedules(1, Hkv, S4K, p)
        c, hit = _exact_probes(Hq, Hkv, S4K, 1, [p], 1, sc, seed=Hq + 7 * i)
        n_probe, rows = n_probe + c, rows | hit
        for even in (0, 1):
            with tuned("B200_ATTN_EVEN", even):
                for ns in (0, 1, S4K // 32):
                    n_mask += _mask_probe(Hq, Hkv, S4K, 1, [p], 1, S4K, ns, seed=p + ns)
    print(f"\n[probes {name} {Hq}/{Hkv}] {n_probe} bit-exact (token, head) probes over {len(rows)} distinct rows; "
          f"{n_mask} mask probes")


@pytest.mark.timeout(300)
def test_mixtral_32k_context():
    """Mixtral 8x7B (32 / 8) at cache_seq 32768, pos 32767: every regime under the host's grid, 16, 17 and one split per
    tile (1024: the staged merge) for both schedules; selection and mean probes under the host's grid."""
    Hq, Hkv, S, p = 32, 8, 32768, 32767
    q0, k0, v = _shape_inputs(Hq, Hkv, S, 1, seed=32768)
    sc = [(e, ns, S) for e in (0, 1) for ns in (0, 16, 17, S // 32)]
    rep = []
    for reg in REGIMES:
        q, k = _regime(reg, q0, k0)
        q, k = q.half(), k.half()
        kc, vt = _engine(k, v)
        rep.append(f"{reg} {_bound_case(q, k, v, kc, vt, [p], 1, sc, Hkv):.3f}")
        del kc, vt
    n_probe, rows = _exact_probes(Hq, Hkv, S, 1, [p], 1, [(0, 0, S), (1, 0, S)], seed=5)
    print(f"\n[mixtral 32k] worst err/tol: " + ", ".join(rep) + f"; {n_probe} bit-exact probes over {len(rows)} rows")


@pytest.mark.timeout(300)
def test_host_chosen_staged_merge_at_a_real_head_count():
    """B200_ATTN_MAX_SPLIT = 64: a 3-token decode batch of 70B's TP = 2 rank (32 / 4) gets more than 16 splits from the
    host itself (capped at 16 by default), and meets the bound and the probes with them."""
    Hq, Hkv, T = 32, 4, 3
    pos = [4095, 2100, 777]
    with tuned("B200_ATTN_MAX_SPLIT", 64):
        ns = ops.attn_split(T, Hkv, S4K)
        assert ns > 16, ns
        g = _gen(3)
        q = torch.randn(T, Hq, 128, generator=g, device=DEV).half()
        k = torch.randn(T, Hkv, S4K, 128, generator=g, device=DEV).half()
        v = (1 + 0.5 * torch.randn(T, Hkv, S4K, 128, generator=g, device=DEV)).half()
        kc, vt = _engine(k, v)
        sc = [(0, 0, S4K), (1, 0, S4K)]
        worst = _bound_case(q, k, v, kc, vt, pos, 1, sc, Hkv)
        n_probe, rows = _exact_probes(Hq, Hkv, S4K, T, pos, 1, sc, seed=9)
        n_mask = _mask_probe(Hq, Hkv, S4K, T, pos, 1, S4K, 0, seed=4)
    assert ops.attn_split(T, Hkv, S4K) == 16
    print(f"\n[staged merge by the host] {ns} splits: worst err/tol {worst:.3f}; {n_probe} bit-exact probes over "
          f"{len(rows)} rows; {n_mask} mask probes")


# ---------------------------------------------------------------------------- D. the engine's launch shapes --------
def _kv(p_end):
    """max_kv_len forward_inference passes for a chunk ending before position p_end."""
    return (p_end + 127) // 128 * 128


def _gemv_chunk(nb, p0, ci):
    return [p0 + j for _ in range(nb) for j in range(ci)]


def _tiny_mixtral_launches():
    """Every attention launch of the (40, 300) continuation at batch 2 with t_max 16: prompt 40 from 0, then 300 from 40."""
    out = []
    for start, plen in ((0, 40), (40, 300)):
        off = 0
        while off < plen:
            ci = min(8, plen - off)
            out.append((_gemv_chunk(2, start + off, ci), ci, min(640, _kv(start + off + ci))))
            off += ci
    return out


#            name               Hq  Hkv   S     [(positions, tokens_per_seq, max_kv_len)]
ENGINE = [
    ("decode_bs2",              32, 32, 4096, [([100, 4000], 1, 4096)]),
    ("decode_bs7",              64, 8,  4096, [([0, 31, 32, 33, 1000, 2047, 4095], 1, 4096)]),
    ("decode_bs32",             40, 40, 4096, [([127 * i + 5 for i in range(32)], 1, 4096)]),
    ("tc_subchunks",            32, 32, 4096, [(list(range(0, 32)), 32, 256), (list(range(224, 256)), 32, 256),
                                               (list(range(4064, 4096)), 32, 4096)]),
    ("tc_short_last",           8,  1,  4096, [(list(range(288, 300)), 12, 384), (list(range(0, 20)), 20, 128)]),
    ("gemv_llama",              16, 2,  4096, [(_gemv_chunk(1, 16, 32), 32, 128), (_gemv_chunk(2, 120, 16), 16, 256),
                                               (_gemv_chunk(4, 60, 8), 8, 128), (_gemv_chunk(32, 33, 1), 1, 128)]),
    ("gemv_llama_tp2",          32, 4,  4096, [(_gemv_chunk(2, 2040, 16), 16, 2176), (_gemv_chunk(4, 4088, 8), 8, 4096)]),
    ("gemv_mixtral",            32, 8,  4096, [(_gemv_chunk(1, 1000, 16), 16, 1024), (_gemv_chunk(2, 250, 8), 8, 384),
                                               (_gemv_chunk(2, 300, 4), 4, 384)]),
    ("tiny_mixtral_40_300",     4,  2,  640,  _tiny_mixtral_launches()),
]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name,Hq,Hkv,S,launches", ENGINE, ids=[e[0] for e in ENGINE])
def test_engine_launch_shapes(name, Hq, Hkv, S, launches):
    """Each launch with the host's grid under both schedules: the float64 bound; batch invariance (every token equals its
    T = 1 launch at the same n_split and max_kv_len); selection, mean and mask probes; repeats and a side stream
    identical; K / V caches byte-unchanged."""
    worst, n_probe, rows, n_mask, n_inv = 0.0, 0, set(), 0, 0
    for li, (pos, tps, mkv) in enumerate(launches):
        T, B = len(pos), len(pos) // tps
        assert T == B * tps and mkv >= max(pos) + 1
        g = _gen(li + Hq)
        q = torch.randn(T, Hq, 128, generator=g, device=DEV).half()
        k = torch.randn(B, Hkv, S, 128, generator=g, device=DEV).half()
        v = (1 + 0.5 * torch.randn(B, Hkv, S, 128, generator=g, device=DEV)).half()
        kc, vt = _engine(k, v)
        kc0, vt0 = kc.clone(), vt.clone()
        sc = [(0, 0, mkv), (1, 0, mkv)]
        worst = max(worst, _bound_case(q, k, v, kc, vt, pos, tps, sc, Hkv))
        for even in (0, 1):
            with tuned("B200_ATTN_EVEN", even):
                out, n_split, _ = _attn(q, kc, vt, _pos(pos), Hkv=Hkv, tps=tps, mkv=mkv)
                again, _, _ = _attn(q, kc, vt, _pos(pos), Hkv=Hkv, tps=tps, mkv=mkv)
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    other, _, _ = _attn(q, kc, vt, _pos(pos), Hkv=Hkv, tps=tps, mkv=mkv)
                assert torch.equal(_bits(out), _bits(again)) and torch.equal(_bits(out), _bits(other)), (li, even)
                for t in range(T):
                    b = t // tps
                    one, _, _ = _attn(q[t:t + 1], kc[b:b + 1], vt[b:b + 1], _pos([pos[t]]), Hkv=Hkv, tps=1, mkv=mkv,
                                      ns=n_split)
                    assert torch.equal(_bits(one[0]), _bits(out[t])), ("batch invariance", li, even, t)
                    n_inv += 1
                n_mask += _mask_probe(Hq, Hkv, S, B, pos, tps, mkv, 0, seed=li)
        assert torch.equal(_bits(kc), _bits(kc0)) and torch.equal(_bits(vt), _bits(vt0)), "K / V cache written"
        c, hit = _exact_probes(Hq, Hkv, S, B, pos, tps, sc, seed=li * 3)
        n_probe, rows = n_probe + c, rows | hit
    print(f"\n[engine {name} {Hq}/{Hkv}] {len(launches)} launches: worst err/tol {worst:.3f}; {n_inv} tokens batch-"
          f"invariant; {n_probe} bit-exact probes over {len(rows)} rows; {n_mask} mask probes")


# --------------------------------------------------------------------------------------- E. bit identities --------
@pytest.mark.timeout(180)
def test_kv_evict_first_hint_changes_no_bit():
    Hq, Hkv, T = 32, 8, 4
    pos = [4095, 33, 1500, 2047]
    g = _gen(21)
    q = torch.randn(T, Hq, 128, generator=g, device=DEV).half()
    kc, vt = _engine(torch.randn(T, Hkv, S4K, 128, generator=g, device=DEV),
                     1 + 0.5 * torch.randn(T, Hkv, S4K, 128, generator=g, device=DEV))
    outs = []
    for ef in (1, 0):
        with tuned("B200_KV_EF", ef):
            for ns in (0, 1, 17):
                outs.append(_attn(q, kc, vt, _pos(pos), Hkv=Hkv, tps=1, mkv=S4K, ns=ns)[0])
    for a, b in zip(outs[:3], outs[3:]):
        assert torch.equal(_bits(a), _bits(b))


@pytest.mark.timeout(180)
def test_one_workspace_shared_by_launches_of_different_token_counts():
    """As _prefill_chunk_tc does: sub-chunks of 32, 32 and 7 tokens, then a decode batch, one workspace and counter buffer
    sized for the largest; every launch equals its launch on fresh buffers and leaves the counters at zero."""
    Hq, Hkv, S = 32, 8, 4096
    g = _gen(8)
    k = torch.randn(2, Hkv, S, 128, generator=g, device=DEV)
    v = 1 + 0.5 * torch.randn(2, Hkv, S, 128, generator=g, device=DEV)
    kc, vt = _engine(k, v)
    q = torch.randn(32, Hq, 128, generator=g, device=DEV).half()
    launches = [(list(range(0, 32)), 32, 256), (list(range(32, 64)), 32, 256), (list(range(64, 71)), 7, 256),
                ([70, 3000], 1, S), (list(range(0, 32)), 32, 256)]
    need = max(ops.attn_workspace_bytes(len(p), Hq, _grid(len(p), Hkv, m, 0)[0]) for p, _, m in launches)
    ws = torch.full((need,), 0x7F, dtype=torch.uint8, device=DEV)
    cnt = torch.zeros(32 * Hkv, dtype=torch.int32, device=DEV)
    for pos, tps, mkv in launches:
        T = len(pos)
        shared, _, _ = _attn(q[:T], kc, vt, _pos(pos), Hkv=Hkv, tps=tps, mkv=mkv, ws=ws, cnt=cnt)
        fresh, _, _ = _attn(q[:T], kc, vt, _pos(pos), Hkv=Hkv, tps=tps, mkv=mkv)
        assert torch.equal(_bits(shared), _bits(fresh)), (T, tps)


# ------------------------------------------------------------------------------------------ kernel vs model --------
def _ulps(a, b):
    """fp16 steps between a and b (same-sign order of the bit patterns)."""
    def key(x):
        i = _bits(x).long()
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return int((key(a) - key(b)).abs().max())


@pytest.mark.timeout(180)
def test_kernel_against_the_cpu_arithmetic_model():
    """T = 1 cases against oracle.numerics.attn_kernel_model: the difference in fp16 ulps is reported, not asserted."""
    rep = []
    for Hq, Hkv, p, ns, even in ((32, 32, 2047, 0, 0), (8, 1, 4095, 17, 1), (64, 8, 127, 2, 0), (16, 1, 1000, 1, 0)):
        g = _gen(p + Hq)
        q = torch.randn(1, Hq, 128, generator=g, device=DEV).half()
        k = torch.randn(1, Hkv, S4K, 128, generator=g, device=DEV).half()
        v = (1 + 0.5 * torch.randn(1, Hkv, S4K, 128, generator=g, device=DEV)).half()
        kc, vt = _engine(k, v)
        with tuned("B200_ATTN_EVEN", even):
            out, n_split, _ = _attn(q, kc, vt, _pos([p]), Hkv=Hkv, tps=1, mkv=S4K, ns=ns)
        qc, kcpu, vcpu, r = q.cpu(), k.cpu(), v.cpu(), Hq // Hkv
        model = torch.stack([attn_kernel_model(qc[0, h], kcpu[0, h // r, :p + 1], vcpu[0, h // r, :p + 1], n_split,
                                               even=bool(even), max_kv_len=S4K) for h in range(Hq)])
        rep.append(f"{Hq}/{Hkv} pos {p} n_split {n_split} even {even}: {_ulps(out[0].cpu(), model)} ulp")
    print("\n[kernel vs model] " + "; ".join(rep))
