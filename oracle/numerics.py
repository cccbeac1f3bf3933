"""Shared numerics helpers of the kernel tests: fp16 rounding sides, the fp32 rstd window of the RMSNorm prologues,
NaN-sentinel buffers, set-and-restore of a b200_tune knob, the line-by-line model of moe_route_kernel's routing, and the
split schedules and step-by-step arithmetic model of the decode attention kernel.

Also the float64 checkers that more than one GPU module applies (their bounds are derived in the docstrings of
tests/test_gemv_batched_moe_gpu.py, sections A and B, and tests/test_attn_decode_gpu.py, section A): the GEMV bound,
the RoPE of the QKV epilogue, the SiLU-product range, the router's logit window and routing check, the float64
reference and bound of decode attention, and the LL unit format, sequence numbers and rank-sum model of the fused
tensor-parallel all-reduce (tests/test_tp_allreduce_gpu.py derives its bound).

Test infrastructure only (see oracle/__init__.py).  Every function here is plain torch / numpy; the CUDA library is only
touched by `tuned`, and only when it is entered.
"""
import contextlib
import itertools
import math
import os

import numpy as np
import torch

SENT = 0x7E5A      # NaN bit pattern: a sentinel no kernel writes
RSTD_ULPS = 32     # the kernels' fp32 rstd lies within this many fp32 ulps of rstd64 (test_decode_path_gpu.py derives it)
C_ACC = 2.0 ** -18       # fp32 accumulation constant of the fp16 HMMA kernels, relative to |x| . |w|^T (test_prefill_gpu.py)
SILU_REL = 2.0 ** -20    # fp32 a / (1 + expf(-a)): <= 3.5 u << 16 u (test_decode_path_gpu.py)
SILU_ARGMIN = -1.2784645427610737  # silu has its only minimum there
MAX_AMB = 12             # router: at most 2^12 rounding choices of ambiguous logits per token

# what a b200_tune knob is when neither a b200_tune call nor the environment sets it (csrc: tune_get defaults)
TUNE_DEFAULTS = {"B200_PF_EARLY": 0, "B200_SELF_PF_KB": 0, "B200_STREAM_EF": 1, "B200_QKV_RING_KB": 0, "B200_GEMV1": 1,
                 "B200_GEMV1_GROUPED": 1, "B200_ATTN_EVEN": 0, "B200_ATTN_MAX_SPLIT": 16, "B200_KV_EF": 1}


def nan16(*shape, device="cuda"):
    """fp16 tensor filled with the SENT NaN pattern: any element a kernel writes differs from it."""
    return torch.full(shape, SENT, dtype=torch.int16, device=device).view(torch.float16)


def fp16_sides(v):
    """float64 v -> (nearest fp16, the other fp16 neighbour, |v - the midpoint between them|), signed like v."""
    a = v.abs()
    _, e = torch.frexp(a)
    # the fp16 spacing 2^(e - 11), built from its exponent bits: the device exp2 need not return exact powers of two
    u = ((e.long() - 11 + 1023).clamp_min(1) << 52).view(torch.float64)
    u = torch.where(a < 2.0 ** -14, torch.full_like(a, 2.0 ** -24), u)
    lo = torch.floor(a / u) * u
    mid = lo + u / 2
    near, alt = torch.where(a < mid, lo, lo + u), torch.where(a < mid, lo + u, lo)
    sg = torch.where(v < 0, -1.0, 1.0).double()
    return sg * near, sg * alt, (a - mid).abs()


def rstd64(h, eps):
    """float64 1 / sqrt(mean(h^2) + eps) of every row of h [..., K] (eps as the fp32 value the kernels add)."""
    hd = h.double().reshape(-1, h.shape[-1])
    return 1.0 / torch.sqrt(hd.pow(2).mean(-1) + float(torch.tensor(eps, dtype=torch.float32)))


def rstd_candidates(h, eps, ulps=RSTD_ULPS):
    """fp32 [rows, 2 ulps + 1]: every fp32 value within `ulps` ulps of each row's rstd64."""
    c = rstd64(h, eps).float().view(torch.int32)
    return (c[:, None] + torch.arange(-ulps, ulps + 1, device=h.device, dtype=torch.int32)).view(torch.float32)


def x_candidates(h, gamma, eps, ulps=RSTD_ULPS):
    """h [K] -> [C, K] fp16: x = fp16(fp16(h * rstd) * gamma) for every distinct x that an fp32 rstd of the window gives."""
    rs = rstd_candidates(h.reshape(1, -1), eps, ulps)[0]
    x = (h.float().reshape(1, -1) * rs[:, None]).half() * gamma.reshape(1, -1)
    return torch.unique(x.view(torch.int16), dim=0).view(torch.float16)


@contextlib.contextmanager
def tuned(name, value):
    """A b200_tune override lasts for the whole process: put the knob back to what the environment gives on exit."""
    from llama2_accessory_b200 import _cabi
    lib = _cabi.lib()
    assert lib.b200_tune(name.encode(), value) == 0
    try:
        yield
    finally:
        lib.b200_tune(name.encode(), int(os.environ.get(name, TUNE_DEFAULTS[name])))


# ------------------------------------------------------------------------------------------- moe_route model --------
def kernel_scores(logits16):
    """fp16 [T, E] gate logits -> fp32 [T, E] fp16-valued scores: the fp32 softmax of kernel_scores_f32 rounded to fp16."""
    return kernel_scores_f32(logits16).astype(np.float16).astype(np.float32)


def _route_top_k(sc, k):
    """Top-k of fp32 scores [T, E] in rank order, ties to the lower index (the kernel's strict `>` scan from e = 0)."""
    T, E = sc.shape
    idx = np.zeros((T, k), dtype=np.int64)
    val = np.zeros((T, k), dtype=np.float32)
    used = np.zeros((T, E), dtype=bool)
    for j in range(k):
        masked = np.where(used, -np.inf, sc)
        b = masked.argmax(-1)                          # first maximum = lowest index on ties
        idx[:, j], val[:, j] = b, masked[np.arange(T), b]
        used[np.arange(T), b] = True
    return idx, val


def kernel_route(logits16, k):
    """logits16: fp16 [T, E] -> (idx int64 [T, k], weight fp16 [T, k]) following moe.cu line by line (numpy fp32)."""
    idx, val = _route_top_k(kernel_scores(logits16), k)
    s = np.zeros(idx.shape[0], dtype=np.float32)
    for j in range(k):
        s = (s + val[:, j]).astype(np.float32)
    s16 = s.astype(np.float16).astype(np.float32)
    w = (val / s16[:, None]).astype(np.float32).astype(np.float16)
    return torch.from_numpy(idx), torch.from_numpy(w)


def kernel_scores_f32(logits16):
    """fp16 [T, E] gate logits -> fp32 [T, E] unrounded scores of moe_route_kernel<true>: expf(l - max) / den, den the
    fp32 sum of the exponentials over the experts in index order (thread 0's loop)."""
    lg = logits16.float().cpu().numpy()
    ex = np.exp((lg - lg.max(-1, keepdims=True)).astype(np.float32)).astype(np.float32)
    den = np.zeros(lg.shape[0], dtype=np.float32)
    for e in range(lg.shape[1]):
        den = (den + ex[:, e]).astype(np.float32)
    return (ex / den[:, None]).astype(np.float32)


def kernel_route_f32(logits16, k):
    """logits16: fp16 [T, E] -> (idx int64 [T, k], weight fp16 [T, k]) following moe_route_kernel<true> line by line
    (numpy fp32): top-k on the unrounded fp32 scores (ties to the lower index), the fp32 sum of the chosen scores in rank
    order, weight = fp16(score / sum) rounded once (mixtral_sparse.py:417-428)."""
    idx, val = _route_top_k(kernel_scores_f32(logits16), k)
    s = np.zeros(idx.shape[0], dtype=np.float32)
    for j in range(k):
        s = (s + val[:, j]).astype(np.float32)
    w = (val / s[:, None]).astype(np.float32).astype(np.float16)
    return torch.from_numpy(idx), torch.from_numpy(w)


def route_f32(logits16, k):
    """mixtral_sparse.py:417-428 stated in torch on fp16 logits [T, E]: fp32 softmax, top-k on the fp32 scores (ties:
    lower index), fp32 renormalisation, one cast to fp16.  -> (idx int64 [T, k], weight fp16 [T, k])."""
    p = torch.softmax(logits16.float(), dim=-1)
    w, idx = torch.topk(p, k, dim=-1)
    return idx, (w / w.sum(-1, keepdim=True)).half()


# The fp32 rule's window.  The device expf is within 2 fp32 ulps of exp (CUDA C Programming Guide, its maximum ulp error),
# numpy's float32 exp within 2.5 (measured over [-40, 0]); EXPF_REL = 8 ulps = 2^-20 covers the two with room.  Everything
# else the kernel computes exactly as kernel_scores_f32 does, so a score moves by at most
#   numerator EXPF_REL, denominator EXPF_REL on the exact sum plus (E - 1) u of the sequential fp32 sum on each side,
#   the division u on each side:                      W(E) = 2 EXPF_REL + 2 E u            (u = 2^-24, relative)
# and a weight score / sum, the fp32 sum of k scores:  2 W(E) + 2 k u.
EXPF_REL = 2.0 ** -20


def route_f32_window(E):
    return 2 * EXPF_REL + 2 * E * 2.0 ** -24


def route_weight_window(E, k):
    return 2 * route_f32_window(E) + 2 * k * 2.0 ** -24


def route_f32_explains(lg16, se, sw16, k):
    """True when slot_expert se [k] / slot_weight sw16 [k] (fp16 bits, int16) of one token are a moe_route_kernel<true>
    outcome for fp16 logits lg16 [E] whose exponentials differ from numpy's within EXPF_REL: expert se[j] may stand where the
    scores give another only when the two fp32 scores lie within the window W(E) of each other (the scan is greedy, so
    every pick is judged against every expert not picked before it), and a weight may take the other fp16 rounding of
    score / sum only when that quotient lies within the weight window of an fp16 midpoint."""
    sc = kernel_scores_f32(lg16.reshape(1, -1))[0].astype(np.float64)
    E = sc.shape[0]
    W, RW = route_f32_window(E), route_weight_window(E, k)
    se = [int(e) for e in se]
    if len(set(se)) != k or not all(0 <= e < E for e in se):
        return False
    for j, e in enumerate(se):
        rest = [o for o in range(E) if o not in se[:j + 1]]
        if any(sc[o] - sc[e] > W * (sc[o] + sc[e]) for o in rest):
            return False
    val = sc[se].astype(np.float32)
    s = np.float32(0)
    for v in val:
        s = np.float32(s + v)
    r = torch.from_numpy((val / s).astype(np.float32).astype(np.float64))
    near, alt, dist = fp16_sides(r)
    got = torch.from_numpy(np.asarray(sw16, dtype=np.int16).view(np.float16).astype(np.float64))
    ok = (got == near) | ((got == alt) & (dist <= RW * r.abs()))
    return bool(ok.all())


# ------------------------------------------------------------------------------------- decode attention model --------
ATTN_TILE, ATTN_WARPS = 32, 4      # kv positions per tile, consumer warps per CTA (csrc/attn.cu kTile, kAttnWarps)


def _cdiv(a, b):
    return -(-a // b)


def attn_choose_split(T, Hkv, max_kv_len, sms, cap=16):
    """b200_attn_choose_split: enough splits for two CTAs per SM, at most one per 128 keys, capped at `cap`
    (B200_ATTN_MAX_SPLIT) only while the capped grid still gives every SM a CTA; then rounded to whole 32-key chunks."""
    if T <= 0 or Hkv <= 0 or max_kv_len <= 0:
        return 1
    want = 2 * sms // (T * Hkv)
    want = max(1, min(want, _cdiv(max_kv_len, ATTN_WARPS * ATTN_TILE)))
    if want > cap and T * Hkv * cap >= sms:
        want = max(cap, 1)
    chunk = _cdiv(_cdiv(max_kv_len, want), ATTN_TILE) * ATTN_TILE
    return _cdiv(max_kv_len, chunk)


def attn_host_split(max_kv_len, n_split):
    """b200_attn_decode: a requested split count -> (split count launched, chunk).  The chunk is a whole number of tiles,
    so a request above max_kv_len / 32 launches one split per tile."""
    chunk = _cdiv(_cdiv(max_kv_len, n_split), ATTN_TILE) * ATTN_TILE
    return _cdiv(max_kv_len, chunk), chunk


def attn_split_ranges(kv_len, n_split, chunk, even):
    """[(s_begin, s_end)] of every split of one token whose keys are 0 .. kv_len - 1 (attn_decode_kernel); s_end <= s_begin
    is an empty split.
      even = 0: equal chunks rounded up to whole tiles, sized for the ACTUAL kv_len but never above the launch's chunk;
      even = 1 (B200_ATTN_EVEN): the n_t tiles holding keys dealt out, split i taking tiles [n_t i / n, n_t (i + 1) / n)."""
    out = []
    for sp in range(n_split):
        if even:
            n_t = _cdiv(kv_len, ATTN_TILE)
            b, e = n_t * sp // n_split * ATTN_TILE, min(kv_len, n_t * (sp + 1) // n_split * ATTN_TILE)
        else:
            c = min(chunk, _cdiv(_cdiv(kv_len, n_split), ATTN_TILE) * ATTN_TILE)
            b = sp * c
            e = min(kv_len, b + c)
        out.append((b, max(b, e)))
    return out


def attn_kernel_model(q, k, v, n_split, even=False, max_kv_len=None):
    """q fp16 [128], k / v fp16 [n, 128] (positions 0 .. pos) -> fp16 [128], following attn.cu step by step in torch fp32.

        scores   fp16 q . fp16 k accumulated in fp32, times scale_log2 = fp32(fp32(1/sqrt(128)) * fp32(log2 e))
        splits   the grid b200_attn_decode launches for (max_kv_len, n_split), cut by attn_split_ranges
        warps    inside a split, tile i belongs to consumer warp i % 4; a warp folds ITS tiles in order with the online rule
                 m' = max(m, max_tile), corr = 2^(m - m'), l = l corr + sum(fp16(p)), O = O corr + fp16(p) V, p = 2^(s - m')
        merge    4 warps, then the splits in split order: M = max m, f = 2^(m - M) (0 for an empty part), L = sum l f,
                 o = sum O f; out = fp16(o / L)
    The kernel's HMMA accumulates in another order and its exp2f is not torch's exp2: the model and the kernel agree to a
    few fp16 steps, not bit for bit."""
    n = k.shape[0]
    ns, chunk = attn_host_split(max_kv_len or n, n_split)
    scale_log2 = torch.tensor(1.0 / math.sqrt(128.0), dtype=torch.float32) * torch.tensor(1.4426950408889634,
                                                                                          dtype=torch.float32)
    s_all = (k.float() @ q.float()) * scale_log2                                         # fp32 accumulation of exact products
    ninf = torch.tensor(-math.inf)

    def fold(parts):                                                                     # [(m, l, o)] in order -> (M, L, o)
        M = torch.stack([m for m, _, _ in parts]).max()
        L, o = torch.tensor(0.0), torch.zeros(128)
        for m, l, oo in parts:
            f = torch.tensor(0.0) if m == -math.inf else torch.exp2(m - M)
            L, o = L + l * f, o + oo * f
        return M, L, o
    splits = []
    for s_begin, s_end in attn_split_ranges(n, ns, chunk, even):
        n_tiles = _cdiv(s_end - s_begin, ATTN_TILE)
        warps = []
        for w in range(ATTN_WARPS):
            m, l, o = ninf, torch.tensor(0.0), torch.zeros(128)
            for i in range(w, n_tiles, ATTN_WARPS):
                a, b = s_begin + i * ATTN_TILE, min(s_end, s_begin + (i + 1) * ATTN_TILE)
                s = s_all[a:b]
                m_new = torch.maximum(m, s.max())
                corr = torch.exp2(m - m_new)
                p16 = torch.exp2(s - m_new).half()                                       # P rounded for the second MMA
                l = l * corr + p16.float().sum()
                o = o * corr + p16.float() @ v[a:b].float()
                m = m_new
            warps.append((m, l, o))
        splits.append(fold(warps))
    _, L, o = fold(splits)
    return (o / L).half()


# ------------------------------------------------------------------------------------------- GEMV bound ------------
def _bits16(t):
    return t.contiguous().view(torch.int16)


def gemv_tol(ref, M):
    """The element-wise bound of the multi-token GEMV against float64 ref, M = A . |x| (test_gemv_batched_moe_gpu.py, A)."""
    return ref.abs() * 2.0 ** -11 + C_ACC * M * (1 + 2.0 ** -10) + 2.0 ** -25


def gemv_check(out, ref, M, label):
    """out [T, N] against float64 ref with the GEMV bound -> (worst err / tol, implied C, exact fraction)."""
    o = out.double()
    assert torch.isfinite(o).all(), label
    err = (o - ref).abs()
    tol = gemv_tol(ref, M)
    ratio = float((err / tol).max())
    c_seen = float(((err - ref.abs() * 2.0 ** -11).clamp_min(0) / M.clamp_min(1e-30)).max())
    exact = float((_bits16(out) == _bits16(ref.half())).double().mean())
    assert ratio <= 1.0, (label, ratio)
    return ratio, c_seen, exact


def rope_rotate(y16, cs):
    """fp32 RoPE of the QKV epilogue as separate multiplies and adds: y16 [rows] fp16 of whole heads, cs [rows / 2, 2]."""
    p = y16.float().reshape(-1, 2)
    e, o = p[:, 0], p[:, 1]
    c, s = cs[:, 0], cs[:, 1]
    return torch.stack([e * c - o * s, e * s + o * c], dim=-1).reshape(-1).half()


def qkv_from_y(y, rope, pos, n_q_rows, n_kv_rows):
    """The QKV epilogue's outputs as a function of the F16 launch's y [T, n_q + 2 n_kv] on the same inputs -> (q [T, n_q],
    k [T, n_kv], v [T, n_kv]) fp16: q and k rotated by rope[pos[t]], v = y."""
    rows = []
    for t in range(y.shape[0]):
        cs = rope[int(pos[t])].repeat((n_q_rows + n_kv_rows) // 128, 1)
        rows.append(rope_rotate(y[t, :n_q_rows + n_kv_rows], cs))
    r = torch.stack(rows)
    return r[:, :n_q_rows], r[:, n_q_rows:], y[:, n_q_rows + n_kv_rows:]


def silu_mul_range(ya, ta, yb, tb):
    """[lo, hi] of fp16(fp16(silu(a)) * b) over every fp16 a = fp16(y), |y - ya| <= ta (b likewise): fp16 rounding and
    the product are monotone, silu is monotone on each side of its minimum, and the fp32 silu lies within SILU_REL."""
    def silu(a):
        return a / (1 + torch.exp(-a))
    a_lo, a_hi = (ya - ta).half().double(), (ya + ta).half().double()
    b_lo, b_hi = (yb - tb).half().double(), (yb + tb).half().double()
    s1, s2 = silu(a_lo), silu(a_hi)
    smin = torch.minimum(s1, s2)
    smin = torch.where((a_lo <= SILU_ARGMIN) & (a_hi >= SILU_ARGMIN), torch.full_like(smin, silu(torch.tensor(SILU_ARGMIN, dtype=torch.float64)).item()), smin)
    smax = torch.maximum(s1, s2)
    s_lo = (smin - SILU_REL * smin.abs()).half().double()
    s_hi = (smax + SILU_REL * smax.abs()).half().double()
    c = torch.stack([s_lo * b_lo, s_lo * b_hi, s_hi * b_lo, s_hi * b_hi])
    return c.amin(0).half().double(), c.amax(0).half().double()


# -------------------------------------------------------------------------------------------- router check ----------
def logit_window(xn, gate):
    """float64 logits and the running-error bound R of moe_route_kernel's lane chains + warp tree
    (test_gemv_batched_moe_gpu.py, B)."""
    T, D = xn.shape
    E = gate.shape[0]
    p = xn.double()[:, None, :] * gate.double()[None]                       # [T, E, D] exact products
    # lane l owns uint4 chunks u = l, l + 32, ...: elements 8u .. 8u + 7 in order
    p = p.reshape(T, E, D // 256, 32, 8).permute(0, 1, 3, 2, 4).reshape(T, E, 32, D // 32)
    part = p.cumsum(-1)
    lane = part[..., -1]
    R = 2.0 ** -24 * (part.abs().sum(-1).sum(-1) + 5 * lane.abs().sum(-1)) * (1 + 2.0 ** -10)
    L = lane.sum(-1)
    assert bool((R <= (D / 32 + 5) * 2.0 ** -24 * (xn.double().abs() @ gate.double().abs().T) * 1.01).all())
    return L, R


def route_scores32(logits16):
    """fp16 [T, E] logits -> the kernel's fp32 softmax scores (experts summed in index order) as float64, unrounded."""
    return torch.from_numpy(kernel_scores_f32(logits16)).double()


def route_check(xn, gate, sw, se, k, max_amb=MAX_AMB):
    """moe_route's slot_expert / slot_weight [T, k] against every kernel_route outcome of the logit window of its own
    xn_out -> (tokens matched bit for bit, tokens in the expf window, tokens with too many ambiguous logits)."""
    L, R = logit_window(xn, gate)
    near, alt, dist = fp16_sides(L)
    amb = (dist <= R).cpu()
    near, alt = near.cpu(), alt.cpu()
    se_c, sw_c = se.cpu().long(), _bits16(sw).cpu()
    matched = window = skipped = 0
    for t in range(L.shape[0]):
        ai = torch.nonzero(amb[t]).reshape(-1).tolist()
        if len(ai) > max_amb:
            skipped += 1
            continue
        combos = torch.tensor(list(itertools.product([0, 1], repeat=len(ai))), dtype=torch.bool).reshape(2 ** len(ai), len(ai))
        C = near[t].repeat(combos.shape[0], 1)
        if ai:
            C[:, ai] = torch.where(combos, alt[t, ai][None].expand_as(combos), near[t, ai][None].expand_as(combos))
        lg16 = C.half()
        idx, w = kernel_route(lg16, k)
        hit = (idx == se_c[t][None]).all(1) & (w.view(torch.int16) == sw_c[t][None]).all(1)
        if bool(hit.any()):
            matched += 1
            continue
        s = route_scores32(lg16)
        _, _, sd = fp16_sides(s)
        assert bool((sd <= 2.0 ** -20 * s.abs()).any()), (t, se_c[t].tolist(), idx[:4].tolist())
        window += 1
    return matched, window, skipped


def route_check_f32(xn, gate, sw, se, k, max_amb=MAX_AMB):
    """route_check for the fp32 score rule (moe_route_kernel<true>): every token's slot_expert / slot_weight [T, k] must be
    a kernel_route_f32 outcome, bit for bit, for some fp16 rounding of its ambiguous logits, or one that
    route_f32_explains within the expf window -> (tokens matched bit for bit, tokens in the window, tokens with too many
    ambiguous logits)."""
    L, R = logit_window(xn, gate)
    near, alt, dist = fp16_sides(L)
    amb = (dist <= R).cpu()
    near, alt = near.cpu(), alt.cpu()
    se_c, sw_c = se.cpu().long(), _bits16(sw).cpu()
    matched = window = skipped = 0
    for t in range(L.shape[0]):
        ai = torch.nonzero(amb[t]).reshape(-1).tolist()
        if len(ai) > max_amb:
            skipped += 1
            continue
        combos = torch.tensor(list(itertools.product([0, 1], repeat=len(ai))), dtype=torch.bool).reshape(2 ** len(ai), len(ai))
        C = near[t].repeat(combos.shape[0], 1)
        if ai:
            C[:, ai] = torch.where(combos, alt[t, ai][None].expand_as(combos), near[t, ai][None].expand_as(combos))
        lg16 = C.half()
        idx, w = kernel_route_f32(lg16, k)
        hit = (idx == se_c[t][None]).all(1) & (w.view(torch.int16) == sw_c[t][None]).all(1)
        if bool(hit.any()):
            matched += 1
            continue
        assert any(route_f32_explains(lg16[c], se_c[t].numpy(), sw_c[t].numpy(), k) for c in range(lg16.shape[0])), (
            t, "fp32 rule", se_c[t].tolist(), sw_c[t].view(torch.float16).tolist(), idx[:4].tolist(),
            w[:4].float().tolist())
        window += 1
    return matched, window, skipped


# ------------------------------------------------------------------------------------ decode attention bound --------
ATTN_U = 2.0 ** -24
ATTN_EXP2_REL = 2.0 ** -22           # exp2f: 2 ulp
ATTN_C_LOG2 = 1.4426950408889634 / math.sqrt(128.0)


def attn_tiles_per_warp(kv_len, n_split, chunk, even):
    """largest number of tiles one consumer warp of attn_decode_kernel folds for a token."""
    return max(_cdiv(_cdiv(e - b, ATTN_TILE), ATTN_WARPS) for b, e in attn_split_ranges(kv_len, n_split, chunk, even))


class AttnRef:
    """float64 attention of every (token, head) of a decode-attention launch and the sums its bound is made of
    (test_attn_decode_gpu.py, A).  q [T, Hq, 128], k / v canonical [B, Hkv, S, 128] fp16, token t of sequence t // tps
    attends to rows 0 .. pos[t]."""

    def __init__(self, q, k, v, pos, tps):
        T, Hq, _ = q.shape
        Hkv = k.shape[1]
        r = Hq // Hkv
        dev = q.device
        z3 = lambda: torch.zeros(T, Hq, 128, dtype=torch.float64, device=dev)  # noqa: E731
        z2 = lambda: torch.zeros(T, Hq, dtype=torch.float64, device=dev)  # noqa: E731
        self.out, self.s_eps, self.s_dev, self.s_sub, self.s_absv = z3(), z3(), z3(), z3(), z3()
        self.sw, self.w_eps, self.n_sub = z2(), z2(), z2()
        self.pos = [int(p) for p in pos]
        for t in range(T):
            b, n = t // tps, self.pos[t] + 1
            for g in range(Hkv):
                hs = slice(g * r, (g + 1) * r)
                qq, kk, vv = q[t, hs].double(), k[b, g, :n].double(), v[b, g, :n].double()
                tl = (qq @ kk.T) * ATTN_C_LOG2
                tmax = tl.max(-1, keepdim=True).values
                w = torch.exp2(tl - tmax)
                sw = w.sum(-1)
                o = (w @ vv) / sw[:, None]
                dlt = C_ACC * ATTN_C_LOG2 * (qq.abs() @ kk.abs().T) + 16 * ATTN_U * torch.maximum(tl.abs(), tmax.abs())
                eps = torch.exp2(dlt) - 1 + 2.0 ** -11
                sub = (w < 2.0 ** -13).double()
                dev_ = (vv[None] - o[:, None]).abs()
                self.out[t, hs], self.sw[t, hs] = o, sw
                self.s_eps[t, hs] = torch.einsum("rn,rnd->rd", w * eps, dev_)
                self.s_dev[t, hs] = torch.einsum("rn,rnd->rd", w, dev_)
                self.s_sub[t, hs] = torch.einsum("rn,rnd->rd", sub, dev_)
                self.s_absv[t, hs] = w @ vv.abs()
                self.w_eps[t, hs], self.n_sub[t, hs] = (w * eps).sum(-1), sub.sum(-1)

    def tol(self, tpw, n_split):
        """tpw: tiles per warp of every token (list)."""
        U = ATTN_U
        tw = torch.tensor(tpw, dtype=torch.float64, device=self.out.device).view(-1, 1)
        ec = (tw + 3) * ATTN_EXP2_REL
        den = self.sw - self.w_eps - ec * self.sw - 2.0 ** -25 * self.n_sub
        assert bool((den > 0).all())
        p_err = (2 * (self.s_eps + ec[..., None] * self.s_dev) + 2 * 2.0 ** -25 * self.s_sub) / den[..., None]
        acc = ((C_ACC + (tw[..., None] + n_split + 8) * U) * self.s_absv / self.sw[..., None]
               + (5 * tw[..., None] + n_split // 32 + 20) * U * self.out.abs())
        return (p_err + acc) * (1 + 2.0 ** -11) + 2.0 ** -11 * self.out.abs() + 2.0 ** -25

    def ratio(self, out, n_split, chunk, even):
        """max err / tol of the kernel's out [T, Hq, 128] launched with (n_split, chunk) under schedule `even`."""
        assert bool(torch.isfinite(out).all()), "non-finite output"
        tpw = [attn_tiles_per_warp(p + 1, n_split, chunk, even) for p in self.pos]
        return float(((out.double() - self.out).abs() / self.tol(tpw, n_split)).max())


# ------------------------------------------------------------------- fused tensor-parallel all-reduce (ll.cuh) --------
# An LL buffer holds [tp][N / 2] 8-byte units {payload, seq}: payload = fp16 bits of row 2j (low half) | row 2j + 1 (high
# half) << 16, seq = the sequence number of the step that wrote it (tests/test_tp_allreduce_gpu.py derives the rank-sum
# bound).  Units are numpy int32 [..., 2] here, as they lie in memory.
LL_SENT = 0x7E5A7E5A     # one 32-bit word of two SENT halves: the sentinel of an LL buffer no kernel wrote


def ll_seq(step, period, ident):
    """The sequence number a launch stores / expects: (step * period + id + 1) mod 2^32, as uint32."""
    return (int(step) * int(period) + int(ident) + 1) % (1 << 32)


def ll_encode(parts16, seq):
    """fp16 partials [tp, N] (numpy float16) -> int32 units [tp, N / 2, 2] carrying `seq`."""
    bits = np.ascontiguousarray(parts16, dtype=np.float16).view(np.uint16).astype(np.uint32)
    pay = bits[:, 0::2] | (bits[:, 1::2] << 16)
    units = np.empty(pay.shape + (2,), dtype=np.uint32)
    units[..., 0], units[..., 1] = pay, np.uint32(seq)
    return units.view(np.int32)


def ll_decode(units):
    """int32 units [tp, N / 2, 2] -> (fp16 payloads [tp, N], uint32 sequence numbers [tp, N / 2])."""
    u = np.ascontiguousarray(units).view(np.uint32)
    pay, seq = u[..., 0], u[..., 1]
    halves = np.stack([pay & 0xFFFF, pay >> 16], axis=-1).astype(np.uint16)
    return halves.reshape(u.shape[0], -1).view(np.float16), seq


def ll_rank_sum32(parts16, order=None):
    """fp32 running sum of the partials [tp, N] (numpy float32), in rank order or in the given order of ranks."""
    p = np.asarray(parts16, dtype=np.float16).astype(np.float32)
    order = range(p.shape[0]) if order is None else order
    acc = None
    for r in order:
        acc = p[r].copy() if acc is None else (acc + p[r]).astype(np.float32)
    return acc


def ll_rank_sum(parts16, order=None):
    """The consumer's delta: the rank-order fp32 sum rounded once to fp16."""
    return ll_rank_sum32(parts16, order).astype(np.float16)


def ll_units_decode32(units):
    """int32 LL units [..., 2] whose payload is an fp32 (the attention partials of mega2.cu) -> (float32 payloads, uint32
    sequence numbers)."""
    u = np.ascontiguousarray(units).view(np.uint32)
    return u[..., 0].copy().view(np.float32), u[..., 1].copy()


# ------------------------------------------------------------ persistent whole-step kernels (mega1.cu, mega2.cu) --------
MEGA_TILE, MEGA_WARPS = 32, 16     # kv positions per attention tile, MMA warps per CTA (kTileKV, kConsumerWarps)


def mega_split_ranges(kv_len, n_split):
    """attn_item of mega1.cu / mega2.cu: [(s_begin, s_end)] of every split, equal chunks of whole 32-key tiles sized for
    kv_len; s_end == s_begin is an empty split.  Tile i of a split belongs to MMA warp i % 16."""
    chunk = _cdiv(_cdiv(kv_len, n_split), MEGA_TILE) * MEGA_TILE
    return [(min(kv_len, sp * chunk), min(kv_len, (sp + 1) * chunk)) for sp in range(n_split)]


def mega_tiles_per_warp(kv_len, n_split):
    """largest number of tiles one MMA warp of the persistent kernels folds for one (kv head, split) item."""
    return max(_cdiv(_cdiv(e - b, MEGA_TILE), MEGA_WARPS) for b, e in mega_split_ranges(kv_len, n_split))


def mega_past_boundary_pos(n_split):
    """A position whose kv_len = pos + 1 puts exactly one key into the last of n_split splits (chunk 32 n_split)."""
    return MEGA_TILE * n_split * (n_split - 1)


def mega1_comm_offsets(n_layers, dim, tp=1):
    """(parts, logits) byte offsets of mega1's communication block: u32 counters [5L + 3] padded to 256 B, then fp16
    partials [2][tp][dim] (wo | w2) padded to 256 B, then fp32 logits (b200_step1_comm_logits_offset)."""
    bar = ((5 * n_layers + 3) * 4 + 255) // 256 * 256
    return bar, bar + (2 * tp * dim * 2 + 255) // 256 * 256


def ll_layout(n_layers, D, Hq, Hkv, F, V, n_split, tp=1):
    """Byte offsets of mega2's communication block (make_layout): ctl | yq | ykv | att | po | act | pf | logits | total."""
    al = lambda v: (v + 255) // 256 * 256  # noqa: E731
    sizes = [("ctl", 64 + (5 * n_layers + 1) * 4), ("yq", Hq * 128 * 4), ("ykv", Hkv * 2 * 128 * 4),
             ("att", Hq * n_split * 130 * 8), ("po", tp * D * 4), ("act", F * 4), ("pf", tp * D * 4), ("logits", V * tp * 4)]
    off, out = 0, {}
    for k, n in sizes:
        out[k] = off
        off = al(off + n)
    out["total"] = off
    return out


def merge_splits64(O, m, lsum):
    """float64 cross-split merge of per-split partials O [H, ns, 128], m, l [H, ns] (log2 units) -> [H, 128], and the
    magnitude sum_sp |O_sp| f_sp / L that bounds the fp32 rounding of the kernels' own merge."""
    O, m, lsum = O.double(), m.double(), lsum.double()
    M = m.max(-1, keepdim=True).values
    f = torch.where(torch.isinf(m), torch.zeros_like(m), torch.exp2(m - M))
    L = (lsum * f).sum(-1, keepdim=True)
    return (O * f[..., None]).sum(1) / L, (O.abs() * f[..., None]).sum(1) / L


def ll_rank_sum_bound(parts16):
    """-> (float64 exact sum s, bound) with |delta - s| <= 1/2 ulp16(s32) + (tp - 1) 2^-24 sum |p_r| (1 + 2^-20): tp - 1
    fp32 additions, each off by at most 2^-24 of a partial sum bounded by sum |p_r| (up to its own rounding), then one
    fp16 rounding of the fp32 sum s32 (half an fp16 spacing at |s32|; 2^-25 below the normal range)."""
    p = np.asarray(parts16, dtype=np.float16).astype(np.float64)
    s32 = np.abs(ll_rank_sum32(parts16).astype(np.float64))
    half_ulp = 2.0 ** (np.floor(np.log2(np.maximum(s32, 2.0 ** -14))) - 11)
    return p.sum(0), half_ulp + (p.shape[0] - 1) * 2.0 ** -24 * np.abs(p).sum(0) * (1 + 2.0 ** -20)
