"""Shared numerics helpers of the kernel tests: fp16 rounding sides, the fp32 rstd window of the RMSNorm prologues,
NaN-sentinel buffers, set-and-restore of a b200_tune knob, the line-by-line model of moe_route_kernel's routing, and the
split schedules and step-by-step arithmetic model of the decode attention kernel.

Test infrastructure only (see oracle/__init__.py).  Every function here is plain torch / numpy; the CUDA library is only
touched by `tuned`, and only when it is entered.
"""
import contextlib
import math
import os

import numpy as np
import torch

SENT = 0x7E5A      # NaN bit pattern: a sentinel no kernel writes
RSTD_ULPS = 32     # the kernels' fp32 rstd lies within this many fp32 ulps of rstd64 (test_decode_path_gpu.py derives it)

# what a b200_tune knob is when neither a b200_tune call nor the environment sets it (csrc: tune_get defaults)
TUNE_DEFAULTS = {"B200_PF_EARLY": 0, "B200_SELF_PF_KB": 0, "B200_STREAM_EF": 1, "B200_QKV_RING_KB": 0, "B200_GEMV1": 1,
                 "B200_ATTN_EVEN": 0, "B200_ATTN_MAX_SPLIT": 16, "B200_KV_EF": 1}


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
    """fp16 [T, E] gate logits -> fp32 [T, E] fp16-valued scores: fp32 softmax with the experts summed in index order."""
    lg = logits16.float().cpu().numpy()
    ex = np.exp((lg - lg.max(-1, keepdims=True)).astype(np.float32)).astype(np.float32)
    den = np.zeros(lg.shape[0], dtype=np.float32)
    for e in range(lg.shape[1]):                       # sequential fp32 sum over experts, as thread 0 does
        den = (den + ex[:, e]).astype(np.float32)
    return (ex / den[:, None]).astype(np.float32).astype(np.float16).astype(np.float32)


def kernel_route(logits16, k):
    """logits16: fp16 [T, E] -> (idx int64 [T, k], weight fp16 [T, k]) following moe.cu line by line (numpy fp32)."""
    sc = kernel_scores(logits16)
    T, E = sc.shape
    idx = np.zeros((T, k), dtype=np.int64)
    val = np.zeros((T, k), dtype=np.float32)
    used = np.zeros((T, E), dtype=bool)
    for j in range(k):
        masked = np.where(used, -np.inf, sc)
        b = masked.argmax(-1)                          # first maximum = lowest index on ties
        idx[:, j], val[:, j] = b, masked[np.arange(T), b]
        used[np.arange(T), b] = True
    s = np.zeros(T, dtype=np.float32)
    for j in range(k):
        s = (s + val[:, j]).astype(np.float32)
    s16 = s.astype(np.float16).astype(np.float32)
    w = (val / s16[:, None]).astype(np.float32).astype(np.float16)
    return torch.from_numpy(idx), torch.from_numpy(w)


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
