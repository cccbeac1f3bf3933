"""Shared numerics helpers of the kernel tests: fp16 rounding sides, the fp32 rstd window of the RMSNorm prologues,
NaN-sentinel buffers, set-and-restore of a b200_tune knob, and the line-by-line model of moe_route_kernel's routing.

Test infrastructure only (see oracle/__init__.py).  Every function here is plain torch / numpy; the CUDA library is only
touched by `tuned`, and only when it is entered.
"""
import contextlib
import os

import numpy as np
import torch

SENT = 0x7E5A      # NaN bit pattern: a sentinel no kernel writes
RSTD_ULPS = 32     # the kernels' fp32 rstd lies within this many fp32 ulps of rstd64 (test_decode_path_gpu.py derives it)

# what a b200_tune knob is when neither a b200_tune call nor the environment sets it (csrc: tune_get defaults)
TUNE_DEFAULTS = {"B200_PF_EARLY": 0, "B200_SELF_PF_KB": 0, "B200_STREAM_EF": 1, "B200_QKV_RING_KB": 0, "B200_GEMV1": 1}


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
