"""CPU: the top-p threshold search of csrc/sample.cu's large-vocabulary kernel (sample_top_p_radix_kernel), emulated in
numpy on the probabilities as the kernel forms them, equals the nucleus rule -- cut = the smallest probability whose
strictly-larger mass is <= top_p -- stated directly by sorting; and b200_sample_top_p's host-side checks accept
vocabularies that do not fit in shared memory (V > 57856 with the H100's 227 KB opt-in) instead of refusing them.  The
return code cannot tell which of the two kernels was launched: the switch between them is exercised on the GPU, at
V = 57856 / 57857 in tests/test_sample_large_vocab_gpu.py.

The emulation follows the kernel step for step: 4 radix passes of 8 bits over the bit pattern of p, masses summed in
2^-56 fixed point (a p > 0 below 2^-56 counts as 2^-56), the lowest non-empty bin whose largest member has at most
top_p of mass strictly above it."""
import numpy as np
import pytest
import torch

from oracle import sampling

FIX = 2.0 ** 56


def _fixed_mass(prob):
    f = np.floor(prob.astype(np.float64) * FIX).astype(np.uint64)  # exact: p * 2^56 has p's 24 significant bits
    return np.where(prob > 0, np.maximum(f, np.uint64(1)), np.uint64(0))


def _limit(top_p):
    return int(np.floor(np.float64(np.float32(top_p)) * FIX))


def radix_cut(prob, top_p):
    """The kernel's descent -> cut (fp32); the kept set is p >= cut, p > 0."""
    if top_p >= 1.0:
        return np.float32(0)
    bits, mass, limit = prob.view(np.uint32), _fixed_mass(prob), _limit(top_p)
    prefix, above = 0, 0
    for shift in (24, 16, 8, 0):
        fixed = 0 if shift == 24 else (0xFFFFFFFF << (shift + 8)) & 0xFFFFFFFF
        sel = (prob > 0) & ((bits & np.uint32(fixed)) == np.uint32(prefix))
        hist = np.zeros(256, np.uint64)
        np.add.at(hist, (bits[sel] >> np.uint32(shift)) & np.uint32(255), mass[sel])
        a, found = above, None
        for d in range(255, -1, -1):           # from the top bin down; the last qualifying bin is the lowest
            if hist[d] and a <= limit:
                found = (d, a)
            a += int(hist[d])
        assert found is not None
        prefix |= found[0] << shift
        above = found[1]
    return np.uint32(prefix).view(np.float32)


def sorted_cut(prob, top_p):
    """The rule by sorting, with the same exact fixed-point masses."""
    if top_p >= 1.0:
        return np.float32(0)
    pos = prob[prob > 0]
    vals, inv = np.unique(pos, return_inverse=True)        # ascending distinct probabilities
    group = np.zeros(vals.size, np.uint64)
    np.add.at(group, inv, _fixed_mass(pos))
    strictly_above = np.concatenate([np.cumsum(group[::-1])[::-1][1:], [np.uint64(0)]])
    return vals[np.nonzero(strictly_above <= np.uint64(_limit(top_p)))[0][0]]


def _prob32(logits, temperature):
    return sampling.nucleus_bisect(logits, temperature, 1.0)[0]  # softmax as the kernels form it


@pytest.mark.parametrize("V,temperature,top_p", [(103168, 1.0, 0.9), (103168, 0.7, 0.5), (57857, 1.3, 0.95),
                                                  (256000, 1.0, 0.99), (32000, 0.3, 0.05), (4096, 1.0, 1e-6)])
def test_radix_descent_equals_the_sorted_rule(V, temperature, top_p):
    g = torch.Generator().manual_seed(V + int(top_p * 1000))
    for _ in range(3):
        logits = (torch.randn(V, generator=g) * 2.5).float()
        prob = _prob32(logits.numpy(), temperature)
        cut = radix_cut(prob, top_p)
        assert cut == sorted_cut(prob, top_p)
        kept = (prob >= cut) & (prob > 0)
        assert kept[int(torch.argmax(logits))]
        # against meta.py:558-561 itself: disagreement only on a token sitting on the cut within fp32 summation noise
        ref = sampling.nucleus_reference(torch.from_numpy(prob), top_p).numpy()
        diff = np.nonzero(ref != kept)[0]
        if diff.size:
            order = np.argsort(-prob, kind="stable")
            before = np.cumsum(prob[order].astype(np.float64)) - prob[order]
            pos = np.empty(V, np.int64)
            pos[order] = np.arange(V)
            assert all(abs(before[pos[i]] - top_p) < 2e-6 for i in diff), diff


def test_radix_descent_keeps_ties_together_and_handles_degenerate_rows():
    # three tokens at 0.2 with 0.3 strictly above: all three stay at top_p = 0.6, as in the shared-memory kernel
    prob = np.array([0.3, 0.2, 0.2, 0.2, 0.1], np.float32)
    big = np.zeros(70000, np.float32)
    big[[5, 70, 600, 6000, 69999]] = prob
    for p in (prob, big):
        cut = radix_cut(p, 0.6)
        assert cut == np.float32(0.2) == sorted_cut(p, 0.6)
    assert radix_cut(prob, 0.29) == np.float32(0.3)        # only the arg-max
    flat = np.full(100000, np.float32(1e-5))               # all equal: kept or dropped together -> all kept
    assert radix_cut(flat, 0.5) == np.float32(1e-5)
    tiny = np.zeros(60000, np.float32)                      # masses below 2^-56 still make their bin non-empty
    tiny[[3, 9]] = [np.float32(1.0), np.float32(1e-30)]
    assert radix_cut(tiny, 0.5) == np.float32(1.0) and radix_cut(tiny, 1.0) == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box WITHOUT a GPU (the launch must not run)")
def test_large_vocabularies_reach_the_launch():
    import llama2_accessory_b200 as pkg
    from llama2_accessory_b200 import _cabi
    pkg.build()
    lib = _cabi.lib()
    buf = torch.zeros(16, dtype=torch.int64)
    p = buf.data_ptr()
    # rc > 0: every host-side check passed and the call reached the CUDA runtime (no driver here); rc < 0 = refused
    for V in (32000, 57856, 57857, 103168, 256000):
        for T in (1, 32):
            rc = lib.b200_sample_top_p(p, p, p, T, V, 0.8, 0.95, None)
            assert rc > 0, (V, T, rc, lib.b200_last_error().decode())
    assert lib.b200_sample_top_p(p, p, p, 1, 103168, 0.0, 0.9, None) < 0   # temperature 0 is b200_argmax
    assert lib.b200_sample_top_p(p, p, p, 1, 103168, 1.0, 0.0, None) < 0   # top_p 0
