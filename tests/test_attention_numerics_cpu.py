"""CPU restatement of the arithmetic of the split-KV decode attention kernel (csrc/attn.cu) -- what is rounded where -- checked
against an exact softmax attention and against the reference's own fp16 SDPA call (llama.py:191-206).

    scores      fp16 q . fp16 k accumulated in fp32 (HMMA), times log2(e) / sqrt(128)         attn.cu "S = Q K^T", scale_log2
    split       the kv range [0, pos] is cut into n_split chunks (multiples of the 32-position tile)
    warp        inside a split, tile i belongs to consumer warp i % 4; a warp folds ITS tiles in order with the online rule
                m' = max(m, max_tile), corr = 2^(m - m'), l = l * corr + sum(fp16(p)), O = O * corr + fp16(p) V  (fp32)
                with p = 2^(s - m'): P is rounded to fp16 for the second MMA and the row sum uses the ROUNDED values, so the
                result stays a convex combination of V rows (no normalisation bias)
    merge       4 warps, then the splits in split order: M = max m, f = 2^(m - M), L = sum l f, o = sum O f; out = fp16(o / L)

No GPU: this pins the numerics MODEL (DESIGN.md section 2, oracle.numerics.attn_kernel_model); the kernel itself is
compared with float64 and with this model by tests/test_attn_decode_gpu.py.
"""
import math

import pytest
import torch

from oracle.numerics import ATTN_TILE as TILE
from oracle.numerics import attn_host_split, attn_kernel_model as kernel_model, attn_split_ranges


@pytest.mark.parametrize("even", [0, 1])
@pytest.mark.parametrize("max_kv_len", [1, 31, 32, 33, 200, 2048, 2400, 4096, 32768])
def test_both_split_schedules_cut_every_context_into_whole_tiles_once(max_kv_len, even):
    """Every kv length up to the launch's max_kv_len, every requested split count: the non-empty splits are consecutive,
    cover [0, kv_len) once, begin on a tile, and none exceeds the launch's chunk; the even schedule's tile counts differ by
    at most one."""
    for req in sorted({1, 2, 3, 7, 16, 17, 33, max(1, max_kv_len // 32), max_kv_len // 32 + 5}):
        ns, chunk = attn_host_split(max_kv_len, req)
        assert ns <= req and chunk % TILE == 0 and (ns - 1) * chunk < max_kv_len <= ns * chunk
        for kv_len in sorted({1, 2, 31, 32, 33, max_kv_len // 2 + 1, max_kv_len - 1, max_kv_len} - {0}):
            if kv_len > max_kv_len:
                continue
            r = [(b, e) for b, e in attn_split_ranges(kv_len, ns, chunk, even) if e > b]
            assert r[0][0] == 0 and r[-1][1] == kv_len and all(r[i][1] == r[i + 1][0] for i in range(len(r) - 1))
            assert all(b % TILE == 0 and e - b <= chunk for b, e in r), (req, kv_len, r)
            if even:
                nt = [-(-(e - b) // TILE) for b, e in attn_split_ranges(kv_len, ns, chunk, even)]
                assert max(nt) - min(nt) <= 1, (req, kv_len, nt)


def exact(q, k, v):
    s = (k.double() @ q.double()) / math.sqrt(128.0)
    return torch.softmax(s, 0) @ v.double()


@pytest.mark.parametrize("n,n_split", [(1, 1), (31, 1), (33, 1), (200, 1), (200, 3), (2048, 1), (2048, 16), (2049, 7)])
def test_kernel_arithmetic_model_is_within_half_precision_of_exact_attention(n, n_split):
    g = torch.Generator().manual_seed(n * 31 + n_split)
    q = torch.randn(128, generator=g).half()
    k = torch.randn(n, 128, generator=g).half()
    v = (torch.randn(n, 128, generator=g) * 0.5).half()
    got = kernel_model(q, k, v, n_split).double()
    ref = exact(q, k, v)
    # output rounding (half an fp16 ulp of the value) + the fp16 rounding of P (relative 2^-11 per weight, averaged out)
    tol = 2.0 ** -11 * ref.abs().clamp(min=2.0 ** -6) + 2.0 ** -11 * float(v.float().abs().max())
    assert ((got - ref).abs() <= tol).all(), float((got - ref).abs().max())


@pytest.mark.parametrize("n,n_split,max_kv_len", [(33, 16, 4096), (200, 3, 200), (2048, 16, 2048), (2049, 7, 4096)])
def test_even_schedule_model_is_within_half_precision_of_exact_attention(n, n_split, max_kv_len):
    """B200_ATTN_EVEN = 1 and a grid sized for a longer context than the keys present (the captured-graph case)."""
    g = torch.Generator().manual_seed(n * 17 + n_split)
    q = torch.randn(128, generator=g).half()
    k = torch.randn(n, 128, generator=g).half()
    v = (torch.randn(n, 128, generator=g) * 0.5).half()
    ref = exact(q, k, v)
    tol = 2.0 ** -11 * ref.abs().clamp(min=2.0 ** -6) + 2.0 ** -11 * float(v.float().abs().max())
    for even in (False, True):
        got = kernel_model(q, k, v, n_split, even=even, max_kv_len=max_kv_len).double()
        assert ((got - ref).abs() <= tol).all(), (even, float((got - ref).abs().max()))


def test_split_count_moves_the_result_by_at_most_one_output_rounding_step():
    """P = 2^(s - m) is rounded to fp16 relative to the running maximum of the warp that folds the tile, so the split / warp
    structure changes WHICH roundings happen (not their size): outputs of different split counts differ by at most one fp16
    step -- the reason the persistent kernels (another split structure) are not bit-identical to the separate kernels in
    the attention output, and only there."""
    g = torch.Generator().manual_seed(5)
    q = torch.randn(128, generator=g).half()
    k = torch.randn(1500, 128, generator=g).half()
    v = torch.randn(1500, 128, generator=g).half()
    outs = [kernel_model(q, k, v, ns) for ns in (1, 2, 5, 12)]
    ref = exact(q, k, v)
    for o in outs:
        # each one is within its own output rounding + the averaged P rounding of the exact result ...
        assert float((o.double() - ref).abs().max()) <= 2.0 ** -11 * float(ref.abs().max()) + 2.0 ** -13 * float(v.float().abs().max())
    for o in outs[1:]:
        # ... and any two differ by at most one fp16 step at the magnitude of the largest output
        assert float((o.float() - outs[0].float()).abs().max()) <= 2.0 ** -10 * float(outs[0].float().abs().max())


def test_model_against_the_reference_sdpa_in_fp16_and_fp32():
    """llama.py:191-206 on the CPU: F.scaled_dot_product_attention over the cached rows; the kernel model must be as close
    to the fp32 result as that fp16 call is (both round the output to fp16; the reference also rounds the scores)."""
    g = torch.Generator().manual_seed(11)
    n = 777
    q = torch.randn(128, generator=g).half()
    k = torch.randn(n, 128, generator=g).half()
    v = torch.randn(n, 128, generator=g).half()
    ref32 = exact(q, k, v)
    sdpa16 = torch.nn.functional.scaled_dot_product_attention(q.view(1, 1, 1, 128), k.view(1, 1, n, 128), v.view(1, 1, n, 128))
    ours = kernel_model(q, k, v, 4)
    e_ref = float((sdpa16.view(128).double() - ref32).abs().max())
    e_ours = float((ours.double() - ref32).abs().max())
    assert e_ours <= max(e_ref, 2.0 ** -11 * float(ref32.abs().max())) * 1.5, (e_ours, e_ref)
