"""CPU: the C-ABI library loads, exports every declared symbol, and the packer's layouts are exactly
what the kernels' codecs (csrc/gemv.cu Codec<BITS>::block) consume.

The codec emulation below restates, in numpy, the register-level extraction of gemv.cu (masks, shifts,
which x pairs feed which HMMA) -- no GPU needed to pin the index math of packer <-> kernel.
"""
import ctypes as C
import re
import os

import numpy as np
import pytest
import torch

import llama2_accessory_b200 as pkg
from llama2_accessory_b200 import _cabi, quant

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "b200_decode.h")).read()
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", hdr))
    declared -= {n for n in declared if n.endswith("_t")}
    lib = C.CDLL(_cabi.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in b200_decode.h but not exported"
    assert declared == set(_cabi.SYMBOLS), declared ^ set(_cabi.SYMBOLS)
    assert _cabi.lib().b200_version() >= 100
    # INTEGRATION.md's entry-point index (what a maintainer binds, with the reference interface each stands in for) lists
    # exactly the declared symbols
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    index = doc[doc.index("## Entry-point index"):doc.index("## Round-2 entry points")]
    assert set(re.findall(r"`(b200_[a-z0-9_]+)`", index)) == declared


def test_missing_library_fails_loudly(monkeypatch):
    monkeypatch.setattr(_cabi, "_lib", None)
    monkeypatch.setattr(_cabi, "LIB_PATH", "/nonexistent/libb200decode.so")
    with pytest.raises(RuntimeError, match="no CPU or PyTorch fallback"):
        _cabi.lib()


@pytest.mark.parametrize("bits,N,K", [(4, 32, 128), (4, 48, 704), (2, 32, 256), (3, 32, 256), (3, 16, 512)])
def test_pack_roundtrip(bits, N, K):
    g = torch.Generator().manual_seed(bits * 1000 + K)
    q = torch.randint(0, 2 ** bits, (N, K), generator=g, dtype=torch.uint8)
    s = torch.rand(N, 1, generator=g).half()
    z = torch.full((N, 1), 3.0).half()
    pl = quant.pack_quantized(q, s, z, bits, 0, "cpu")
    assert pl.qweight.numel() == _cabi.lib().b200_packed_weight_bytes(bits, N, K)
    assert torch.equal(quant.unpack_quantized(pl), q)


def test_pack_rejects_bad_input():
    lib = _cabi.lib()
    q = np.full((16, 64), 17, dtype=np.uint8)
    out = np.zeros(lib.b200_packed_weight_bytes(4, 16, 64), dtype=np.uint8)
    assert lib.b200_pack_weight(4, 16, 64, q.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)) < 0
    assert b"out of range" in lib.b200_last_error()
    assert lib.b200_pack_weight(4, 15, 64, q.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)) < 0


@pytest.mark.parametrize("zbad", [7.5, -0.5, 1025.0, -1025.0, 2048.0, float("nan"), float("inf")])
def test_pack_rejects_zero_points_outside_the_format(zbad):
    """The prompt GEMM dequantises (1024 + q) - (1024 + z) in fp16: exact only for integer z with |z| <= 1024."""
    q = torch.zeros(16, 64, dtype=torch.uint8)
    s = torch.full((16, 1), 1e-3).half()
    z = torch.full((16, 1), 8.0).half()
    for zok in (-1024.0, -1023.0, 0.0, 1000.0, 1024.0):  # the edges of the format still pack
        z[5, 0] = zok
        quant.pack_quantized(q, s, z, 4, 0, "cpu")
    z[5, 0] = zbad
    with pytest.raises(ValueError, match="zero points"):
        quant.pack_quantized(q, s, z, 4, 0, "cpu")
    zg = torch.full((16, 2), 8.0).half()  # grouped scales are checked the same way
    zg[15, 1] = zbad
    with pytest.raises(ValueError, match="zero points"):
        quant.pack_quantized(q, s.expand(16, 2).contiguous(), zg, 4, 32, "cpu")


# ---- numpy restatement of Codec<BITS>::block -------------------------------------------------------
def _halves(reg):
    return (reg & 0xFFFF).astype(np.float64), (reg >> 16).astype(np.float64)


def _mma(acc, tile, g, a, b):
    """a: 4 regs (row g k-lo, row g+8 k-lo, row g k-hi, row g+8 k-hi); b: 2 x-pairs. fields are raw integers."""
    for (ra, rb, xp) in ((a[0], a[1], b[0]), (a[2], a[3], b[1])):
        lo0, hi0 = _halves(np.uint32(ra))
        lo1, hi1 = _halves(np.uint32(rb))
        acc[tile * 16 + g] += lo0 * xp[0] + hi0 * xp[1]
        acc[tile * 16 + g + 8] += lo1 * xp[0] + hi1 * xp[1]


def emulate(bits, words, N, K, x):
    """words: uint32 [tiles, KB, 32, 4]; returns sum_k q[n,k] x[k] exactly as the kernel accumulates it."""
    tiles, KB = words.shape[:2]
    kblk = {4: 64, 2: 128, 3: 80}[bits]
    xp = np.zeros(KB * kblk + 64)
    xp[:K] = x
    acc = np.zeros(N)
    for tile in range(tiles):
        for blk in range(KB):
            for lane in range(32):
                g, t = lane >> 2, lane & 3
                w = [int(v) for v in words[tile, blk, lane]]
                if bits == 4:
                    base = blk * 64 + t * 16
                    pr = lambda o: (xp[base + o], xp[base + o + 1])  # noqa: E731
                    ML, MH = 0x000F000F, 0x00F000F0
                    for (u0, u1, off) in ((w[0], w[1], 0), (w[2], w[3], 8)):
                        s0, s1 = u0 >> 8, u1 >> 8
                        lo = np.zeros(N)
                        hi = np.zeros(N)
                        _mma(lo, tile, g, [u0 & ML, u1 & ML, s0 & ML, s1 & ML], [pr(off), pr(off + 2)])
                        _mma(hi, tile, g, [u0 & MH, u1 & MH, s0 & MH, s1 & MH], [pr(off + 4), pr(off + 6)])
                        acc += lo + hi / 16.0
                elif bits == 2:
                    base = blk * 128 + t * 32
                    pr = lambda o: (xp[base + o], xp[base + o + 1])  # noqa: E731
                    M = [0x00030003 << (2 * c) for c in range(5)]
                    cls = [np.zeros(N) for _ in range(5)]
                    for (u0, u1, off) in ((w[0], w[1], 0), (w[2], w[3], 16)):
                        s0, s1 = u0 >> 10, u1 >> 10
                        _mma(cls[0], tile, g, [u0 & M[0], u1 & M[0], s0 & M[0], s1 & M[0]], [pr(off), pr(off + 2)])
                        _mma(cls[1], tile, g, [u0 & M[1], u1 & M[1], s0 & M[1], s1 & M[1]], [pr(off + 4), pr(off + 6)])
                        _mma(cls[2], tile, g, [u0 & M[2], u1 & M[2], s0 & M[2], s1 & M[2]], [pr(off + 8), pr(off + 10)])
                    _mma(cls[3], tile, g, [w[0] & M[3], w[1] & M[3], w[2] & M[3], w[3] & M[3]], [pr(12), pr(28)])
                    _mma(cls[4], tile, g, [w[0] & M[4], w[1] & M[4], w[2] & M[4], w[3] & M[4]], [pr(14), pr(30)])
                    acc += sum(cls[c] / (4.0 ** c) for c in range(5))
                else:
                    base = blk * 80 + t * 20
                    pr = lambda o: (xp[base + o], xp[base + o + 1])  # noqa: E731
                    M0, M1, M2 = 0x00070007, 0x00380038, 0x01C001C0
                    cls = [np.zeros(N) for _ in range(3)]
                    s = [v >> 9 for v in w]
                    _mma(cls[0], tile, g, [w[0] & M0, w[1] & M0, s[0] & M0, s[1] & M0], [pr(0), pr(2)])
                    _mma(cls[1], tile, g, [w[0] & M1, w[1] & M1, s[0] & M1, s[1] & M1], [pr(4), pr(6)])
                    _mma(cls[0], tile, g, [w[2] & M0, w[3] & M0, s[2] & M0, s[3] & M0], [pr(10), pr(12)])
                    _mma(cls[1], tile, g, [w[2] & M1, w[3] & M1, s[2] & M1, s[3] & M1], [pr(14), pr(16)])
                    _mma(cls[2], tile, g, [w[0] & M2, w[1] & M2, w[2] & M2, w[3] & M2], [pr(8), pr(18)])
                    acc += cls[0] + cls[1] / 8.0 + cls[2] / 64.0
    return acc


@pytest.mark.parametrize("bits,N,K", [(4, 32, 192), (2, 32, 256), (3, 32, 192), (3, 16, 320)])
def test_codec_emulation_matches_plain_dot(bits, N, K):
    g = torch.Generator().manual_seed(11 + bits)
    q = torch.randint(0, 2 ** bits, (N, K), generator=g, dtype=torch.uint8)
    x = torch.randn(K, generator=g).double().numpy()
    pl = quant.pack_quantized(q, torch.ones(N, 1).half(), torch.zeros(N, 1).half(), bits, 0, "cpu")
    kblk = {4: 64, 2: 128, 3: 80}[bits]
    KB = (K + kblk - 1) // kblk
    words = pl.qweight.numpy().view(np.uint32).reshape(N // 16, KB, 32, 4)
    got = emulate(bits, words, N, K, x)
    ref = q.double().numpy() @ x
    assert np.allclose(got, ref, rtol=0, atol=1e-9), np.abs(got - ref).max()


def test_fp16_pack_is_hmma_a_fragment():
    N, K = 32, 64
    w = torch.randn(N, K).half()
    pl = quant.pack_fp16(w, "cpu")
    h = pl.qweight.numpy().view(np.float16).reshape(N // 16, K // 16, 32, 4, 2)
    for tile, blk, lane in ((0, 0, 0), (1, 3, 13), (0, 2, 31)):
        g, t = lane >> 2, lane & 3
        k0 = blk * 16 + 4 * t
        r0, r1 = tile * 16 + g, tile * 16 + g + 8
        exp = [[w[r0, k0], w[r0, k0 + 1]], [w[r1, k0], w[r1, k0 + 1]], [w[r0, k0 + 2], w[r0, k0 + 3]],
               [w[r1, k0 + 2], w[r1, k0 + 3]]]
        assert np.array_equal(h[tile, blk, lane], np.array(exp, dtype=np.float16))


def test_scale_layouts():
    N, K = 32, 256
    s = (torch.arange(N * 2).reshape(N, 2) / 64 + 0.01).half()
    z = (torch.arange(N * 2).reshape(N, 2) % 7).half()
    q = torch.zeros(N, K, dtype=torch.uint8)
    pl = quant.pack_quantized(q, s, z, 4, 128, "cpu")
    sz = pl.scales.numpy().view(np.float16).reshape(N // 16, 2, 16, 2)
    assert sz[1, 1, 5, 0] == s[21, 1] and sz[1, 1, 5, 1] == z[21, 1]
    pc = quant.pack_quantized(q, s[:, :1].contiguous(), z[:, :1].contiguous(), 4, 0, "cpu")
    szc = pc.scales.numpy().view(np.float16).reshape(N, 2)
    assert szc[21, 0] == s[21, 0] and szc[21, 1] == z[21, 0]


def test_product_quantiser_equals_oracle_restatement():
    from oracle import omniquant
    g = torch.Generator().manual_seed(5)
    w = ((torch.rand(32, 512, generator=g) * 2 - 1) / 20).half()
    for bits, gs in ((4, 0), (4, 128), (3, 0), (2, 128)):
        q, s, z, gg = quant.quantize_weight(w, bits, gs)
        r = omniquant.quantize_weight(w, bits, gs)
        assert torch.equal(q, r["q"]) and torch.equal(s, r["scale"]) and torch.equal(z, r["zero"])
        assert torch.equal(quant.dequantize(q, s, z, gg), r["w_hat"])


def test_container_fallbacks():
    assert quant.container_bits(3, 128, 512) == 4
    assert quant.container_bits(3, 0, 512) == 3
    assert quant.container_bits(2, 64, 512) == 4
    assert quant.container_bits(2, 128, 512) == 2
    assert quant.container_bits(4, 64, 512) == 4


def test_tuning_knob_table_accepts_and_rejects():
    """b200_tune: host-side override table of the launchers' knobs (no device work): set, overwrite, reject bad names."""
    import ctypes as C
    lib = _cabi.lib()
    assert lib.b200_tune(b"B200_TEST_KNOB", 3) == 0
    assert lib.b200_tune(b"B200_TEST_KNOB", 0) == 0          # overwrite, not a second entry
    assert lib.b200_tune(b"X" * 64, 1) != 0                  # name too long for the table
    assert lib.b200_tune(None, 1) != 0
    assert lib.b200_timeline_cta(None, 0, 0, 0) == 0         # off: nothing to validate
