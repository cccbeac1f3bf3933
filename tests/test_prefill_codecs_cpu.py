"""CPU (no GPU present): the tensor-core prompt GEMM (csrc/prefill.cu) over its three weight codecs -- per-channel W4, W3
(80-k blocks) and fp16 linears.

  - k order: a numpy restatement of what the activation loaders store (logical k of a B stage <- physical k of x) and of
    what the consumers read from the packed stage (fragment position (row, logical k) <- packed field), run over the real
    packer's output of weights whose every (n, k) is distinguishable: each fragment position must meet the activation of
    its own physical k, every k < K exactly once, and the padded tail of a partial W3 block must meet zero activations;
  - the library's host checks of b200_prefill_gemm_w4 for every codec;
  - 7B W3 / fp16 and a 70B W3 TP = 8 rank at prompt 300 through forward_inference: every launch passes the real library's
    host checks, and the linears reach b200_prefill_gemm_w4 in layer order, 256 + 44 tokens per linear.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import llama2_accessory_b200 as pkg
from llama2_accessory_b200 import _cabi, ops
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig
from llama2_accessory_b200.quant import random_packed

# ---------------------------------------------------------------------------------------------------- k order ---------
# one pipeline stage per codec: logical k width, 16-k steps, packed 16-k blocks of one tile (fp16)
STAGE_K = {4: 64, 3: 80, 16: 64}
W3_BASE = [0, 3, 1, 4, 2]  # pack.cpp kW3Base: field of pair j


def _loader_map(bits, K):
    """[KB, kK] physical k of x the loaders store at logical k of stage kb (-1: zero activation), as prefill.cu's loader
    branches compute it.  Logical chunk c of a stage = logical k 8c .. 8c+7, its u32 word u = logical k 8c + 2u, +1."""
    kK = STAGE_K[bits]
    KB = -(-K // kK)
    m = np.full((KB, kK), -2, dtype=np.int64)

    def put(kb, chunk, word, phys_word, zero):  # phys_word: u32 index in the stage's x range (2 halves each)
        for e in range(2):
            assert m[kb, 8 * chunk + 2 * word + e] == -2, "logical k written twice"
            m[kb, 8 * chunk + 2 * word + e] = -1 if zero else kb * kK + 2 * phys_word + e
    for kb in range(KB):
        for h in range(2):
            if bits == 4:      # v[u] = uint4 h + 2u of the block; chunk 2 comp + h word u = component comp of v[u]
                for comp in range(4):
                    for u in range(4):
                        put(kb, 2 * comp + h, u, 4 * (h + 2 * u) + comp, False)
            elif bits == 16:   # blocks j = 2h, 2h+1: chunk 2j = (lo.x, lo.z, hi.x, hi.z), chunk 2j+1 = (lo.y, lo.w, hi.y, hi.w)
                for jj in range(2):
                    j = 2 * h + jj
                    for hh in range(2):
                        for u, word in enumerate((hh, 2 + hh, 4 + hh, 6 + hh)):
                            put(kb, 2 * j + hh, u, 8 * j + word, False)
            else:              # words 20h .. 20h+19; chunk (j, hh) bytes 8h .. 8h+7 = (w[5hh + j], w[10 + 5hh + j])
                for j in range(5):
                    for hh in range(2):
                        for u, i in enumerate((5 * hh + j, 10 + 5 * hh + j)):
                            phys = 20 * h + i  # in uint4 phys // 4, zero-filled when its first k is >= K
                            put(kb, 2 * j + hh, 2 * h + u, phys, kb * kK + 8 * (phys // 4) >= K)
    assert (m != -2).all()
    return m


def _fragment_map(bits, packed, N, K):
    """[N, KB * kK] field value the consumers put at fragment position (row, logical k): warp w = tile, lane (g, t),
    register r (row g + 8 (r & 1), k half r >> 1), k-step j, element e <-> logical k 16j + 8 (r >> 1) + 2t + e."""
    kK = STAGE_K[bits]
    KB = -(-K // kK)
    out = np.zeros((N, KB * kK), dtype=np.int64)
    g, t = np.meshgrid(np.arange(8), np.arange(4), indexing="ij")
    lane = (4 * g + t).ravel()
    g, t = g.ravel(), t.ravel()
    for tile in range(N // 16):
        for kb in range(KB):
            for j in range(kK // 16):
                for r in range(4):
                    row = 16 * tile + g + 8 * (r & 1)
                    for e in range(2):
                        lk = kb * kK + 16 * j + 8 * (r >> 1) + 2 * t + e
                        if bits == 16:  # the lane's uint4 of 16-k block 4 kb + j, u32 r, half e
                            half = ((((tile * (K // 16) + 4 * kb + j) * 32 + lane) * 4 + r) * 2 + e)
                            out[row, lk] = packed.view(np.uint16)[half]
                        else:
                            w = packed.view(np.uint32)[((tile * KB + kb) * 32 + lane) * 4 + r].astype(np.int64)
                            if bits == 4:  # deq_pair<J>: pair shift (j & 1) 8 + (j >> 1) 4, odd element 16 higher
                                out[row, lk] = (w >> ((j & 1) * 8 + (j >> 1) * 4 + 16 * e)) & 15
                            else:          # deq_pair_w3<J>: field 3 kW3Base[j], odd element 16 higher
                                out[row, lk] = (w >> (3 * W3_BASE[j] + 16 * e)) & 7
    return out


def _pack(bits, plane):
    lib = _cabi.lib()
    N, K = plane.shape
    if bits == 16:
        src = np.ascontiguousarray(plane.astype(np.uint16))
        out = np.zeros(N * K * 2, dtype=np.uint8)
        assert lib.b200_pack_f16(N, K, src.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)) == 0
    else:
        src = np.ascontiguousarray(plane.astype(np.uint8))
        out = np.zeros(lib.b200_packed_weight_bytes(bits, N, K), dtype=np.uint8)
        assert lib.b200_pack_weight(bits, N, K, src.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)) == 0
    return out


@pytest.mark.parametrize("bits,K", [(4, 512), (3, 1040), (3, 1024), (3, 4096), (3, 336), (16, 512), (16, 4096)])
def test_fragment_positions_meet_their_own_activations(bits, K):
    """Index n K + k written in base-2^bits digit planes, each plane packed by the real packer and read back through the
    consumer model: the fragment at (row, logical k) must hold index row K + p, p = the physical k the loaders put at that
    logical k; every k < K is stored once; logical k of the padded tail (p >= K) get zero activations."""
    pkg.build()
    N = 32  # two tiles: the tile-major stride between them is part of the address
    idx = np.arange(N * K, dtype=np.int64).reshape(N, K)
    base = 1 << min(bits, 16)
    n_dig = int(np.ceil(np.log(N * K) / np.log(base))) + 1
    frag = np.zeros((N, -(-K // STAGE_K[bits]) * STAGE_K[bits]), dtype=np.int64)
    for d in range(n_dig):
        plane = (idx // base ** d) % base
        frag += _fragment_map(bits, _pack(bits, plane), N, K) * base ** d
    lmap = _loader_map(bits, K).ravel()
    live = lmap >= 0
    phys = lmap[live]
    assert np.array_equal(np.sort(phys), np.arange(K)), "every physical k < K exactly once"
    rows = np.arange(N)[:, None]
    assert np.array_equal(frag[:, live], rows * K + phys[None, :])
    tail = ~live
    assert tail.sum() == frag.shape[1] - K
    if bits == 3 and K % 80:
        assert tail.sum() > 0 and (frag[:, tail] == 0).all()  # q = 0 padding of the packer meets zero activations


# ------------------------------------------------------------------------------------------------ host checks ---------
_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box WITHOUT a GPU (the launches must not run)")


@_no_gpu
def test_prefill_gemm_host_checks_per_codec():
    """rc > 0: the call passed every host-side check and reached its first CUDA runtime call (no driver here);
    rc < 0 with a prefill_gemm_w4: message: refused."""
    pkg.build()
    lib = _cabi.lib()
    x = torch.zeros(16, 8192, dtype=torch.float16)
    out = torch.zeros(16, 8192, dtype=torch.float16)

    def call(pl, **kw):
        ls = pl.c_struct()
        for k, v in kw.items():
            setattr(ls, k, v)
        rc = lib.b200_prefill_gemm_w4(C.byref(ls), x.data_ptr(), out.data_ptr(), 16, None)
        return rc, lib.b200_last_error().decode()

    good = [random_packed(4, 256, 512, 0, "cpu", 0), random_packed(3, 256, 1040, 0, "cpu", 0),
            random_packed(3, 1280, 4096, 0, "cpu", 0), random_packed(3, 8192, 3584, 0, "cpu", 0),
            random_packed(16, 256, 512, 0, "cpu", 0), random_packed(16, 384, 4096, 0, "cpu", 0)]
    for pl in good:
        rc, msg = call(pl)
        assert rc > 0, (pl.bits, pl.N, pl.K, rc, msg)
    w4g = random_packed(4, 256, 512, 128, "cpu", 0)
    w3 = random_packed(3, 256, 1040, 0, "cpu", 0)
    w2 = random_packed(2, 256, 512, 0, "cpu", 0)
    f16 = random_packed(16, 256, 512, 0, "cpu", 0)
    bad = [call(w4g),                                   # grouped W4
           call(w3, group_size=80),                     # grouped scales on the 3-bit codec
           call(f16, group_size=128),                   # grouped fp16: no such codec
           call(w2),                                    # native W2
           call(w3, K=1000), call(w3, N=192),           # W3: K % 16 != 0, N % 128 != 0
           call(f16, K=528), call(f16, N=144),          # fp16: K % 64 != 0, N % 128 != 0
           call(w3, scales=None),                       # W3 without scales
           call(f16, bits=8)]                           # a width the GEMM has no codec for
    for rc, msg in bad:
        assert rc < 0 and msg.startswith("prefill_gemm_w4:"), (rc, msg)


# ----------------------------------------------------------------------------------- launches of the engine ---------
LAUNCHES = ("b200_gemv", "b200_attn_decode", "b200_embed", "b200_prefill_gemm_w4", "b200_prefill_rmsnorm",
            "b200_prefill_rope_kv", "b200_prefill_silu_mul", "b200_argmax", "b200_advance_pos")
L7 = dict(dim=4096, n_heads=32, vocab_size=32000, multiple_of=256)
L70 = dict(dim=8192, n_heads=64, n_kv_heads=8, vocab_size=32000, multiple_of=4096, ffn_dim_multiplier=1.3)


class Validator:
    """Calls the real entry point; rc < 0 is a rejection, rc > 0 (no driver) an acceptance.  Records the linear and token
    count of every prompt GEMM."""

    def __init__(self, real):
        self.real, self.rejected, self.accepted, self.gemms = real, [], {}, []

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        if name not in LAUNCHES:
            return fn

        def call(*args):
            if name == "b200_prefill_gemm_w4":
                ls = args[0]._obj
                self.gemms.append((ls.bits, ls.N, ls.K, ls.group_size, ls.qweight, args[3]))
            rc = fn(*args)
            if rc < 0:
                self.rejected.append((name, rc, self.real.b200_last_error().decode()))
            else:
                self.accepted[name] = self.accepted.get(name, 0) + 1
            return 0
        return call


@pytest.fixture()
def validator(monkeypatch):
    pkg.build()
    v = Validator(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", v)
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0))
    monkeypatch.setattr(ops, "_f16", lambda t, name: None)
    monkeypatch.setattr(torch.distributed, "all_gather", lambda parts, t, group=None: [p.copy_(t) for p in parts])
    monkeypatch.setattr(torch.distributed, "all_reduce", lambda t, group=None, op=None: None)
    return v


@_no_gpu
@pytest.mark.parametrize("margs,bits,tp", [(L7, 3, 1), (L7, 16, 1), (L70, 3, 8)], ids=["7B_W3", "7B_fp16", "70B_W3_tp8"])
def test_w3_and_fp16_prompts_take_the_tensor_core_gemm(validator, margs, bits, tp):
    prompt = 300
    args = dict(margs, n_layers=1, max_seq_len=prompt + 32, max_batch_size=1)
    rank = tp - 1
    eng = DecodeEngine(EngineConfig.from_model_args("llama", args, bits=bits, group_size=0, tp_rank=rank, tp_world=tp), "cpu")
    eng.load_random(seed=0)
    eng.use_graph = False
    if tp > 1:
        base = 0x7000_0000_0000
        eng._peer_buffers = lambda nbytes: (base + rank * 0x1000_0000, [base + r * 0x1000_0000 for r in range(tp)])
    assert eng.prefill_tc_supported()
    toks = torch.randint(1, args["vocab_size"], (1, prompt + 2), generator=torch.Generator().manual_seed(1))
    eng.forward_inference(toks[:, :prompt], 0)
    for j in range(2):
        eng.forward_inference(toks[:, prompt + j:prompt + j + 1], prompt + j)
    assert not validator.rejected, validator.rejected[:4]
    lw = eng.layers[0]
    lins = (lw.wqkv, lw.wo, lw.w13, lw.w2)
    want = [(pl.bits, pl.N, pl.K, 0, pl.qweight.data_ptr(), T) for T in (256, prompt - 256) for pl in lins]
    assert validator.gemms == want
    assert all(g[0] == bits for g in validator.gemms)
    if bits == 3:
        assert any(g[2] % 80 for g in validator.gemms)  # a partial last 80-k block is among the real widths


@_no_gpu
def test_prefill_tc_rule_per_codec():
    """Dense LLaMA: per-channel W4 / W3 / fp16 take the tensor-core path, grouped codecs and W2 do not; B200_PREFILL_TC=0
    (use_prefill_tc False) turns it off for every codec."""
    pkg.build()
    args = dict(L7, n_layers=1, max_seq_len=64, max_batch_size=1)
    for bits, gs, want in [(4, 0, True), (3, 0, True), (16, 0, True), (4, 128, False), (3, 128, False), (2, 64, False),
                           (2, 0, False)]:
        eng = DecodeEngine(EngineConfig.from_model_args("llama", args, bits=bits, group_size=gs), "cpu")
        eng.load_random(seed=0)
        assert eng.prefill_tc_supported() == want, (bits, gs)
        eng.use_prefill_tc = False
        assert not eng.prefill_tc_supported()
