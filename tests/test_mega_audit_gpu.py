"""GPU: the persistent whole-step decode kernels (csrc/mega1.cu grid barriers, csrc/mega2.cu LL dataflow) phase by phase
against float64, at the widths of one real tensor-parallel rank launched at tp_world = 1.

Shapes (D, Hq / Hkv, F, V): 7B, 13B and a GQA model with n_rep 4 are built as `DecodeEngine`s and launched through
`_step1_args`; one rank of 70B at TP = 8 (n_rep 8, one kv head) and the widest shape the host check admits (D 8192,
F 16384, 128 query heads) are not engine shapes (dim / n_heads != 128), so the test fills `Step1Args` itself and chains the
separate kernels with the engine's launch arguments.

1. One-layer audit.  With one layer every phase's input and output is still readable after the launch: mega1 keeps h0, q,
   the per-split attention partials in attn_ws, the wo / w2 fp16 partials in the communication block, h1, act and the
   logits; mega2 keeps the LL vectors yq, ykv, att, po, act, pf (each unit must carry this launch's sequence number) and
   the logits.  Each phase is checked against float64 of its own inputs:
     * RMSNorm (QKV, W13, head).  mega1 stages x through gemv1's prologue; mega2's `stage_norm` does the same per lane: two
       8-element pieces chained with fmaf (<= 16 terms), the 5-level warp tree, then the 16 warp partials in warp order:
       depth <= 37, so ssq lies within 37u of sum h^2 (u = 2^-24); the division by D and the eps add round once each (2u),
       sqrtf halves the relative error and rounds (0.5u), the reciprocal rounds (0.5u): rstd lies within 21u of rstd64,
       inside the window of RSTD_ULPS = 32 fp32 ulps that `x_candidates` enumerates (test_decode_path_gpu.py derives the
       same window for gemv1 and, at depth <= 53, for the fp16 head's prologue, which both kernels run unchanged).
     * GEMVs: exact integer dots, so 2^-20 max|y| of fp32 recombination noise plus the fp16 rounding of the output.
     * Epilogues: q, the K / V cache rows and mega2's LL copies are the RoPE / identity of the fp16 y that the separate
       gemv1 F16 launch computes from the same input (`qkv_from_y`), bit for bit; act is fp16(silu(a)) * b of the w13 y,
       bit for bit except where the fp32 silu lies within SILU_REL of an fp16 midpoint.
     * Attention: every split's O / l against float64 attention over that split's key range, with the bound of
       oracle.numerics.AttnRef for this kernel's tile assignment: tile i of an item is folded by warp i % 16 (online
       rescale chain of ceil(tiles / 16) steps), then 16 warp partials are merged, so tpw = ceil(tiles / 16) and 16 merged
       partials; m against the float64 maximum score of the split within the score error; an empty split is (0, -inf, 0).
       The float64 merge of the kernel's partials must also meet the bound against float64 attention over all keys
       (16 + n_split merged partials).
     * wo: against float64 of that merge, rounded to fp16; an element whose merge lies within 2^-20 of the magnitude sum
       (fp32 merge over <= 8 splits, exp2f) of an fp16 midpoint may take either rounding.
     * Residual adds: h1 = h0 + wo and the head's h = h1 + w2 are fp16 adds, bit for bit.
     * Head: the fp16 HMMA GEMV bound C_ACC16 relative to |x| . |w|, over the rstd window.
   Positions 0, 31, 32, 2047, cache_seq - 1 (where every warp folds >= 2 tiles), and kv_len one key past a split boundary;
   mega1 also at n_split 1, 3 and 8.  The cache holds noise below pos, the NaN sentinel in row pos and in every later
   tile, zeros after pos inside pos's tile; every scratch element outside the outputs holds the sentinel.  After the
   launch nothing but row pos of the cache and the phase outputs has changed, and no output holds a NaN.
2. Bit identity where attention cannot differ: at pos 0 the attention output is v for any split structure, so mega1,
   mega2 and the separate kernels must give the same logits and the same K / V row of every layer, for 1, 2 and 32 layers
   at 7B and 96 layers at D 1024; repeated launches and CUDA-graph replays too.
3. Two layers at pos 2047 and at cache_seq - 1: mega1 and mega2 against the separate kernels on the same cache.  Layer 0's
   K / V rows are bit-identical, mega1 and mega2 are bit-identical to each other; layer 1's rows and the logits differ
   from the separate kernels through attention alone, within the tolerance stated at CHAIN_ULPS.
mega2's error word must read 0 after every launch.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import _cabi, kvlayout, ops, quant  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig, _interleave_w13, rope_table  # noqa: E402
from oracle import numerics as nx  # noqa: E402
from oracle.numerics import SENT, AttnRef, fp16_sides, nan16, x_candidates  # noqa: E402

DEV = "cuda"
EPS = 1e-5
C_ACC16 = 2.0 ** -18     # fp32 accumulation of the fp16 HMMA head, relative to |x| . |w|^T (test_decode_path_gpu.py)
MERGE_AMB = 2.0 ** -20   # fp32 cross-split merge (<= 8 terms, exp2f 2 ulp, one division) relative to sum |O| f / L
WS_SENT = 0x7FC05A5A     # fp32 NaN pattern of the attention workspace
LL_SENT32 = 0x7E5A7E5A   # 32-bit word of the LL areas: a sequence number no launch here reaches
TOK = 7

#               D     Hq  Hkv  F      V      engine  cache_seq
SHAPES = {"7b": (4096, 32, 32, 11008, 32000, True, 4096),
          "13b": (5120, 40, 40, 13824, 32000, True, 4096),
          "gqa_nrep4": (4096, 32, 8, 14336, 32000, True, 8192),
          "70b_tp8_rank": (8192, 8, 1, 3584, 4000, False, 8192),
          "widest": (8192, 128, 16, 16384, 4096, False, 8192)}


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _ulp16(v):
    near, alt, _ = fp16_sides(v)
    return (alt - near).abs()


def _split_of(Hkv):
    """mega2's ll_split and the engine's b200_step1_choose_split: one (kv head, split) item per SM, at most 8."""
    return max(1, min(8, torch.cuda.get_device_properties(0).multi_processor_count // Hkv))


# ------------------------------------------------------------------------------------------------ the model -----------
def _w4(N, K, seed, w13=False):
    """Random per-channel W4 (codes, scales ~ 2 / (15 sqrt K), zeros 0..15) -> (PackedLinear, float64 w_hat [N, K])."""
    g = _gen(seed)

    def one(n):
        q = torch.randint(0, 16, (n, K), generator=g, device=DEV, dtype=torch.uint8)
        s = ((0.75 + 0.5 * torch.rand(n, 1, generator=g, device=DEV)) * 2.0 / (15 * math.sqrt(K))).half()
        return q, s, torch.randint(0, 16, (n, 1), generator=g, device=DEV).half()
    if w13:
        (q1, s1, z1), (q3, s3, z3) = one(N // 2), one(N // 2)
        q, s, z = _interleave_w13(q1, q3), _interleave_w13(s1, s3), _interleave_w13(z1, z3)
    else:
        q, s, z = one(N)
    return quant.pack_quantized(q, s, z, 4, 0, DEV), (q.double() - z.double()) * s.double()


class Rig:
    """One model, its buffers and the three ways of running a decode step: mega1, mega2 and the separate kernels."""

    def __init__(self, name, n_layers, seed=0):
        D, Hq, Hkv, F, V, via_engine, S = SHAPES[name]
        self.name, self.L, self.D, self.Hq, self.Hkv, self.F, self.V, self.S = name, n_layers, D, Hq, Hkv, F, V, S
        self.nq, self.nkv = Hq * 128, Hkv * 128
        g = _gen(seed)
        self.tok_emb = ((torch.rand(V, D, generator=g, device=DEV) * 2 - 1) / math.sqrt(D)).half()
        wh = ((torch.rand(V, D, generator=g, device=DEV) * 2 - 1) / math.sqrt(D)).half()
        self.lm_head, self.Wh = quant.pack_fp16(wh, DEV), wh.double()
        del wh
        self.final_norm = (1 + 0.2 * torch.randn(D, generator=g, device=DEV)).half()
        self.layers = []
        for i in range(n_layers):
            s = seed + 100 * (i + 1)
            lw = dict(attn_norm=(1 + 0.2 * torch.randn(D, generator=g, device=DEV)).half(),
                      ffn_norm=(1 + 0.2 * torch.randn(D, generator=g, device=DEV)).half())
            for k, (N, K, w13) in dict(wqkv=(self.nq + 2 * self.nkv, D, False), wo=(D, self.nq, False),
                                       w13=(2 * F, D, True), w2=(D, F, False)).items():
                lw[k], lw["W" + k] = _w4(N, K, s, w13)
                s += 1
            self.layers.append(lw)
        self.eng = None
        if via_engine:
            cfg = EngineConfig(kind="llama", n_layers=n_layers, dim=D, n_heads=Hq, n_kv_heads=Hkv, ffn_hidden=F,
                               vocab_size=V, max_seq_len=S, bits=4, group_size=0)
            e = self.eng = DecodeEngine(cfg, DEV)
            e.use_graph = False
            e.tok_emb, e.final_norm, e.lm_head = self.tok_emb, self.final_norm, self.lm_head
            for lw, el in zip(self.layers, e.layers):
                for k in ("attn_norm", "ffn_norm", "wqkv", "wo", "w13", "w2"):
                    setattr(el, k, lw[k])
            e.allocate_kv_cache(1)
            assert e.cache_seq == S
            self.kc, self.vt, self.h, self.q, self.act = e.kcache, e.vtcache, e.h, e.q, e.act
            self.attn, self.o, self.f, self.tokens, self.pos, self.rope = e.attn, e.o, e.f, e.tokens, e.pos, e.rope
        else:
            z = lambda *s, dt=torch.float16: torch.zeros(*s, dtype=dt, device=DEV)  # noqa: E731
            self.kc = z(n_layers, 1, Hkv, S, 128)
            self.vt = z(n_layers, 1, Hkv, S // 32, 128, 32)
            self.h, self.q, self.act = [z(2, D), z(2, D)], z(2, self.nq), z(2, F)
            self.attn, self.o, self.f = z(2, self.nq), z(2, D), z(2, D)
            self.tokens, self.pos = z(2, dt=torch.int64), z(2, dt=torch.int32)
            self.rope = rope_table(128, 2 * S, 10000.0, None).to(DEV)
        self.logits = torch.zeros(1, V, device=DEV)
        lib = _cabi.lib()
        self.ws = torch.zeros(lib.b200_step1_attn_ws_bytes(Hq, 8), dtype=torch.uint8, device=DEV)
        self._own = {}
        self.tokens[0] = TOK

    # ---------------------------------------------------------------------------------------------- launches --------
    def _own_args(self, dataflow):
        """Step1Args at tp_world = 1, filled field by field as DecodeEngine._step1_args does."""
        if dataflow in self._own:
            return self._own[dataflow]
        lib, L, D = _cabi.lib(), self.L, self.D
        nb = (lib.b200_step1_ll_comm_bytes(L, D, self.Hq, self.Hkv, self.F, self.V, 1) if dataflow
              else lib.b200_step1_comm_bytes(L, D, self.V, 1))
        comm = torch.zeros(nb, dtype=torch.uint8, device=DEV)
        keep = dict(comm=comm, comm_arr=(C.c_void_p * 1)(comm.data_ptr()),
                    an=(C.c_void_p * L)(*[lw["attn_norm"].data_ptr() for lw in self.layers]),
                    fn=(C.c_void_p * L)(*[lw["ffn_norm"].data_ptr() for lw in self.layers]))
        for k in ("wqkv", "wo", "w13", "w2"):
            keep[k] = (_cabi.Linear * L)(*[lw[k].c_struct() for lw in self.layers])
        a = _cabi.Step1Args()
        a.n_layers, a.dim, a.n_heads, a.n_kv_heads, a.ffn = L, D, self.Hq, self.Hkv, self.F
        a.vocab, a.cache_seq, a.eps = self.V, self.S, EPS
        a.token, a.tok_emb, a.pos, a.rope = self.tokens.data_ptr(), self.tok_emb.data_ptr(), self.pos.data_ptr(), self.rope.data_ptr()
        a.kcache, a.vtcache, a.kv_layer_stride = self.kc.data_ptr(), self.vt.data_ptr(), self.kc.stride(0)
        a.h0, a.h1, a.q, a.act = (t.data_ptr() for t in (self.h[0], self.h[1], self.q, self.act))
        a.attn_ws = self.ws.data_ptr()
        a.wqkv, a.wo, a.w13, a.w2 = keep["wqkv"], keep["wo"], keep["w13"], keep["w2"]
        a.attn_norm, a.ffn_norm, a.final_norm = keep["an"], keep["fn"], self.final_norm.data_ptr()
        a.lm_head = self.lm_head.c_struct()
        a.comm, a.tp_world, a.tp_rank = keep["comm_arr"], 1, 0
        a.timeline, a.n_split, a.use_pdl = None, _split_of(self.Hkv), 1
        self._own[dataflow] = (a, keep)
        return a, keep

    def mega_args(self, kind, n_split=None):
        """-> (Step1Args, communication block) of a mega1 / mega2 launch; mega1 takes n_split from the block."""
        if self.eng is not None:
            self.eng.use_mega, self.eng.mega_dataflow = True, kind == "mega2"
            a = self.eng._step1_args()
            comm = self.eng._mega["keep"]["comm"]
        else:
            a, keep = self._own_args(kind == "mega2")
            comm = keep["comm"]
        if kind == "mega1":
            a.attn_ws = self.ws.data_ptr()  # sized for 8 splits
            a.n_split = n_split or _split_of(self.Hkv)
        return a, comm

    def ll_lay(self):
        return nx.ll_layout(self.L, self.D, self.Hq, self.Hkv, self.F, self.V, _split_of(self.Hkv))

    def run_mega(self, kind, n_split=None):
        a, comm = self.mega_args(kind, n_split)
        ops.decode_step1(a, dataflow=kind == "mega2")
        torch.cuda.synchronize()
        if kind == "mega2":
            assert int(comm[:16].view(torch.int32)[2]) == 0, "mega2 error word"
            off = self.ll_lay()["logits"]
        else:
            off = nx.mega1_comm_offsets(self.L, self.D)[1]
        return comm[off:off + 4 * self.V].view(torch.float32).clone()

    def run_separate(self, record=False):
        """The separate kernels with the engine's launch arguments (DecodeEngine._layers / _head, T = 1, TP = 1).
        record: per layer, the fp16 residual entering each norm and every phase output."""
        if self.eng is not None and not record:
            self.eng.use_mega = False
            return self.eng._step(1, 1, self.S).reshape(-1).clone()
        D, S, rec = self.D, self.S, []
        ops.embed(self.tokens, self.tok_emb, self.h[0], 1, D, self.V)
        cur, delta = 0, None
        ns = ops.attn_split(1, self.Hkv, S)
        ws = torch.zeros(ops.attn_workspace_bytes(1, self.Hq, ns), dtype=torch.uint8, device=DEV)
        cnt = torch.zeros(self.Hkv, dtype=torch.int32, device=DEV)
        for i, lw in enumerate(self.layers):
            kc, vt = self.kc[i], self.vt[i]
            r = dict(h_in=(self.h[cur][0] + delta[0]) if delta is not None else self.h[cur][0].clone())
            ops.gemv(lw["wqkv"], 1, resid=self.h[cur], delta=delta, h_out=self.h[1 - cur] if delta is not None else None,
                     gamma=lw["attn_norm"], eps=EPS, epilogue=ops.B200_EPI_QKV, out=self.q,
                     qkv=dict(n_q_rows=self.nq, n_kv_rows=self.nkv, rope=self.rope, pos=self.pos, tokens_per_seq=1,
                              kcache=kc, vtcache=vt, cache_seq=S, prefetch_kv=False))
            if delta is not None:
                cur = 1 - cur
            ops.attn_decode(self.q, kc, vt, self.pos, self.attn, T=1, Hq=self.Hq, Hkv=self.Hkv, cache_seq=S,
                            tokens_per_seq=1, max_kv_len=S, ws=ws, counters=cnt, n_split=ns)
            ops.gemv(lw["wo"], 1, xin=self.attn, epilogue=ops.B200_EPI_F16, out=self.o)
            ops.gemv(lw["w13"], 1, resid=self.h[cur], delta=self.o, h_out=self.h[1 - cur], gamma=lw["ffn_norm"], eps=EPS,
                     epilogue=ops.B200_EPI_SILU, out=self.act)
            cur = 1 - cur
            ops.gemv(lw["w2"], 1, xin=self.act, epilogue=ops.B200_EPI_F16, out=self.f)
            delta = self.f
            if record:
                torch.cuda.synchronize()
                r.update(q=self.q[0].clone(), attn=self.attn[0].clone(), o=self.o[0].clone(), h1=self.h[cur][0].clone(),
                         act=self.act[0].clone(), f=self.f[0].clone(), ns=ns)
                rec.append(r)
        ops.gemv(self.lm_head, 1, resid=self.h[cur], delta=delta, gamma=self.final_norm, eps=EPS,
                 epilogue=ops.B200_EPI_F32, out=self.logits)
        torch.cuda.synchronize()
        out = self.logits.reshape(-1).clone()
        if record:
            rec.append(dict(h_in=self.h[cur][0] + delta[0]))
        return (out, rec) if record else out

    # ------------------------------------------------------------------------------------------------ caches --------
    def fill_cache(self, pos, seed):
        """Noise below pos, the sentinel in row pos and in every later tile, zeros after pos inside pos's tile."""
        g = _gen(seed)
        self.kc.normal_(0.0, 0.5, generator=g)
        self.vt.normal_(0.0, 0.5, generator=g)
        t, r = pos // 32, pos % 32
        s16 = torch.tensor(SENT, dtype=torch.int16, device=DEV).view(torch.float16)
        self.kc[:, :, :, pos] = s16
        self.kc[:, :, :, pos + 1:(t + 1) * 32] = 0
        self.kc[:, :, :, (t + 1) * 32:] = s16
        self.vt[:, :, :, t, :, r] = s16
        self.vt[:, :, :, t, :, r + 1:] = 0
        self.vt[:, :, :, t + 1:] = s16


# ----------------------------------------------------------------------------------------------- phase checks ---------
def _f16_ratio(out, ref, extra=None):
    """largest |out - ref| / tol, tol = half an fp16 ulp of ref + 2^-20 max|ref| (+ an ambiguity term)."""
    tol = ref.abs() * 2.0 ** -11 + float(ref.abs().max()) * 2.0 ** -20 + 1e-7
    if extra is not None:
        tol = tol + extra * (1 + 2.0 ** -10)
    assert torch.isfinite(out).all()
    return float(((out.double().reshape(-1) - ref).abs() / tol).max())


def _gemv_vs_candidates(y16, W, h, gamma, label):
    """fp16 y of a GEMV with the RMSNorm prologue against float64 of every x of the rstd window -> best err/tol."""
    Y = W @ x_candidates(h, gamma, EPS).double().T
    r = min(_f16_ratio(y16, Y[:, c]) for c in range(Y.shape[1]))
    assert r <= 1.0, (label, r)
    return r


def _silu_mismatches(act, y16):
    """act [F] against the fp16 y [2F] of the w13 GEMV: fp16(silu(a)) in fp32 then times b in fp16, either rounding of
    silu(a) where expf may tip it (test_decode_path_gpu.py)."""
    F = act.numel()
    t = y16.reshape(F // 8, 2, 8)
    a, b = t[:, 0].reshape(-1).double(), t[:, 1].reshape(-1).double()
    sl = a / (1 + torch.exp(-a))
    sn, sa, sd = fp16_sides(sl)
    amb = sd <= nx.SILU_REL * sl.abs()
    got = act.double().reshape(-1)
    ok = (got == (sn * b).half().double()) | (amb & (got == (sa * b).half().double()))
    return int((~ok).sum())


def _f16_gemv(pl, N, **kw):
    out = nan16(1, N, device=DEV)
    ops.gemv(pl, 1, out=out, **kw)
    torch.cuda.synchronize()
    return out.reshape(-1)


def _split_attn_ratio(q, kcan, vcan, O, m, lsum, ranges, label):
    """Every split's (O, m, l) against float64 over its key range -> (worst err/tol of O / l, worst |dm| / bound)."""
    Hq, Hkv = q.numel() // 128, kcan.shape[0]
    r = Hq // Hkv
    ra = rm = 0.0
    for sp, (b, e) in enumerate(ranges):
        if e <= b:
            assert bool((O[:, sp] == 0).all() and torch.isinf(m[:, sp]).all() and (lsum[:, sp] == 0).all()), (label, sp)
            continue
        ref = AttnRef(q[None].reshape(1, Hq, 128), kcan[None, :, b:e], vcan[None, :, b:e], [e - b - 1], 1)
        tpw = nx.mega_tiles_per_warp(e - b, 1)
        tol = ref.tol([tpw], nx.MEGA_WARPS)[0]
        out = O[:, sp].double() / lsum[:, sp, None].double()
        assert bool(torch.isfinite(out).all()), (label, sp)
        ra = max(ra, float(((out - ref.out[0]).abs() / tol).max()))
        qq = q.double().reshape(Hkv, r, 128)
        kk = kcan[:, b:e].double()
        tl = torch.einsum("grd,gnd->grn", qq, kk) * nx.ATTN_C_LOG2
        dl = nx.C_ACC * nx.ATTN_C_LOG2 * torch.einsum("grd,gnd->grn", qq.abs(), kk.abs()) + 16 * nx.ATTN_U * tl.abs()
        mref = tl.max(-1).values.reshape(Hq)
        rm = max(rm, float(((m[:, sp].double() - mref).abs() / (dl.max(-1).values.reshape(Hq) + 2.0 ** -20)).max()))
    return ra, rm


def audit_one_layer(rig, kind, pos, n_split=None, X=None):
    """One launch of `kind` at pos on a fresh cache; every phase against float64.  -> {phase: worst err/tol}."""
    assert rig.L == 1
    D, Hq, Hkv, F, V, S, nq, nkv = rig.D, rig.Hq, rig.Hkv, rig.F, rig.V, rig.S, rig.nq, rig.nkv
    lw = rig.layers[0]
    label = f"{rig.name}/{kind}/pos={pos}/ns={n_split}"
    rig.fill_cache(pos, seed=pos + 1)
    kc0, vt0 = rig.kc.clone(), rig.vt.clone()
    rig.pos[0] = pos
    a, comm = rig.mega_args(kind, n_split)
    ns = a.n_split if kind == "mega1" else _split_of(Hkv)
    for t in (rig.h[0], rig.h[1], rig.q, rig.act):
        t.view(torch.int16).fill_(SENT)
    rig.ws.view(torch.int32).fill_(WS_SENT)
    if kind == "mega1":
        parts_off, logits_off = nx.mega1_comm_offsets(1, D)
        comm[parts_off:].view(torch.int32).fill_(LL_SENT32)
    else:
        lay = rig.ll_lay()
        assert lay["total"] == comm.numel() and lay["logits"] == _cabi.lib().b200_step1_ll_logits_offset(1, D, Hq, Hkv, F, V, 1)
        comm[lay["yq"]:].view(torch.int32).fill_(LL_SENT32)
        epoch = int(comm[:16].view(torch.int32)[1])
        seq0 = (epoch * 6 + 1) % (1 << 32)
        logits_off = lay["logits"]
    ops.decode_step1(a, dataflow=kind == "mega2")
    torch.cuda.synchronize()
    res = {}

    # ---- caches: only row pos changed, and it is finite
    for now, before in ((rig.kc, kc0), (rig.vt, vt0)):
        diff = _bits(now) != _bits(before)
        assert int(diff.sum()) <= Hkv * 128, label
    k_can, v_can = kvlayout.k_from_engine(rig.kc[0])[0], kvlayout.v_from_engine(rig.vt[0])[0]
    k_row, v_row = k_can[:, pos].reshape(-1), v_can[:, pos].reshape(-1)
    assert bool(torch.isfinite(k_row).all() and torch.isfinite(v_row).all()), label
    k0c = kvlayout.k_from_engine(kc0[0])[0]
    k0c[:, pos] = k_can[:, pos]
    assert _same(k0c, k_can), label

    # ---- read back the phase outputs
    if kind == "mega1":
        for t in (rig.h[0], rig.h[1], rig.q, rig.act):  # row 0 only
            assert bool((_bits(t[1:]) == SENT).all()), label
        h0, h1, q, act = rig.h[0][0], rig.h[1][0], rig.q[0], rig.act[0][:F]
        assert _same(h0, rig.tok_emb[TOK]), label  # the prologue's h_out of layer 0 is the embedding row
        wsf = rig.ws.view(torch.float32)
        n_o, n_ml = Hq * ns * 128, Hq * ns * 2
        O = wsf[:n_o].view(Hq, ns, 128)
        ml = wsf[n_o:n_o + n_ml].view(Hq, ns, 2)
        m, lsum = ml[..., 0], ml[..., 1]
        assert bool((rig.ws.view(torch.int32)[n_o + n_ml:] == WS_SENT).all()), label
        parts = comm[parts_off:parts_off + 4 * D].view(torch.float16).view(2, D)
        wo_out, w2_out = parts[0], parts[1]
        assert bool((comm[parts_off + 4 * D:logits_off].view(torch.int32) == LL_SENT32).all()), label
    else:
        for t in (rig.h[0], rig.h[1], rig.q, rig.act):  # mega2 keeps h on chip and q / act in LL vectors
            assert bool((_bits(t) == SENT).all()), label
        cpu = comm.cpu().numpy()

        def units(key, n):
            return cpu[lay[key]:lay[key] + 8 * n].view(np.int32).reshape(1, n, 2)

        def f16(key, n, ident):
            p, s = nx.ll_decode(units(key, n))
            assert bool((s == (seq0 + ident) % (1 << 32)).all()), (label, key, int((s != seq0 + ident).sum()))
            return torch.from_numpy(p.reshape(-1).copy()).to(DEV)
        q = f16("yq", nq // 2, 0)
        ykv = f16("ykv", nkv, 0).view(Hkv, 2, 128)
        assert _same(ykv[:, 0].reshape(-1), k_row) and _same(ykv[:, 1].reshape(-1), v_row), label
        att_p, att_s = nx.ll_units_decode32(cpu[lay["att"]:lay["att"] + Hq * ns * 130 * 8].view(np.int32).reshape(Hq, ns, 130, 2))
        assert bool((att_s == (seq0 + 1) % (1 << 32)).all()), (label, "att seq")
        att = torch.from_numpy(att_p.copy()).to(DEV)
        O, m, lsum = att[..., :128], att[..., 128], att[..., 129]
        wo_out = f16("po", D // 2, 2)
        act = f16("act", F // 2, 3)
        w2_out = f16("pf", D // 2, 4)
        h0 = rig.tok_emb[TOK]
        h1 = h0 + wo_out
    logits = comm[logits_off:logits_off + 4 * V].view(torch.float32)
    for t in (q, O, wo_out, act, w2_out, logits):
        assert bool(torch.isfinite(t).all()), label

    # ---- QKV: RMSNorm of the embedding row, gemv1, RoPE + cache append
    e = rig.tok_emb[TOK].reshape(1, D)
    y16 = _f16_gemv(lw["wqkv"], nq + 2 * nkv, resid=e, gamma=lw["attn_norm"], eps=EPS)
    res["qkv"] = X["qkv"] if X and "qkv" in X else _gemv_vs_candidates(y16, lw["Wwqkv"], e, lw["attn_norm"], label)
    if X is not None:
        X["qkv"] = res["qkv"]
    q_e, k_e, v_e = nx.qkv_from_y(y16.reshape(1, -1).cpu(), rig.rope.cpu(), [pos], nq, nkv)
    assert _same(q.cpu(), q_e.reshape(-1)), (label, "q", int((_bits(q.cpu()) != _bits(q_e.reshape(-1))).sum()))
    assert _same(k_row.cpu(), k_e.reshape(-1)) and _same(v_row.cpu(), v_e.reshape(-1)), (label, "kv row")

    # ---- attention: every split over its own key range, then the merge over all keys
    ranges = nx.mega_split_ranges(pos + 1, ns)
    res["attn_split"], res["attn_m"] = _split_attn_ratio(q, k_can, v_can, O, m, lsum, ranges, label)
    assert res["attn_split"] <= 1.0 and res["attn_m"] <= 1.0, (label, res)
    a64, amag = nx.merge_splits64(O, m, lsum)
    full = AttnRef(q.reshape(1, Hq, 128), k_can[None], v_can[None], [pos], 1)
    tol = full.tol([nx.mega_tiles_per_warp(pos + 1, ns)], nx.MEGA_WARPS + ns)[0]
    res["attn_merge"] = float(((a64 - full.out[0]).abs() / tol).max())
    assert res["attn_merge"] <= 1.0, (label, res["attn_merge"])

    # ---- wo against float64 of the merge (either rounding near an fp16 midpoint)
    a64, amag = a64.reshape(-1), amag.reshape(-1)
    near, alt, dist = fp16_sides(a64)
    amb = dist <= MERGE_AMB * (amag + a64.abs())
    Wo = lw["Wwo"]
    res["wo"] = _f16_ratio(wo_out, Wo @ near, Wo.abs() @ ((alt - near).abs() * amb))
    assert res["wo"] <= 1.0, (label, res["wo"])

    # ---- residual add, W13 + SiLU * mul
    h1_e = h0 + wo_out
    assert _same(h1, h1_e), (label, "h1")
    y13 = _f16_gemv(lw["w13"], 2 * F, resid=e, delta=wo_out.reshape(1, D), gamma=lw["ffn_norm"], eps=EPS)
    res["w13"] = _gemv_vs_candidates(y13, lw["Ww13"], h1_e, lw["ffn_norm"], label)
    bad = _silu_mismatches(act, y13)
    assert bad == 0, (label, "act", bad)

    # ---- W2: exact input; the separate gemv1 on the same act gives the same bits
    res["w2"] = _f16_ratio(w2_out, lw["Ww2"] @ act.double())
    assert res["w2"] <= 1.0, (label, res["w2"])
    assert _same(_f16_gemv(lw["w2"], D, xin=act.reshape(1, F)), w2_out), (label, "w2 vs separate gemv1")

    # ---- head: residual add, final RMSNorm, fp16 HMMA GEMV
    hf = h1_e + w2_out
    Xc = x_candidates(hf, rig.final_norm, EPS).double()
    Y, M = rig.Wh @ Xc.T, rig.Wh.abs() @ Xc.abs().T
    got = logits.double()
    res["head"] = float(((got[:, None] - Y).abs() / (Y.abs() * 2.0 ** -11 + C_ACC16 * M + 1e-7)).amax(0).min())
    assert res["head"] <= 1.0, (label, res["head"])
    return res


# ------------------------------------------------------------------------------------ 1. one-layer audit -------------
@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", list(SHAPES))
def test_one_layer_phase_audit_against_float64(name):
    """mega1 and mega2, one layer, every phase against float64 at the positions of the module docstring; mega1 also at
    n_split 1, 3, 8.  cache_seq - 1 makes every warp fold >= 2 tiles (4096 keys at 4 / 3 splits, 8192 at 8)."""
    rig = Rig(name, 1, seed=len(name))
    S, nsc = rig.S, _split_of(rig.Hkv)
    assert nx.mega_tiles_per_warp(S, nsc) >= 2
    positions = [0, 31, 32, 2047, nx.mega_past_boundary_pos(nsc), S - 1]
    runs = [(k, p, None) for p in positions for k in ("mega1", "mega2")]
    runs += [("mega1", p, n) for n in (1, 3, 8) if n != nsc for p in (max(nx.mega_past_boundary_pos(n), 32), 2047, S - 1)]
    worst, cache = {}, {}
    for kind, p, n in runs:
        r = audit_one_layer(rig, kind, p, n, cache)
        for ph, v in r.items():
            key = (kind, ph)
            worst[key] = max(worst.get(key, 0.0), v)
    print(f"\n[{name}] D {rig.D} Hq/Hkv {rig.Hq}/{rig.Hkv} F {rig.F} V {rig.V}, split {nsc}, tiles/warp at {S - 1}: "
          f"{nx.mega_tiles_per_warp(S, nsc)}; {len(runs)} launches")
    for kind in ("mega1", "mega2"):
        print(f"  {kind}: " + ", ".join(f"{ph} {v:.3f}" for (k, ph), v in worst.items() if k == kind))


# --------------------------------------------------------------- 2. bit identity where attention cannot differ -------
@pytest.mark.timeout(600)
@pytest.mark.parametrize("dims,n_layers", [("7b", 1), ("7b", 2), ("7b", 32), ("d1024", 96)])
def test_pos0_mega_and_separate_kernels_bit_identical(dims, n_layers):
    """At pos 0 attention returns v for any split structure, so DESIGN §2 makes every kernel path bit-identical: logits,
    every layer's K / V row, repeated launches and graph replays."""
    if dims == "7b":
        cfg = EngineConfig(kind="llama", n_layers=n_layers, dim=4096, n_heads=32, ffn_hidden=11008, vocab_size=32000,
                           max_seq_len=256, bits=4, group_size=0)
    else:
        cfg = EngineConfig(kind="llama", n_layers=n_layers, dim=1024, n_heads=8, ffn_hidden=2816, vocab_size=32000,
                           max_seq_len=256, bits=4, group_size=0)
    eng = DecodeEngine(cfg, DEV)
    eng.load_random(seed=n_layers)
    g = _gen(5)
    for lw in eng.layers:  # norms that are not all ones
        lw.attn_norm = (1 + 0.2 * torch.randn(cfg.dim, generator=g, device=DEV)).half()
        lw.ffn_norm = (1 + 0.2 * torch.randn(cfg.dim, generator=g, device=DEV)).half()
    eng.allocate_kv_cache(1)
    eng.fill_kv_cache_noise(0.5, seed=6)
    k0, v0 = eng.kcache.clone(), eng.vtcache.clone()
    tok = torch.tensor([TOK], device=DEV)
    assert eng.kcache.shape[0] == n_layers <= 96

    def run(kind, graph=False):
        eng.kcache.copy_(k0)
        eng.vtcache.copy_(v0)
        eng.use_mega, eng.mega_dataflow = kind != "sep", kind == "mega2"
        eng.use_graph = graph
        eng._graphs.clear()
        eng.tokens[0], eng.pos[0] = TOK, 0
        out = (eng.decode_step(tok, 0) if graph else eng._step(1, 1, eng.cache_seq)).reshape(-1).clone()
        if graph:
            out2 = eng._replay(1).reshape(-1).clone()  # a second replay of the same captured step
            assert _same(out, out2), (kind, "graph replay")
        torch.cuda.synchronize()
        if kind == "mega2":
            assert int(eng._mega["keep"]["comm"][:16].view(torch.int32)[2]) == 0
        return out, eng.kcache.clone(), eng.vtcache.clone()

    base = run("sep")
    diffk = _bits(base[1]) != _bits(k0)
    assert 0 < int(diffk.sum()) <= n_layers * eng.Hkv * 128  # one K row per layer and kv head (noise may match a value)
    report = []
    for kind in ("mega1", "mega2"):
        for rep in range(2):
            got = run(kind)
            for i, (x, y) in enumerate(zip(got, base)):
                assert _same(x, y), (kind, rep, ["logits", "kcache", "vcache"][i], int((_bits(x) != _bits(y)).sum()))
        report.append(kind)
    for kind in ("sep", "mega1", "mega2"):
        got = run(kind, graph=True)
        for x, y in zip(got, base):
            assert _same(x, y), (kind, "graph")
    print(f"\n[pos 0, {dims}, {n_layers} layers] separate / mega1 / mega2, eager x2 and graph: logits and "
          f"{n_layers} x {eng.Hkv} K / V rows bit-identical")


# ---------------------------------------------------------------------------- 3. two layers at pos > 0 ---------------
CHAIN_ULPS = 8  # |mega - separate| of the logits and of layer 1's K / V row, in fp16 steps of the largest reference value


@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", list(SHAPES))
def test_two_layer_chain_matches_separate_kernels_within_attention_bound(name):
    """Two layers at pos 2047 and cache_seq - 1 on the same noise cache.  Before the first attention nothing differs:
    layer 0's K / V row is bit-identical on all three paths.  mega1 and mega2 run the same (kv head, split) items with the
    same 16-warp fold and merge order (both take n_split = SMs / Hkv, at most 8), so they are bit-identical everywhere.
    Against the separate kernels the only difference is attention's split structure.  The one-layer audit puts both
    paths' attention within 0.19 of the float64 bound (about one fp16 step of the output), so layer 0's attention
    outputs differ by at most two fp16 steps; wo and w2 mix that into the residual stream, whose own fp16 rounding is one
    step, and layer 1's attention adds two more.  CHAIN_ULPS = 8 fp16 steps of the largest reference value bounds the
    logits and layer 1's K / V row with room for the norm's rescaling (|gamma| <= 1.8 here)."""
    rig = Rig(name, 2, seed=3 + len(name))
    report = []
    for pos in (2047, rig.S - 1):
        rig.fill_cache(pos, seed=pos)
        kc0, vt0 = rig.kc.clone(), rig.vt.clone()
        rig.pos[0] = pos
        ref = rig.run_separate(record=True)[0]
        if rig.eng is not None:  # the engine's own step runs the same launches
            rig.kc.copy_(kc0), rig.vt.copy_(vt0)
            assert _same(rig.run_separate(), ref), (name, pos, "engine step vs the chained launches")
        kc_s, vt_s = rig.kc.clone(), rig.vt.clone()
        runs = {}
        for kind in ("mega1", "mega2"):
            rig.kc.copy_(kc0), rig.vt.copy_(vt0)
            got = rig.run_mega(kind)
            assert bool(torch.isfinite(got).all()), (name, kind, pos)
            for now, before in ((rig.kc, kc0), (rig.vt, vt0)):  # nothing but row pos of each layer changed
                assert int((_bits(now) != _bits(before)).sum()) <= 2 * rig.nkv, (name, kind, pos)
            runs[kind] = (got, rig.kc.clone(), rig.vt.clone())
            ratios = []
            for i in range(2):
                for can, now, sep in ((kvlayout.k_from_engine, rig.kc, kc_s), (kvlayout.v_from_engine, rig.vt, vt_s)):
                    a_, b_ = can(now[i])[0, :, pos].reshape(-1), can(sep[i])[0, :, pos].reshape(-1)
                    if i == 0:
                        assert _same(a_, b_), (name, kind, pos, "layer 0 K / V row")
                    else:
                        tol = CHAIN_ULPS * float(_ulp16(b_.double().abs().max().reshape(1))[0])
                        ratios.append(float((a_.double() - b_.double()).abs().max()) / tol)
            tol = CHAIN_ULPS * float(_ulp16(ref.double().abs().max().reshape(1))[0])
            r_log = float((got.double() - ref.double()).abs().max()) / tol
            report.append(f"{kind}@{pos}: K/V layer 1 {max(ratios):.3f}, logits {r_log:.3f}")
            assert max(ratios + [r_log]) <= 1.0, (name, kind, pos, ratios, r_log)
        for x, y in zip(runs["mega1"], runs["mega2"]):
            assert _same(x, y), (name, pos, "mega1 vs mega2")
    print(f"\n[{name} 2 layers] |mega - separate| / {CHAIN_ULPS} fp16 steps: " + "; ".join(report) +
          "; mega1 == mega2 bit for bit")
