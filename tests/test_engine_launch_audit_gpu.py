"""GPU: every launch DecodeEngine.forward_inference (and forward_full) makes, on the GEMV-chunk path and on the tensor-core
prompt path, audited one at a time on the engine's own buffers against float64.

The kernel modules test each kernel on inputs the test allocates; this module tests the glue between them.  The `ops`
entry points the engine calls (and the engine's `_step`, `_prefill_chunk_tc` and `_allreduce`) are wrapped.  For every
launch the wrapper synchronises, clones what the launch reads and snapshots every engine buffer (h[0], h[1], q, attn, o, f,
act, xn, slot_w, slot_e, act_slots, y_slot, logits_loc, kcache, vtcache, counters, and the prompt buffers of
_prefill_bufs: p_h0, p_h1, p_x, p_qkv, p_q, p_attn, p_o, p_gu, p_act, p_f, p_pos, p_tok, p_slot_w, p_slot_e, p_y_slot),
runs the real launch, synchronises, and checks the launch against float64 computed from its own inputs.  The inputs are
teacher-forced, so an error is the launch's own.  `ws` is scratch.

  embed            rows bit for bit from the table; the tokens and positions staged for the chunk are the expected ones
  RMSNorm prologue h_out = fp16(resid + delta) bit for bit; resid is the residual the previous prologue (or embed) wrote,
                   delta the previous block's output (the h[cur] / h[1 - cur] ping-pong)
  gemv F16 / F32   the section A bound of test_gemv_batched_moe_gpu.py with M = A . |x| built from the engine's own
                   PackedLinear (q, s, z unpacked); with the prologue, for one x of the rstd window (x_candidates).
                   T = 1 launches of quantised linears take the integer-path gemv1; its bound (test_decode_path_gpu.py:
                   half an ulp plus 2^-20 |y| per channel) lies inside this one because M >= |y|
  gemv SILU / QKV  an F16 launch on the cloned inputs gives y (held to the bound); act, q and the K / V cache slots must
                   follow from y bit for bit.  K / V land at cache row row0 + t // tokens_per_seq, position pos[t], of the
                   current layer; every other element of both caches keeps its bytes
  bias (internlm)  QKV with B200_BIAS_ACC: the F16 relaunch carries the same bias, y is held to the bound of
                   x . w_hat + b widened by the one fp32 add (BIAS_ADD_REL, Audit._y_bound), q / K / V follow from y bit
                   for bit.  wo with B200_BIAS_OUT: the launch without the bias gives y0 (held to the bound), and
                   o = fp16(y0 + b) bit for bit.  A bias on any other launch, or the other mode, fails
  attn_decode      the float64 bound of test_attn_decode_gpu.py on the cache rows of the chunk's sequences; counters back
                   at zero
  moe_route        h_out bit for bit, xn_out one candidate, slot_expert / slot_weight a kernel_route outcome of the logit
                   window of its own xn_out (section B); with scores_f32 (mixtral_sparse, which must pass it, and only
                   it) a kernel_route_f32 outcome, or one inside the expf window (oracle.numerics.route_check_f32)
  moe_expert_ffn   section B ranges for act and the bound for y_slot, on every slot routed to a local expert
  moe_combine      bit for bit
  _head            the F32 bound, and its rows are the last token of every sequence (or every row of a decode step)
Every launch: no engine buffer changes outside the output elements its checker verified (the declared rows, and within
them the declared columns), and a launch kind without a checker fails, as does an argument its checker does not take
(no checker swallows keyword arguments: a new epilogue argument fails the audit until a checker checks it).

The tensor-core prompt path (_prefill_chunk_tc: one sequence, <= 256 positions per chunk, every intermediate materialised,
so no checker re-launches anything):
  prefill_rmsnorm  h_out = fp16(resid + delta) bit for bit (None on layer 0), the ping-pong tracked across layers;
                   x_out one of x_candidates(h, gamma, eps, ulps=prefill_rstd_ulps(D)).  The window: each of the 256
                   threads chains D / 256 fmaf of exact fp32 squares, then a 5-level warp tree, then the 8 warp partials in
                   order, so the depth is d = D / 256 + 13 (29 at D = 4096, 45 at 8192) and ssq lies within d u of sum h^2
                   (u = 2^-24, non-negative terms).  / D and + eps round once each: (d + 2) u; sqrtf halves that and
                   rounds (+ u); the reciprocal rounds (+ u): rstd within (d / 2 + 3) u of rstd64, i.e. fewer than
                   d / 2 + 3 fp32 ulps; rounding rstd64 to fp32 adds half an ulp.  fp16(h * rstd) * gamma is then
                   computed exactly from each candidate rstd.
  prefill_gemm_w4  (W4, W3, fp16) |out - ref| <= ulp16(ref) + C_ACC |x| . |w_hat|^T elementwise (test_prefill_gpu.py),
                   ref = float64 x . w_hat^T with w_hat = fp16(fp16(q - z) s) rebuilt from the engine's PackedLinear bytes
                   (the weight itself for fp16), in blocks of output rows; out rows >= T keep their bytes.  internlm's
                   biases as for the GEMV: ACC around ref + b, OUT through a relaunch without the bias
  prefill_rope_kv  q_out = qkv_from_y(qkv rows) bit for bit; K / V at cache row row0 (the chunk's sequence), position
                   pos[t], of the current layer; every other cache byte (other sequences' rows too) keeps its value
  prefill_silu_mul bit for bit outside the SILU_REL band (Mixtral: T k slot rows of the experts' width fe)
  prefill_moe_gemm for every local expert over its slots, the GEMM bound with w13 reading row slot // k of x and w2 row
                   slot of act; slots routed elsewhere and rows >= T k keep their bytes
  attn_decode      sub-launches of <= 32 tokens at their row offset, tokens_per_seq = min(chunk, tn), the host's split
  _head            resid / delta are index_select copies: equal to h[cur][want_rows] / delta[want_rows] bit for bit
Every input a launch reads must have been written by the launch that produces it in this layer (writer tracking), a chunk
writes no buffer of the GEMV path, and every _step / _prefill_chunk_tc call must match the restated path choice of
forward_inference (or forward_full, whose output rows must equal fp16 of each chunk's audited logits).

The module also prints, per launch kind, the launches audited and the worst err / tol, and every routing decision that
differs from the route of the float64 logits of its own input, with the float64 score gap of the experts involved.
"""
import contextlib
import ctypes as C
import inspect
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import _cabi, kvlayout, ops, quant  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig  # noqa: E402
from oracle import cases, omniquant, weights  # noqa: E402
from oracle.llama_port import PortModel  # noqa: E402
from oracle.numerics import (C_ACC, SILU_REL, TUNE_DEFAULTS, AttnRef, attn_host_split, fp16_sides,  # noqa: E402
                             gemv_check, gemv_tol, kernel_route, kernel_route_f32, logit_window, qkv_from_y,
                             route_check, route_check_f32, route_scores32, rstd_candidates, silu_mul_range,
                             x_candidates)
from test_prefill_moe_gpu import BAND_ABS, BAND_FACTOR  # noqa: E402

DEV = "cuda"
BUFS = ("h0", "h1", "q", "attn", "o", "f", "act", "xn", "slot_w", "slot_e", "act_slots", "y_slot", "logits_loc",
        "kcache", "vtcache", "counters")
# the tensor-core prompt path's buffers (DecodeEngine._prefill_bufs), "p_" + their key
PBUFS = ("p_h0", "p_h1", "p_x", "p_qkv", "p_q", "p_attn", "p_o", "p_gu", "p_act", "p_f", "p_pos", "p_tok", "p_slot_w",
         "p_slot_e", "p_y_slot")
SHARED = ("logits_loc", "kcache", "vtcache", "counters")  # the only GEMV-path buffers a tensor-core chunk may write
# the one extra fp32 rounding of a B200_BIAS_ACC launch, relative to |float64 x . w_hat + b| (Audit._y_bound)
BIAS_ADD_REL = 2.0 ** -23
MIXTRAL_WIDTH = dict(dim=4096, hidden_dim=14336, n_layers=1, n_heads=32, n_kv_heads=8, norm_eps=1e-5, rope_theta=1e6,
                     vocab_size=2048, max_seq_len=64, max_batch_size=2, moe=dict(num_experts=8, num_experts_per_tok=2))


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _raw(t):
    t = t.contiguous()
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _same(a, b):
    return torch.equal(_raw(a), _raw(b))


def _dense(pl):
    """float32 (exact) w_hat = (q - z) s and A = s (q + |z|) of a PackedLinear, from its packed bytes; |w| for fp16."""
    N, K = pl.N, pl.K
    if pl.bits == 16:
        src = np.ascontiguousarray(pl.qweight.cpu().numpy())
        out = np.empty((N, K), dtype=np.uint16)
        _cabi.check(_cabi.lib().b200_unpack_f16(N, K, src.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
        w = torch.from_numpy(out.view(np.float16)).to(DEV).float()
        return w, w.abs()
    q = quant.unpack_quantized(pl).to(DEV).float()
    sz = pl.scales.view(torch.float16).float()
    if pl.group_size == 0:
        sz = sz.reshape(N, 1, 2)
    else:
        G = K // pl.group_size
        sz = sz.reshape(N // 16, G, 16, 2).permute(0, 2, 1, 3).reshape(N, G, 2)
    s = sz[..., 0].repeat_interleave(K // sz.shape[1], dim=1)
    z = sz[..., 1].repeat_interleave(K // sz.shape[1], dim=1)
    return (q - z) * s, s * (q + z.abs())


def _w_hat(pl):
    """fp16 [N, K] w_hat = fp16(fp16(q - z) s) of a per-channel PackedLinear (the weight itself for fp16): the weight the
    prompt GEMM's dequant stage rebuilds."""
    if pl.bits == 16:
        return _dense(pl)[0].half()
    assert pl.group_size == 0
    q = quant.unpack_quantized(pl).to(DEV)
    sz = pl.scales.view(torch.float16).reshape(pl.N, 2)
    return quant.dequantize(q, sz[:, :1].contiguous(), sz[:, 1:].contiguous(), pl.K)


def _ulp16(a):
    """fp16 spacing at |a| (subnormal spacing 2^-24 below 2^-14), as in test_prefill_gpu.py."""
    e = torch.floor(torch.log2(a.double().abs().clamp_min(2.0 ** -24)))
    return torch.exp2(e.clamp_min(-14) - 10)


def prefill_rstd_ulps(D):
    """The rstd window of prefill.cu's rmsnorm_kernel at width D (module docstring): ceil(d / 2 + 3.5), d = D / 256 + 13."""
    return math.ceil((D // 256 + 13) / 2 + 3.5)


def _silu_check(g, got, label):
    """g fp16 [n, 2F] in the EPI_SILU layout (w1 / w3 rows interleaved 8 + 8), got [n, F]: fp16(fp16(silu(a)) * b) bit for
    bit, or the other rounding of silu(a) where fp32 silu lies within SILU_REL of an fp16 midpoint."""
    n = g.shape[0]
    t = g.reshape(n, -1, 2, 8)
    a, b = t[:, :, 0].reshape(n, -1).double(), t[:, :, 1].reshape(n, -1).double()
    sl = a / (1 + torch.exp(-a))
    sn, sa, sd = fp16_sides(sl)
    amb = sd <= SILU_REL * sl.abs()
    got = got.double()
    ok = (got == (sn * b).half().double()) | (amb & (got == (sa * b).half().double()))
    assert bool(ok.all()), (label, "silu", int((~ok).sum()))


class Audit:
    """The wrappers, the per-launch checkers and what they found (module docstring)."""

    def __init__(self, eng):
        self.eng, self.c = eng, eng.cfg
        self.real = {}
        self.dense_cache = {}
        self.stats = {}            # kind -> [launches, worst err / tol]
        self.flips = []            # routing decisions that differ from the float64 route of their own input
        self.ties = 0              # tokens routed with two exactly equal float64 gate logits
        self.routed = 0            # tokens routed
        self.route_window = 0      # tokens routed inside the expf window rather than bit for bit
        self.queue, self.ctx = [], None
        self.layer, self.resid, self.delta = -1, None, None
        self.n_engine = 0          # launch_count increments inside audited engine launches
        self.n_checker = 0         # launch_count increments of the checkers' own relaunches
        self.start_pos = 0
        self.even = int(os.environ.get("B200_ATTN_EVEN", TUNE_DEFAULTS["B200_ATTN_EVEN"]))
        self.tc = False            # inside a _prefill_chunk_tc call
        self.n_norm = 0            # prefill_rmsnorm launches of the current chunk
        self.x_norm = None         # which norm ("attn" / "ffn") last wrote p_x
        self.attn_t0 = 0           # first token of the next attention sub-launch of the current tensor-core layer
        self.writer = {}           # buffer -> (launch kind, layer) of its last writer in the current chunk
        self.done = []             # the _step / _prefill_chunk_tc calls made, with the logits they returned
        self.w_hat_cache = {}
        self.hidden = None         # a dict to record the residual stream: (start_pos, layer, "attn" / "block", seq, off) -> fp16

    # ------------------------------------------------------------------------------------------ plumbing ---------
    def bufs(self):
        e = self.eng
        out = dict(h0=e.h[0], h1=e.h[1])
        for n in BUFS[2:]:
            t = getattr(e, n, None)
            if t is not None:
                out[n] = t
        if e._pf is not None:
            out.update(p_h0=e._pf["h"][0], p_h1=e._pf["h"][1])
            out.update({n: e._pf[n[2:]] for n in PBUFS[2:] if n[2:] in e._pf})
        return out

    def name(self, t):
        if t is None:
            return None
        for n, b in self.bufs().items():
            if t.data_ptr() == b.data_ptr() and t.dtype == b.dtype:
                return n
        return "other"

    def locate(self, t):
        """A buffer or a row-offset view of one (b["q"][t0:], ...) -> (name, first row); ("other", None) otherwise."""
        for n, b in self.bufs().items():
            if t.dtype != b.dtype:
                continue
            off, row = t.data_ptr() - b.data_ptr(), b[0].numel() * b.element_size() if b.dim() > 1 else b.element_size()
            if 0 <= off < b.numel() * b.element_size() and off % row == 0:
                return n, off // row
        return "other", None

    def pair(self):
        return ("p_h0", "p_h1") if self.tc else ("h0", "h1")

    def p(self, n):
        """The buffer `n` of the path running: the tensor-core chunk's own copy of it, if it has one."""
        return "p_" + n if self.tc else n

    def wrote(self, n, kind):
        """The buffer n holds what `kind` wrote in the current layer of the current chunk."""
        assert self.writer.get(n) == (kind, self.layer), (n, "last written by", self.writer.get(n), "not", kind, self.layer)

    def w_hat(self, pl):
        if id(pl) not in self.w_hat_cache:
            self.w_hat_cache[id(pl)] = (pl, _w_hat(pl))
        return self.w_hat_cache[id(pl)][1]

    def gemm_check(self, out, X, pl, label, bias=None):
        """out [n, N] fp16 against float64 X [n, K] . w_hat^T with the prompt GEMM's bound, in blocks of output rows (a
        70B-width w13's w_hat is 3.8 GB in float64) -> worst err / tol.  bias (B200_BIAS_ACC, out = fp16(fl32(acc + b))):
        ref + b, and the one extra fp32 rounding of the add, BIAS_ADD_REL |ref + b| (as Audit._y_bound derives it)."""
        W = self.w_hat(pl)
        assert torch.isfinite(out).all(), label
        Xd = X.double()
        Xa = Xd.abs()
        blk = max(128, (1 << 25) // pl.K // 128 * 128)
        worst = 0.0
        for n0 in range(0, pl.N, blk):
            w = W[n0:n0 + blk].double()
            ref, mag = Xd @ w.T, Xa @ w.abs().T
            tol = C_ACC * mag
            if bias is not None:
                ref = ref + bias[n0:n0 + blk].double()[None]
                tol = tol + BIAS_ADD_REL * ref.abs()
            err = (out[:, n0:n0 + blk].double() - ref).abs()
            worst = max(worst, float((err / (_ulp16(ref) + tol)).max()))
        assert worst <= 1.0, (label, worst)
        return worst

    def dense(self, pl):
        if id(pl) not in self.dense_cache:
            self.dense_cache[id(pl)] = (pl,) + _dense(pl)
        _, W, A = self.dense_cache[id(pl)]
        return W.double(), A.double()

    def note(self, kind, ratio):
        s = self.stats.setdefault(kind, [0, 0.0])
        s[0] += 1
        s[1] = max(s[1], ratio)

    @contextlib.contextmanager
    def installed(self):
        """Wrap every ops function that launches (those counting launch_count), the engine's _step and _allreduce."""
        names = [n for n, f in vars(ops).items() if callable(f) and getattr(f, "__module__", None) == ops.__name__
                 and "launch_count" in getattr(getattr(f, "__code__", None), "co_names", ())]
        assert {"embed", "gemv", "attn_decode", "moe_route", "moe_expert_ffn", "moe_combine", "prefill_rmsnorm",
                "prefill_gemm_w4", "prefill_rope_kv", "prefill_silu_mul", "prefill_moe_gemm_w4"} <= set(names), names
        for n in names:
            self.real[n] = getattr(ops, n)
            setattr(ops, n, self._wrap(n, self.real[n]))
        eng = self.eng
        eng._step = self._step_wrapper(eng._step)
        eng._prefill_chunk_tc = self._chunk_wrapper(eng._prefill_chunk_tc)
        eng._allreduce = self._allreduce
        try:
            yield self
        finally:
            for n in names:
                setattr(ops, n, self.real[n])
            del eng._step, eng._prefill_chunk_tc, eng._allreduce

    def _wrap(self, kind, real):
        def launch(*a, **kw):
            torch.cuda.synchronize()
            before = {n: b.clone() for n, b in self.bufs().items()}
            n0 = ops.launch_count
            real(*a, **kw)
            self.n_engine += ops.launch_count - n0
            torch.cuda.synchronize()
            check = getattr(self, "check_" + kind, None)
            assert check is not None, f"launch {kind} has no checker: the audit does not know what it may write"
            try:
                inspect.signature(check).bind(before, *a, **kw)
            except TypeError as err:
                raise AssertionError(f"launch {kind}: an argument its checker does not check ({err})") from None
            declared = check(before, *a, **kw)
            self.no_stray_writes(kind, before, declared)
            for n in declared:
                self.writer[n] = (kind, self.layer)
        return launch

    def no_stray_writes(self, kind, before, declared):
        """declared: name -> n (rows [0, n) verified whole by the checker), (n, c) (only columns [0, c) of those rows
        verified: the rest of the rows must keep their bytes), slice(r0, r1) (rows [r0, r1) verified), ("flat", n) (the
        first n elements of the buffer, read as one flat array, verified) or 'checked' (the whole buffer verified)."""
        for n, b in self.bufs().items():
            d = declared.get(n, 0)
            if d == "checked":
                continue
            if isinstance(d, slice):
                assert _same(b[:d.start], before[n][:d.start]) and _same(b[d.stop:], before[n][d.stop:]), (
                    kind, self.layer, n, "written outside the declared output rows")
                continue
            if isinstance(d, tuple) and d[0] == "flat":
                assert _same(b.view(-1)[d[1]:], before[n].view(-1)[d[1]:]), (kind, self.layer, n,
                                                                              "written outside the declared output")
                continue
            rows, cols = d if isinstance(d, tuple) else (d, None)
            assert _same(b[rows:], before[n][rows:]), (kind, self.layer, n, "written outside the declared output rows")
            if cols is not None:
                assert _same(b[:rows, cols:], before[n][:rows, cols:]), (kind, self.layer, n,
                                                                         "written outside the declared output columns")

    def _allreduce(self, t, T):
        assert self.c.tp_world == 1
        before = {n: b.clone() for n, b in self.bufs().items()}
        type(self.eng)._allreduce(self.eng, t, T)
        torch.cuda.synchronize()
        assert self.name(t) in (self.p("o"), self.p("f"))
        self.no_stray_writes("allreduce", before, {})
        self.note("allreduce (TP = 1: no-op)", 0.0)

    def expect(self, toks, start_pos):
        """The _step / _prefill_chunk_tc calls forward_inference must make for tokens [bsz, seqlen] at start_pos
        (engine.py): the tensor-core path when (seqlen >= TC_MIN_PROMPT.get(bits, 33) or force_tc) and
        prefill_tc_supported(), one sequence at a time in chunks of <= T_PREFILL positions; else single-token decode steps
        or the GEMV chunks."""
        e = self.eng
        bsz, seqlen = toks.shape
        tm, S = e.t_max, e.cache_seq
        self.start_pos = start_pos
        if (seqlen >= e.TC_MIN_PROMPT.get(e.cfg.bits, 33) or e.force_tc) and e.prefill_tc_supported():
            for b0 in range(bsz):
                off = 0
                while off < seqlen:
                    ci = min(e.T_PREFILL, seqlen - off)
                    last = off + ci >= seqlen
                    self.queue.append(dict(tc=True, T=ci, tps=ci, kv=min(S, (start_pos + off + ci + 127) // 128 * 128),
                                           row0=b0, want=last, rows=[ci - 1] if last else None, tok=toks[b0, off:off + ci],
                                           pos=list(range(start_pos + off, start_pos + off + ci)), seq=[b0] * ci,
                                           off=list(range(off, off + ci))))
                    off += ci
            return
        if seqlen == 1:
            kv = min(S, (start_pos + 128) // 128 * 128)
            for b0 in range(0, bsz, tm):
                b1 = min(bsz, b0 + tm)
                self.queue.append(dict(T=b1 - b0, tps=1, kv=kv, row0=b0 if bsz > tm else 0, want=True, rows=None,
                                       tok=toks[b0:b1, 0], pos=[start_pos] * (b1 - b0), seq=list(range(b0, b1)),
                                       off=[0] * (b1 - b0)))
            return
        gb = min(bsz, tm)
        for b0 in range(0, bsz, gb):
            nb = min(bsz, b0 + gb) - b0
            ci_max, off = max(1, tm // nb), 0
            while off < seqlen:
                ci = min(ci_max, seqlen - off)
                last = off + ci >= seqlen
                self.queue.append(dict(T=nb * ci, tps=ci, kv=min(S, (start_pos + off + ci + 127) // 128 * 128), row0=b0,
                                       want=last, rows=list(range(ci - 1, nb * ci, ci)) if last else None,
                                       tok=toks[b0:b0 + nb, off:off + ci].reshape(-1),
                                       pos=[start_pos + off + j for _ in range(nb) for j in range(ci)],
                                       seq=[b0 + b for b in range(nb) for _ in range(ci)],
                                       off=[off + j for _ in range(nb) for j in range(ci)]))
                off += ci

    def expect_full(self, toks):
        """The _step calls forward_full must make for tokens [bsz, seqlen]: the GEMV chunks from position 0, every chunk
        with the logits of all its rows."""
        e = self.eng
        bsz, seqlen = toks.shape
        tm, S = e.t_max, e.cache_seq
        self.start_pos = 0
        gb = min(bsz, tm)
        for b0 in range(0, bsz, gb):
            nb = min(bsz, b0 + gb) - b0
            ci_max, off = max(1, tm // nb), 0
            while off < seqlen:
                ci = min(ci_max, seqlen - off)
                self.queue.append(dict(T=nb * ci, tps=ci, kv=min(S, (off + ci + 127) // 128 * 128), row0=b0, want=True,
                                       rows=None, nb=nb, ci=ci, off0=off, tok=toks[b0:b0 + nb, off:off + ci].reshape(-1),
                                       pos=[off + j for _ in range(nb) for j in range(ci)],
                                       seq=[b0 + b for b in range(nb) for _ in range(ci)],
                                       off=[off + j for _ in range(nb) for j in range(ci)]))
                off += ci

    def _step_wrapper(self, real):
        def step(T, tokens_per_seq, max_kv_len, row0=0, want_logits=True, last_rows=None):
            assert self.queue, "a _step the schedule does not call for"
            e = self.queue.pop(0)
            assert not e.get("tc"), "a GEMV _step where the tensor-core path was due"
            rows = None if last_rows is None else last_rows.tolist()
            got = dict(T=T, tps=tokens_per_seq, kv=max_kv_len, row0=row0, want=want_logits, rows=rows)
            assert got == {k: e[k] for k in got}, ("_step arguments", got, {k: e[k] for k in got})
            self.ctx, self.layer, self.tc, self.writer = e, -1, False, {}
            lg = real(T, tokens_per_seq, max_kv_len, row0=row0, want_logits=want_logits, last_rows=last_rows)
            e["logits"] = None if lg is None else lg.clone()
            self.done.append(e)
            return lg
        return step

    def _chunk_wrapper(self, real):
        def chunk(tokens, pos, tokens_per_seq, row0, max_kv_len, want_rows):
            assert self.queue, "a _prefill_chunk_tc the schedule does not call for"
            e = self.queue.pop(0)
            assert e.get("tc"), "a tensor-core chunk where the GEMV path was due"
            rows = None if want_rows is None else want_rows.tolist()
            got = dict(T=tokens.numel(), tps=tokens_per_seq, kv=max_kv_len, row0=row0, rows=rows)
            assert got == {k: e[k] for k in got}, ("_prefill_chunk_tc arguments", got, {k: e[k] for k in got})
            assert torch.equal(tokens.cpu(), e["tok"].cpu()) and pos.tolist() == e["pos"], "chunk tokens / positions"
            self.eng._prefill_bufs()
            gemv_before = {n: b.clone() for n, b in self.bufs().items() if n in BUFS and n not in SHARED}
            self.ctx, self.layer, self.tc, self.writer, self.n_norm = e, -1, True, {}, 0
            lg = real(tokens, pos, tokens_per_seq, row0, max_kv_len, want_rows)
            torch.cuda.synchronize()
            self.tc = False
            assert self.layer == len(self.eng.layers) - 1, ("layers run", self.layer)
            for n, b in gemv_before.items():
                assert _same(self.bufs()[n], b), (n, "a GEMV-path buffer written by a tensor-core chunk")
            assert (lg is None) == (rows is None)
            e["logits"] = None if lg is None else lg.clone()
            self.done.append(e)
            return lg
        return chunk

    # ------------------------------------------------------------------------------------------- checkers --------
    def check_embed(self, before, tokens, table, h, T, D, vocab):
        e, x = self.eng, self.ctx
        h0 = self.pair()[0]
        toks, pos = (e._pf["tok"], e._pf["pos"]) if self.tc else (e.tokens, e.pos)
        assert self.name(h) == h0 and tokens.data_ptr() == toks.data_ptr()
        assert T == x["T"] and torch.equal(toks[:T].cpu(), x["tok"].cpu()), "tokens staged for the chunk"
        assert pos[:T].tolist() == x["pos"], "positions staged for the chunk"
        assert _same(h[:T], table[tokens[:T]]), "embed rows"
        self.resid, self.delta, self.layer = h0, None, -1
        self.note("embed", 0.0)
        return {h0: T}

    def _prologue(self, resid, delta, h_out, T):
        """The residual stream of an RMSNorm prologue: -> (h [T, K] the normalised rows, declared h_out rows)."""
        b = self.bufs()
        assert self.name(resid) == self.resid, ("resid", self.name(resid), self.resid)
        assert self.name(delta) == self.delta, ("delta", self.name(delta), self.delta)
        if delta is None:
            assert h_out is None
            return resid[:T].clone(), {}
        pr = self.pair()
        other = pr[1] if self.resid == pr[0] else pr[0]
        assert self.name(h_out) == other, ("h_out", self.name(h_out))
        h = resid[:T] + delta[:T]
        assert _same(h_out[:T], h), (self.layer, "h_out != fp16(resid + delta)")
        self.resid = other
        return b[other][:T].clone(), {other: T}

    def _y_bound(self, y, h, gamma, eps, pl, bias=None):
        """y [T, N] (fp16 or fp32) against float64 for the best rstd candidate of every row -> worst err / tol.

        bias (B200_BIAS_ACC): y = fp16(fl32(acc + b)) against Y = x . w_hat + b.  With |acc - x . w_hat| <= C_ACC M the
        extra fp32 add rounds once, fl32(acc + b) = (acc + b)(1 + d), |d| <= 2^-24, so |fl32(acc + b) - Y| <=
        C_ACC M (1 + 2^-24) + 2^-24 |Y|, and the fp16 rounding adds half an ulp of a value within (1 + 2^-23) |Y| +
        2 C_ACC M.  The GEMV bound (gemv_tol: 2^-11 |Y| + C_ACC M (1 + 2^-10) + 2^-25) covers all of it but the
        2^-24 |Y| (1 + 2^-11) + 2^-35 |Y| of the add, which BIAS_ADD_REL |Y| = 2^-23 |Y| covers."""
        W, A = self.dense(pl)
        b = None if bias is None else bias.double()
        worst = 0.0
        for t in range(y.shape[0]):
            X = x_candidates(h[t], gamma, eps).double()
            Y, M = X @ W.T, X.abs() @ A.T
            tol = gemv_tol(Y, M)
            if b is not None:
                Y = Y + b[None]
                tol = gemv_tol(Y, M) + BIAS_ADD_REL * Y.abs()
            r = ((y[t].double()[None] - Y).abs() / tol).amax(1)
            worst = max(worst, float(r.min()))
        assert worst <= 1.0, (self.layer, pl.N, pl.K, worst)
        return worst

    def _relaunch(self, name, *a, **kw):
        """A checker's own launch of the real entry point `name`, synchronised and counted apart from the engine's."""
        n0 = ops.launch_count
        self.real[name](*a, **kw)
        torch.cuda.synchronize()
        self.n_checker += ops.launch_count - n0

    def _f16_relaunch(self, pl, T, resid, delta, gamma, eps, bias=None, bias_mode=ops.B200_BIAS_NONE):
        y = torch.empty(T, pl.N, dtype=torch.float16, device=DEV)
        n0 = self.n_checker
        self._relaunch("gemv", pl, T, out=y, epilogue=ops.B200_EPI_F16, resid=resid, delta=delta, gamma=gamma, eps=eps,
                       bias=bias, bias_mode=bias_mode)
        assert self.n_checker == n0 + 1
        return y

    def _bias_role(self, lin, bias, bias_mode):
        """The bias a launch of `lin` must carry: internlm's Wqkv bias before RoPE (B200_BIAS_ACC, one rounding of acc + b)
        and its out_proj bias on the fp16 output (B200_BIAS_OUT); none on any other linear, or on a model without them."""
        lw = self.eng.layers[self.layer]
        want = {id(lw.wqkv): (lw.bqkv, ops.B200_BIAS_ACC), id(lw.wo): (lw.bo, ops.B200_BIAS_OUT)}.get(id(lin), (None, None))
        if want[0] is None:
            assert bias is None and bias_mode in (None, ops.B200_BIAS_NONE), (self.layer, "a bias this linear does not have")
            return None
        assert bias is want[0] and bias_mode == want[1], (self.layer, "bias / bias_mode", bias_mode, "expected", want[1])
        return bias

    def check_gemv(self, before, lin, T, *, out, epilogue=ops.B200_EPI_F16, xin=None, resid=None, delta=None, h_out=None,
                   gamma=None, eps=1e-5, qkv=None, moe=None, use_pdl=False, ring_bytes=0, prefetch=None, ar=None,
                   prefetch_const=None, bias=None, bias_mode=ops.B200_BIAS_NONE):
        """use_pdl, ring_bytes, prefetch and prefetch_const change nothing a launch computes (test_decode_path_gpu.py holds
        them to bit identity); every other argument is checked."""
        e, x = self.eng, self.ctx
        assert moe is None and ar is None, "moe-slot / fused all-reduce gemv: no checker"
        if epilogue not in (ops.B200_EPI_QKV, ops.B200_EPI_F16):
            assert bias is None and bias_mode == ops.B200_BIAS_NONE, "a bias on a gemv epilogue without a bias checker"
        if epilogue == ops.B200_EPI_QKV:
            return self._check_qkv(before, lin, T, out, resid, delta, h_out, gamma, eps, qkv, bias, bias_mode)
        if epilogue == ops.B200_EPI_SILU:
            assert self.c.kind == "llama" and lin is e.layers[self.layer].w13 and self.name(out) == "act"
            rb, db = resid.clone(), delta.clone()
            h, decl = self._prologue(resid, delta, h_out, T)
            y = self._f16_relaunch(lin, T, rb, db, gamma, eps)
            r = self._y_bound(y, h, gamma, eps, lin)
            _silu_check(y, out[:T, :lin.N // 2], self.layer)
            self.note("gemv SILU (w13)", r)
            return dict(decl, act=(T, lin.N // 2))
        if epilogue == ops.B200_EPI_F32:  # _head
            assert lin is e.lm_head and self.name(out) == "logits_loc" and x["want"]
            rows = x["rows"] if x["rows"] is not None else list(range(x["T"]))
            assert T == len(rows)
            b = self.bufs()
            assert _same(resid[:T], b[self.resid][rows]), "_head: resid rows are not the last token of every sequence"
            assert _same(delta[:T], b[self.delta][rows]), "_head: delta rows are not the last token of every sequence"
            assert h_out is None and gamma is e.final_norm
            h = resid[:T] + delta[:T]
            r = self._y_bound(out[:T], h, gamma, eps, lin)
            assert torch.equal(out[:T], out[:T].half().float())
            self.note("gemv F32 (lm_head)", r)
            return {"logits_loc": T}
        assert epilogue == ops.B200_EPI_F16 and resid is None, "gemv launch kind without a checker"
        lw = e.layers[self.layer]
        src, dst = self.name(xin), self.name(out)
        if lin is lw.wo:
            assert (src, dst) == ("attn", "o")
            kind = "gemv F16 (wo)"
            self.delta = "o"
        else:
            assert lin is lw.w2 and (src, dst) == ("act", "f")
            kind = "gemv F16 (w2)"
            self.delta = "f"
        b = self._bias_role(lin, bias, bias_mode)
        W, A = self.dense(lin)
        xd = xin[:T, :lin.K].double()
        y = out[:T]
        if b is not None:
            # B200_BIAS_OUT: the launch without the bias gives y0 (held to the bound); out = fp16(y0 + b) bit for bit
            y = torch.empty(T, lin.N, dtype=torch.float16, device=DEV)
            self._relaunch("gemv", lin, T, xin=xin, out=y, epilogue=ops.B200_EPI_F16, use_pdl=use_pdl,
                           ring_bytes=ring_bytes, prefetch=prefetch, prefetch_const=prefetch_const)
            assert _same(out[:T], (y.float() + b.float()[None]).half()), (self.layer, kind, "out != fp16(y0 + b)")
            kind += " BIAS_OUT"
        r, _, _ = gemv_check(y, xd @ W.T, xd.abs() @ A.T, (kind, self.layer))
        self.note(kind, r)
        return {dst: T}

    def _check_qkv(self, before, lin, T, out, resid, delta, h_out, gamma, eps, qkv, bias, bias_mode):
        """The F16 relaunch carries the launch's own bias (B200_BIAS_ACC: y = fp16(acc + b), the value RoPE starts from),
        so q and K / V follow from y bit for bit with or without one; y is held to the bound of x . w_hat (+ b)."""
        e, x = self.eng, self.ctx
        self.layer += 1
        i, row0, tps = self.layer, x["row0"], x["tps"]
        lw = e.layers[i]
        assert lin is lw.wqkv and gamma is lw.attn_norm and self.name(out) == "q"
        b = self._bias_role(lin, bias, bias_mode)
        assert qkv["tokens_per_seq"] == tps and qkv["pos"].data_ptr() == e.pos.data_ptr() and qkv["rope"] is e.rope
        assert qkv["kcache"].data_ptr() == e.kcache[i, row0].data_ptr(), ("K cache slice", i, row0)
        assert qkv["vtcache"].data_ptr() == e.vtcache[i, row0].data_ptr(), ("V cache slice", i, row0)
        assert set(qkv) <= {"n_q_rows", "n_kv_rows", "rope", "pos", "tokens_per_seq", "kcache", "vtcache", "cache_seq",
                            "prefetch_kv"} and qkv["cache_seq"] == e.cache_seq, sorted(qkv)
        rb, db = resid.clone(), None if delta is None else delta.clone()
        h, decl = self._prologue(resid, delta, h_out, T)
        y = self._f16_relaunch(lin, T, rb, db, gamma, eps, bias=b, bias_mode=bias_mode if b is not None else
                               ops.B200_BIAS_NONE)
        r = self._y_bound(y, h, gamma, eps, lin, bias=b)
        nq, nkv = qkv["n_q_rows"], qkv["n_kv_rows"]
        assert (nq, nkv) == (e.Hq * 128, e.Hkv * 128)
        pos = x["pos"]
        q, k, v = qkv_from_y(y, e.rope, pos, nq, nkv)
        assert _same(out[:T], q), (i, "q != RoPE(y)")
        self._kv_written(before, [row0 + t // tps for t in range(T)], pos, k, v)
        self.note("gemv QKV BIAS_ACC" if b is not None else "gemv QKV", r)
        return dict(decl, q=T, kcache="checked", vtcache="checked")

    def _kv_written(self, before, rows, pos, k, v):
        """Token t's K / V (k, v [T, n_kv]) at cache row rows[t], position pos[t], of the current layer; every other
        element of both caches keeps its bytes."""
        e, i = self.eng, self.layer
        kc = kvlayout.k_from_engine(before["kcache"][i])
        vc = kvlayout.v_from_engine(before["vtcache"][i])
        for t, b in enumerate(rows):
            kc[b, :, pos[t]] = k[t].view(-1, 128)
            vc[b, :, pos[t]] = v[t].view(-1, 128)
        kexp, vexp = before["kcache"].clone(), before["vtcache"].clone()
        kexp[i], vexp[i] = kvlayout.k_to_engine(kc), kvlayout.v_to_engine(vc)
        assert _same(e.kcache, kexp), (i, rows[0], "K cache: a slot other than (row, pos[t]) or a wrong value")
        assert _same(e.vtcache, vexp), (i, rows[0], "V cache: a slot other than (row, pos[t]) or a wrong value")

    def check_attn_decode(self, before, q, kcache, vtcache, pos, out, *, T, Hq, Hkv, cache_seq, tokens_per_seq, max_kv_len,
                          ws=None, counters=None, n_split=0, scale=None, use_pdl=False, prefetch=None):
        e, x = self.eng, self.ctx
        assert scale is None, "attention scale other than 1 / sqrt(128): the float64 bound assumes that one"
        i, row0 = self.layer, x["row0"]
        t0, tps, kind = 0, x["tps"], "attn_decode"
        if self.tc:
            # <= 32-token sub-launches at row offsets t0 = 0, 32, ... of the chunk (one sequence: cache row row0)
            t0, kind = self.attn_t0, "attn_decode (tensor-core chunk)"
            assert t0 < x["T"] and T == min(32, x["T"] - t0), ("attention sub-launch", t0, T)
            tps = min(x["tps"], T)
            row0 += t0 // x["tps"]
            assert n_split == ops.attn_split(T, Hkv, max_kv_len), "not the host's split"
            self.wrote("p_q", "prefill_rope_kv")
        assert (self.locate(q), self.locate(out)) == ((self.p("q"), t0), (self.p("attn"), t0))
        assert self.locate(pos) == ("p_pos", t0) if self.tc else pos.data_ptr() == e.pos.data_ptr()
        assert self.name(counters) == "counters"
        assert (self.tc or T == x["T"]) and tokens_per_seq == tps
        assert max_kv_len == x["kv"] and (Hq, Hkv, cache_seq) == (e.Hq, e.Hkv, e.cache_seq)
        assert kcache.data_ptr() == e.kcache[i, row0].data_ptr() and vtcache.data_ptr() == e.vtcache[i, row0].data_ptr()
        nseq = -(-T // tokens_per_seq)
        kc = kvlayout.k_from_engine(kcache[:nseq])
        vc = kvlayout.v_from_engine(vtcache[:nseq])
        ref = AttnRef(q[:T].view(T, Hq, 128), kc, vc, x["pos"][t0:t0 + T], tokens_per_seq)
        n_launched, chunk = attn_host_split(max_kv_len, n_split)
        r = ref.ratio(out[:T].view(T, Hq, 128), n_launched, chunk, self.even)
        assert r <= 1.0, (i, "attention", r)
        assert int(counters.abs().sum()) == 0, "attention counters not reset"
        self.note(kind, r)
        if self.tc:
            self.attn_t0 += T
            return {"p_attn": slice(t0, t0 + T)}
        return {"attn": T}

    def check_moe_route(self, before, *, T, D, E, topk, resid, delta, h_out, gamma, eps, gate_w, xn_out, slot_weight,
                        slot_expert, use_pdl=False, scores_f32=False):
        """scores_f32 must be the model's rule (mixtral_sparse: fp32, route_check_f32; Mixtral: fp16, route_check); the
        float64 flip report routes the float64 logits by the same rule."""
        e, x = self.eng, self.ctx
        i, k = self.layer, topk
        lw = e.layers[i]
        assert gate_w is lw.gate and gamma is lw.ffn_norm and T == x["T"]
        assert bool(scores_f32) == e.cfg.sparse_moe and scores_f32 in (0, 1, False, True), ("score rule", scores_f32)
        assert (D, E, topk) == (e.cfg.dim, e.cfg.num_experts, e.cfg.experts_per_tok)
        xn_n, sw_n, se_n = self.p("x") if self.tc else "xn", self.p("slot_w"), self.p("slot_e")
        assert (self.name(xn_out), self.name(slot_weight), self.name(slot_expert)) == (xn_n, sw_n, se_n)
        if self.tc:
            self.wrote("p_o", "prefill_gemm_w4")
        h, decl = self._prologue(resid, delta, h_out, T)
        xn = xn_out[:T]
        for t in range(T):
            X = x_candidates(h[t], gamma, eps)
            assert bool((_raw(X) == _raw(xn[t])[None]).all(1).any()), (i, t, "xn_out is no candidate of the rstd window")
        se, sw = slot_expert[:T * k].view(T, k), slot_weight[:T * k].view(T, k)
        check, route = (route_check_f32, kernel_route_f32) if scores_f32 else (route_check, kernel_route)
        matched, window, skipped = check(xn, gate_w, sw, se, k)
        assert skipped == 0 and matched + window == T
        self.route_window += window
        # the float64 route of the same input: logits rounded to nearest fp16, then the kernel's routing rule
        L, R = logit_window(xn, gate_w)
        near = fp16_sides(L)[0].half().cpu()
        idx64, _ = route(near, k)
        p64 = torch.softmax(L, -1).cpu()
        s32 = route_scores32(near)
        se_c = se.cpu().long()
        for t in torch.nonzero((idx64 != se_c).any(1)).reshape(-1).tolist():
            j = int(torch.nonzero(idx64[t] != se_c[t])[0])
            a, b = int(se_c[t, j]), int(idx64[t, j])
            self.flips.append(dict(start_pos=self.start_pos, layer=i, seq=x["seq"][t], pos=x["pos"][t],
                                   kernel=se_c[t].tolist(), float64=idx64[t].tolist(), rule="fp32" if scores_f32 else "fp16",
                                   gap=float(p64[t, a] - p64[t, b]), gap32=float(s32[t, a] - s32[t, b]),
                                   logit_gap=float(L[t, a] - L[t, b]), window=float(R[t, a] + R[t, b])))
        Lc = L.cpu()
        self.ties += sum(int(Lc[t].unique().numel() < Lc.shape[1]) for t in range(T))
        self.routed += T
        kind = "moe_route" + (" fp32 rule" if scores_f32 else "")
        self.note(kind + (" (tensor-core chunk)" if self.tc else ""), 0.0)
        return dict(decl, **{xn_n: T, sw_n: T * k, se_n: T * k})

    def check_moe_expert_ffn(self, before, w13, w2, *, T, D, F, topk, e_first, xn, slot_expert, act, y_slot, use_pdl=False):
        e = self.eng
        lw = e.layers[self.layer]
        assert w13 == lw.e_w13 and w2 == lw.e_w2 and e_first == e.e_first and F == e.F
        assert (self.name(xn), self.name(slot_expert), self.name(act), self.name(y_slot)) == ("xn", "slot_e", "act_slots",
                                                                                              "y_slot")
        ns = T * topk
        se = slot_expert[:ns].long()
        fe = w2[0].K  # the experts' own FFN width: act_slots columns [fe, F) are not theirs
        worst = 0.0
        for j in range(len(w13)):
            sl = torch.nonzero(se == e_first + j).reshape(-1)
            if sl.numel() == 0:
                continue
            W13, A13 = self.dense(w13[j])
            X = xn[sl // topk].double()
            yy, MM = X @ W13.T, X.abs() @ A13.T
            tol = C_ACC * MM * (1 + 2.0 ** -10) + 2.0 ** -25
            n = sl.numel()
            ya, yb = yy.reshape(n, -1, 2, 8)[:, :, 0].reshape(n, -1), yy.reshape(n, -1, 2, 8)[:, :, 1].reshape(n, -1)
            ta, tb = tol.reshape(n, -1, 2, 8)[:, :, 0].reshape(n, -1), tol.reshape(n, -1, 2, 8)[:, :, 1].reshape(n, -1)
            lo, hi = silu_mul_range(ya, ta, yb, tb)
            got = act[sl, :fe].double()
            ok = (got >= lo) & (got <= hi)
            assert bool(ok.all()), (self.layer, j, "act outside its range", int((~ok).sum()))
            W2, A2 = self.dense(w2[j])
            r, _, _ = gemv_check(y_slot[sl], got @ W2.T, got.abs() @ A2.T, (self.layer, j, "y_slot"))
            worst = max(worst, r)
        off = (se < e_first) | (se >= e_first + len(w13))
        assert not bool(off.any()), "a slot routed off this rank at TP = 1"
        self.note("moe_expert_ffn (y_slot; act in range)", worst)
        return {"act_slots": (ns, fe), "y_slot": ns}

    def check_moe_combine(self, before, y_slot, slot_weight, slot_expert, out, *, T, D, topk, e_first, e_count):
        assert (self.name(y_slot), self.name(slot_weight), self.name(slot_expert), self.name(out)) == (
            self.p("y_slot"), self.p("slot_w"), self.p("slot_e"), self.p("f"))
        if self.tc:
            assert T == self.ctx["T"] and (e_first, e_count) == (self.eng.e_first, self.eng.E_loc)
            self.wrote("p_y_slot", "prefill_moe_gemm_w4")
        acc = torch.zeros(T, D, device=DEV)
        for j in range(topk):
            sl = torch.arange(T, device=DEV) * topk + j
            local = (slot_expert[sl] >= e_first) & (slot_expert[sl] < e_first + e_count)
            prod = (y_slot[sl].float() * slot_weight[sl].float()[:, None]).half().float()
            acc = acc + torch.where(local[:, None], prod, torch.zeros_like(prod))
        assert _same(out[:T], acc.half()), (self.layer, "moe_combine")
        self.delta = self.p("f")
        self.note("moe_combine (tensor-core chunk)" if self.tc else "moe_combine", 0.0)
        return {self.p("f"): T}

    # ------------------------------------------------------------------- the tensor-core prompt path's launches -----
    def check_prefill_rmsnorm(self, before, resid, delta, h_out, gamma, eps, x_out, T, D):
        e, x, c = self.eng, self.ctx, self.eng.cfg
        assert self.tc and T == x["T"] and D == c.dim and eps == c.norm_eps and self.name(x_out) == "p_x"
        # LLaMA: attn_norm, ffn_norm per layer; Mixtral: attn_norm only (its ffn norm is moe_route's prologue)
        per = 2 if c.kind == "llama" else 1
        which = "attn" if self.n_norm % per == 0 else "ffn"
        if which == "attn":
            self.layer += 1
            self.attn_t0 = 0
        else:
            self.wrote("p_o", "prefill_gemm_w4")
        assert self.layer == self.n_norm // per and self.layer < len(e.layers)
        self.n_norm += 1
        lw = e.layers[self.layer]
        assert gamma is (lw.attn_norm if which == "attn" else lw.ffn_norm), (self.layer, which, "gamma")
        h, decl = self._prologue(resid, delta, h_out, T)
        rs = rstd_candidates(h, eps, prefill_rstd_ulps(D))                                   # [T, C] fp32
        X = (h.float()[:, None, :] * rs[:, :, None]).half() * gamma.reshape(1, 1, -1)       # [T, C, D] every candidate x
        hit = (_raw(X) == _raw(x_out[:T])[:, None]).all(-1).any(-1)
        assert bool(hit.all()), (self.layer, which, "x_out is no candidate of the rstd window",
                                 torch.nonzero(~hit).reshape(-1)[:8].tolist())
        self.x_norm = which
        self.note("prefill_rmsnorm", 0.0)
        return dict(decl, p_x=T)

    def check_prefill_gemm_w4(self, before, lin, x_in, out, T, bias=None, bias_mode=None):
        """b200_prefill_gemm_w4, or b200_prefill_gemm_w4_bias with internlm's biases: B200_BIAS_ACC (Wqkv) held to the
        GEMM bound around ref + b; B200_BIAS_OUT (wo) relaunched without the bias to y0, y0 held to the bound and
        out = fp16(y0 + b) bit for bit."""
        e, x = self.eng, self.ctx
        assert self.tc and T == x["T"]
        lw = e.layers[self.layer]
        src, dst = self.name(x_in), self.name(out)
        if lin is lw.wqkv:
            io, producer, kind = ("p_x", "p_qkv"), "prefill_rmsnorm", "wqkv"
            assert self.x_norm == "attn", "wqkv on an x the attention norm did not write"
        elif lin is lw.wo:
            io, producer, kind = ("p_attn", "p_o"), "attn_decode", "wo"
            assert self.attn_t0 == T, ("wo before attention covered the chunk", self.attn_t0, T)
            self.delta = "p_o"
        elif lin is lw.w13:
            io, producer, kind = ("p_x", "p_gu"), "prefill_rmsnorm", "w13"
            assert self.x_norm == "ffn", "w13 on an x the ffn norm did not write"
        else:
            assert lin is lw.w2, "prefill_gemm_w4 of a linear this layer does not have"
            io, producer, kind = ("p_act", "p_f"), "prefill_silu_mul", "w2"
            self.delta = "p_f"
        assert (src, dst) == io, (kind, src, dst)
        self.wrote(src, producer)
        b = self._bias_role(lin, bias, bias_mode)
        X = x_in.view(-1)[:T * lin.K].view(T, lin.K)
        got = out.view(-1)[:T * lin.N].view(T, lin.N)
        if b is not None and bias_mode == ops.B200_BIAS_OUT:
            y0 = torch.empty(T, lin.N, dtype=torch.float16, device=DEV)
            self._relaunch("prefill_gemm_w4", lin, x_in, y0, T)
            assert _same(got, (y0.float() + b.float()[None]).half()), (self.layer, kind, "out != fp16(y0 + b)")
            r = self.gemm_check(y0, X, lin, (self.layer, kind))
        else:
            r = self.gemm_check(got, X, lin, (self.layer, kind), bias=b)
        if self.hidden is not None and kind in ("wo", "w2"):
            # the residual after the block's attention (wo) or after the block (w2), as the next prologue forms it
            h = (self.bufs()[self.resid][:T] + out[:T]).float().cpu()
            for t in range(T):
                self.hidden[(self.start_pos, self.layer, "attn" if kind == "wo" else "block", x["seq"][t], x["off"][t])] = h[t]
        tag = "" if b is None else " BIAS_OUT" if bias_mode == ops.B200_BIAS_OUT else " BIAS_ACC"
        self.note(f"prefill_gemm_w4 ({'fp16' if lin.bits == 16 else f'W{lin.bits}'} {kind}{tag})", r)
        return {dst: ("flat", T * lin.N)}

    def check_prefill_rope_kv(self, before, qkv, q_out, kcache, vtcache, rope, pos, T, n_q_rows, n_kv_rows, tokens_per_seq,
                              cache_seq):
        e, x = self.eng, self.ctx
        i, row0 = self.layer, x["row0"]
        assert self.tc and T == x["T"] and tokens_per_seq == x["tps"] == T and cache_seq == e.cache_seq
        assert (self.name(qkv), self.name(q_out), self.name(pos)) == ("p_qkv", "p_q", "p_pos") and rope is e.rope
        assert (n_q_rows, n_kv_rows) == (e.Hq * 128, e.Hkv * 128)
        assert kcache.data_ptr() == e.kcache[i, row0].data_ptr(), ("K cache slice", i, row0)
        assert vtcache.data_ptr() == e.vtcache[i, row0].data_ptr(), ("V cache slice", i, row0)
        self.wrote("p_qkv", "prefill_gemm_w4")
        q, k, v = qkv_from_y(qkv[:T], e.rope, x["pos"], n_q_rows, n_kv_rows)
        assert _same(q_out[:T], q), (i, "q != RoPE(qkv)")
        self._kv_written(before, [row0] * T, x["pos"], k, v)  # one sequence per chunk: cache row row0
        self.note("prefill_rope_kv", 0.0)
        return dict(p_q=T, kcache="checked", vtcache="checked")

    def check_prefill_silu_mul(self, before, gu, act, T, F):
        e, x, c = self.eng, self.ctx, self.eng.cfg
        assert self.tc and (self.name(gu), self.name(act)) == ("p_gu", "p_act")
        if c.kind == "llama":
            assert (T, F) == (x["T"], e.F)
            self.wrote("p_gu", "prefill_gemm_w4")
        else:
            assert (T, F) == (x["T"] * c.experts_per_tok, e.layers[self.layer].e_w2[0].K)
            self.wrote("p_gu", "prefill_moe_gemm_w4")
        _silu_check(gu.view(-1)[:T * 2 * F].view(T, 2 * F), act.view(-1)[:T * F].view(T, F), (self.layer, "prefill"))
        self.note("prefill_silu_mul", 0.0)
        return {"p_act": ("flat", T * F)}

    def check_prefill_moe_gemm_w4(self, before, experts, x_in, out, *, slot_expert, n_slots, src_div, e_first):
        e, x, c = self.eng, self.ctx, self.eng.cfg
        lw, k = e.layers[self.layer], c.experts_per_tok
        ns = x["T"] * k
        assert self.tc and n_slots == ns and e_first == e.e_first and self.name(slot_expert) == "p_slot_e"
        self.wrote("p_slot_e", "moe_route")
        src, dst = self.name(x_in), self.name(out)
        if experts is lw.e_w13:
            assert (src, dst, src_div) == ("p_x", "p_gu", k), ("w13", src, dst, src_div)
            self.wrote("p_x", "moe_route")
            kind = "w13"
        else:
            assert experts is lw.e_w2, "a grouped GEMM over experts this layer does not have"
            assert (src, dst, src_div) == ("p_act", "p_y_slot", 1), ("w2", src, dst, src_div)
            self.wrote("p_act", "prefill_silu_mul")
            kind = "w2"
        N, K = experts[0].N, experts[0].K
        X = x_in.view(-1)[:((ns - 1) // src_div + 1) * K].view(-1, K)
        O = out.view(-1)[:ns * N].view(ns, N)
        se = slot_expert[:ns].long()
        off = (se < e_first) | (se >= e_first + len(experts))
        assert not bool(off.any()), "a slot routed off this rank at TP = 1"
        worst = 0.0
        for j, pl in enumerate(experts):
            sl = torch.nonzero(se == e_first + j).reshape(-1)
            if sl.numel():
                worst = max(worst, self.gemm_check(O[sl], X[sl // src_div], pl, (self.layer, kind, j)))
        self.note(f"prefill_moe_gemm_w4 ({kind})", worst)
        return {dst: ("flat", ns * N)}

    # ------------------------------------------------------------------------------------------ running ----------
    def run(self, toks, calls):
        """calls: [(start_pos, length)] in order over toks [bsz, *] (CPU)."""
        with self.installed():
            lc0, n0, c0 = ops.launch_count, self.n_engine, self.n_checker
            for sp, n in calls:
                chunk = toks[:, sp:sp + n].contiguous()
                self.expect(chunk, sp)
                assert torch.isfinite(self.eng.forward_inference(chunk.to(DEV), sp)).all()
                assert not self.queue, "forward_inference made fewer _step calls than its schedule"
            checker_launches = ops.launch_count - lc0 - (self.n_engine - n0)
        assert checker_launches == self.n_checker - c0, "a launch outside the audited entry points"

    def run_full(self, toks, forward):
        """forward(tokens) -> [bsz, seqlen, vocab] fp16 through DecodeEngine.forward_full, every launch audited; every
        chunk's rows of the output must equal fp16 of the logits its audited _head launch wrote."""
        with self.installed():
            lc0, n0, c0 = ops.launch_count, self.n_engine, self.n_checker
            self.expect_full(toks)
            out = forward(toks.to(DEV))
            assert not self.queue, "forward_full made fewer _step calls than its schedule"
            checker_launches = ops.launch_count - lc0 - (self.n_engine - n0)
        assert checker_launches == self.n_checker - c0, "a launch outside the audited entry points"
        assert out.shape == (*toks.shape, self.c.vocab_size) and out.dtype == torch.float16
        for e in self.done:
            b0, nb, off, ci = e["row0"], e["nb"], e["off0"], e["ci"]
            assert _same(out[b0:b0 + nb, off:off + ci], e["logits"].reshape(nb, ci, -1).half()), (
                "forward_full: output rows are not the chunk's logits", b0, off)
        self.note("forward_full output rows", 0.0)
        return out

    def report(self, label):
        lines = [f"\n[audit {label}]"]
        for k, (n, w) in sorted(self.stats.items()):
            lines.append(f"  {k:40s} {n:6d} launches, worst err/tol {w:.3f}")
        if self.routed:
            lines.append(f"  tokens routed with two exactly equal gate logits: {self.ties}; routed inside the expf window "
                         f"(not bit for bit): {self.route_window} of {self.routed}")
        lines.append(f"  routing decisions differing from the float64 route of their own input: {len(self.flips)}")
        for f in self.flips:
            lines.append(f"    start {f['start_pos']} layer {f['layer']} seq {f['seq']} pos {f['pos']} ({f['rule']} rule): "
                         f"kernel {f['kernel']} float64 {f['float64']}, float64 score gap {f['gap']:.3e}, fp32 score gap "
                         f"{f['gap32']:.3e}, logit gap {f['logit_gap']:.3e} (window {f['window']:.3e})")
        print("\n".join(lines))
        assert all(w <= 1.0 for _, w in self.stats.values())


# ------------------------------------------------------------------------------------------------ engines -----------
def _mixtral_engine(args, bits, gs, seed=0, tied_gate=False):
    """tied_gate: the router's gate row of every odd expert copies its even neighbour, so every token's logits tie exactly
    in pairs (the lower index must win: kernel_route)."""
    sd = weights.mixtral_state_dict(args, seed=seed)
    if tied_gate:
        for i in range(args["n_layers"]):
            g = sd[f"layers.{i}.feed_forward.gate.weight"]
            g[1::2] = g[0::2]
    recs = omniquant.fake_quantize_state_dict(sd, bits, gs)[1] if bits != 16 else None
    eng = DecodeEngine(EngineConfig.from_model_args("mixtral", args, bits=bits, group_size=gs), DEV)
    eng.load_master_state_dict(sd, quant_records=recs)
    return eng


def _llama_engine(args, bits, gs, seed=0):
    sd = weights.llama_state_dict(args, seed=seed)
    recs = omniquant.fake_quantize_state_dict(sd, bits, gs)[1] if bits != 16 else None
    eng = DecodeEngine(EngineConfig.from_model_args("llama", args, bits=bits, group_size=gs), DEV)
    eng.load_master_state_dict(sd, quant_records=recs)
    return eng


def _eager(eng, tc=False):
    eng.use_graph, eng.use_prefill_tc = False, tc
    return eng


def _calls(p0, p1, ndec):
    return [(0, p0)] + ([(p0, p1)] if p1 else []) + [(p0 + p1 + j, 1) for j in range(ndec)]


def audit_schedule(eng, bsz, calls, label, seed=11, tc=False, toks=None):
    """Run `calls` eagerly with every launch audited -> the Audit.  tc = False: the GEMV-chunk path only; tc = True: the
    engine's own choice between the tensor-core prompt path and the GEMV chunks."""
    end = max(sp + n for sp, n in calls)
    if toks is None:
        toks = weights.synthetic_tokens(bsz, end, eng.cfg.vocab_size, seed=seed)
    a = Audit(_eager(eng, tc))
    a.run(toks, calls)
    a.report(label)
    return a


def _paths(a):
    """[(path, T)] of every _step / _prefill_chunk_tc call an audited run made."""
    return [("tc" if e.get("tc") else "gemv", e["T"]) for e in a.done]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("p0,p1", [(5, 40), (100, 200), (40, 300), (250, 33)])
def test_tiny_mixtral_w4_continuation(p0, p1):
    """Batch 2 (t_max 16: 8 tokens per sequence per chunk), a p0-token prompt, a p1-token continuation, 2 decode steps."""
    args = dict(cases.TINY_MIXTRAL, max_seq_len=640)
    audit_schedule(_mixtral_engine(args, 4, 0), 2, _calls(p0, p1, 2), f"tiny mixtral w4 bsz 2 ({p0}, {p1})")


@pytest.mark.timeout(300)
def test_tiny_mixtral_w4_tied_gate_rows():
    """Experts 2i and 2i + 1 share a gate row: every router launch breaks exact ties, and must give them to the lower
    index, as mixtral.py's torch.topk does (kernel_route).  A prompt of 20, a 20-token continuation, 2 decode steps."""
    args = dict(cases.TINY_MIXTRAL, max_seq_len=64)
    a = audit_schedule(_mixtral_engine(args, 4, 0, tied_gate=True), 2, _calls(20, 20, 2), "tiny mixtral w4 tied gate rows")
    assert a.routed > 0 and a.ties == a.routed, (a.ties, a.routed)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("bits,gs", [(16, 0), (4, 128), (3, 0)], ids=["fp16", "w4_g128", "w3"])
def test_tiny_mixtral_gemv_only_codecs(bits, gs):
    """The codecs whose Mixtral prompts never take the tensor cores: prompt 40, a 60-token continuation, 2 decode steps."""
    args = dict(cases.TINY_MIXTRAL, max_seq_len=128)
    audit_schedule(_mixtral_engine(args, bits, gs), 2, _calls(40, 60, 2), f"tiny mixtral bits {bits} gs {gs}")


@pytest.mark.timeout(300)
@pytest.mark.parametrize("kind,bsz", [("mixtral", 17), ("llama", 34)])
def test_batches_above_t_max(kind, bsz):
    """Sequence groups at row0 > 0, and (Mixtral, t_max 16) a last group of one sequence: T = 1 launches."""
    if kind == "mixtral":
        eng = _mixtral_engine(dict(cases.TINY_MIXTRAL, max_seq_len=64), 4, 0)
    else:
        eng = _llama_engine(dict(cases.TINY_LLAMA, max_seq_len=64), 4, 0)
    audit_schedule(eng, bsz, _calls(6, 0, 2), f"tiny {kind} w4 bsz {bsz}")


@pytest.mark.timeout(300)
def test_tiny_llama_chunk_not_dividing_32():
    """Batch 5: ci = 6, T = 30, so one GEMV token group holds the tail of one sequence and the head of the next."""
    eng = _llama_engine(dict(cases.TINY_LLAMA, max_seq_len=64), 4, 0)
    audit_schedule(eng, 5, _calls(13, 0, 2), "tiny llama w4 bsz 5")


@pytest.mark.timeout(600)
def test_real_widths_one_layer():
    """Mixtral-8x7B width, W4-g128, batch 2, a 24-token prompt and 2 decode steps; LLaMA-2-7B width, W3, batch 3, a
    20-token prompt and 1 decode step.  Random packed weights (engine.load_random), one layer each."""
    torch.cuda.empty_cache()
    eng = DecodeEngine(EngineConfig.from_model_args("mixtral", MIXTRAL_WIDTH, bits=4, group_size=128), DEV).load_random(3)
    a = audit_schedule(eng, 2, _calls(24, 0, 2), "mixtral width w4 g128 bsz 2")
    del eng, a
    torch.cuda.empty_cache()
    cfg = EngineConfig(kind="llama", dim=4096, n_layers=1, n_heads=32, ffn_hidden=11008, vocab_size=4096, max_seq_len=64,
                       bits=3, group_size=0)
    eng = DecodeEngine(cfg, DEV).load_random(4)
    audit_schedule(eng, 3, _calls(20, 0, 1), "llama-2-7b width w3 bsz 3")
    del eng
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------- the tensor-core prompt path ---------
def _tc_paths(a, want):
    """The run took exactly the restated paths `want` ([(path, T)])."""
    assert _paths(a) == want, _paths(a)


@pytest.mark.timeout(600)
def test_tiny_llama_w4_tensor_core_prompts():
    """Batch 3, per-channel W4: a 300-token prompt (chunks of 256 + 44 per sequence, cache rows 0 to 2), GEMV
    continuations of 20 and 30 tokens that read the K / V the tensor-core chunks wrote, a 40-token tensor-core
    continuation at positions 350-389 (across the 384 boundary: max_kv_len 512) that reads K / V of both paths, and 2
    decode steps."""
    eng = _llama_engine(dict(cases.TINY_LLAMA, max_seq_len=512), 4, 0)
    a = audit_schedule(eng, 3, [(0, 300), (300, 20), (320, 30), (350, 40), (390, 1), (391, 1)],
                       "tiny llama w4 bsz 3 tc", tc=True)
    _tc_paths(a, [("tc", 256), ("tc", 44)] * 3 + [("gemv", 30)] * 5 + [("tc", 40)] * 3 + [("gemv", 3)] * 2)
    assert [e["kv"] for e in a.done if e.get("tc") and e["T"] == 40] == [512] * 3


@pytest.mark.timeout(600)
@pytest.mark.parametrize("bits", [3, 16], ids=["w3", "fp16"])
def test_tiny_llama_codec_tensor_core_prompts(bits):
    """W3: 48 tokens (its shortest tensor-core prompt), 47 on the GEMV chunks, 100 on the tensor cores (positions 95-194,
    across the 128 boundary), 2 decode steps.  fp16: 33 (tensor cores), 32 (GEMV), 257 (256 + a last chunk of one token:
    the GEMM at T = 1), 2 decode steps.  Batch 2."""
    eng = _llama_engine(dict(cases.TINY_LLAMA, max_seq_len=384), bits, 0)
    if bits == 3:
        calls, want = [(0, 48), (48, 47), (95, 100)], [("tc", 48)] * 2 + [("gemv", 32)] * 2 + [("gemv", 30)] + [("tc", 100)] * 2
    else:
        calls, want = [(0, 33), (33, 32), (65, 257)], [("tc", 33)] * 2 + [("gemv", 32)] * 2 + [("tc", 256), ("tc", 1)] * 2
    end = calls[-1][0] + calls[-1][1]
    calls += [(end, 1), (end + 1, 1)]
    a = audit_schedule(eng, 2, calls, f"tiny llama bits {bits} tc", tc=True)
    _tc_paths(a, want + [("gemv", 2)] * 2)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("p0,p1", [(5, 40), (250, 33), (40, 300)])
def test_tiny_mixtral_w4_tensor_core_prompts(p0, p1):
    """Batch 2, a p0-token prompt, a p1-token continuation (every one of them over 32 tokens on the tensor cores: one
    grouped GEMM per projection over the routed experts), 2 decode steps.  (40, 300) is the schedule the GEMV path misses
    the port rule on by routing flips."""
    args = dict(cases.TINY_MIXTRAL, max_seq_len=640)
    a = audit_schedule(_mixtral_engine(args, 4, 0), 2, _calls(p0, p1, 2), f"tiny mixtral w4 bsz 2 tc ({p0}, {p1})", tc=True)
    assert ("tc", min(p1, 256)) in _paths(a)


@pytest.mark.timeout(600)
def test_tiny_mixtral_w4_tied_gate_rows_tensor_core():
    """Tied gate rows (test_tiny_mixtral_w4_tied_gate_rows) through the tensor-core path: one router launch over a
    256-token chunk breaks an exact tie for every token.  A 260-token prompt, batch 2, 1 decode step."""
    args = dict(cases.TINY_MIXTRAL, max_seq_len=320)
    a = audit_schedule(_mixtral_engine(args, 4, 0, tied_gate=True), 2, _calls(260, 0, 1), "tiny mixtral tied gate tc",
                       tc=True)
    _tc_paths(a, [("tc", 256), ("tc", 4)] * 2 + [("gemv", 2)])
    assert a.routed > 0 and a.ties == a.routed, (a.ties, a.routed)


def _band_report(label, a, rec32, rec16, calls, bsz, n_layers):
    """The residual-band comparison of test_prefill_moe_gpu._locate_excess, after the attention and after every block:
    the engine's residual against the fp32 port's, in units of the fp16 port's own distance from it (below BAND_ABS
    ignored).  Prints the first residual, in the tensor-core path's order (call, sequence, layer, stage, position), to
    leave the band by BAND_FACTOR, and the largest ratio of every (layer, stage) -> that first exit or None."""
    first, worst = None, {}
    for c, (sp, n) in enumerate(calls):
        for b in range(bsz):
            for i in range(n_layers):
                for stage, key in (("attn", "h_attn"), ("block", "h")):
                    for o in range(n):
                        h32, h16 = rec32[c][key][i][b, o].float(), rec16[c][key][i][b, o].float()
                        d_e = float((a.hidden[(sp, i, stage, b, o)] - h32).abs().max())
                        d_16 = float((h16 - h32).abs().max())
                        r = d_e / max(d_16, BAND_ABS)
                        if r > worst.get((i, stage), (0.0,))[0]:
                            worst[(i, stage)] = (r, sp + o, b, d_e, d_16)
                        if first is None and r > BAND_FACTOR:
                            first = (sp + o, b, i, stage, d_e, d_16)
    for (i, stage), (r, pos, b, d_e, d_16) in sorted(worst.items()):
        print(f"[{label}] layer {i} after {stage}: largest |eng-port32| / max(|port16-port32|, 2^-9) {r:.2f} at position "
              f"{pos}, sequence {b} ({d_e:.3e} against {d_16:.3e})")
    print(f"[{label}] first residual outside {BAND_FACTOR} x the band: " + (
        "none" if first is None else "position {}, sequence {}, layer {}, after {}: {:.3e} against {:.3e}".format(*first)))
    return first


@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", ["llama_w3", "llama_fp16", "llama_w4", "mixtral_w4"])
def test_force_tc_golden_schedules(name):
    """B200_FORCE_TC on the golden schedules (cases.CASES): every forward_inference call, single-token steps too, through
    _prefill_chunk_tc, every launch audited.  The logits meet the rule of
    test_prefill_codecs_gpu.test_every_linear_on_tensor_cores_meets_strict_rule_on_golden against the golden references
    (its MAX_FACTOR, the suite's 1.5 where it has none).  For LLaMA the engine's residual stream is compared with the
    port's fp16 / fp32 band after every attention and every block (_band_report), and the largest logit error is split
    into what the last residual carries and what the head adds (DESIGN.md 4.6, the W3 finding)."""
    from test_prefill_codecs_gpu import MAX_FACTOR
    kind, args, bits, gs, bsz, plen, ndec = cases.CASES[name]
    kind, args, sd, sd_ref, recs, toks = cases.build_case(name)
    eng = DecodeEngine(EngineConfig.from_model_args(kind, args, bits=bits or 16, group_size=gs), DEV)
    eng.load_master_state_dict(sd, quant_records=recs if bits else None)
    eng.force_tc = True
    got = []
    real_fi = eng.forward_inference

    def fi(tokens, start_pos):
        out = real_fi(tokens, start_pos)
        got.append(out.float().cpu().clone())
        return out
    eng.forward_inference = fi
    calls = _calls(plen, 0, ndec)
    a = Audit(_eager(eng, True))
    a.hidden = {}
    a.run(toks, calls)
    a.report(f"{name} force_tc")
    _tc_paths(a, [("tc", plen)] * bsz + [("tc", 1)] * (bsz * ndec))
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"{name}.npz"))
    ref16, ref32 = g["logits_fp16"], g["logits_fp32"]
    got = torch.stack(got).numpy()
    e16, e32, floor = np.abs(got - ref16).max(), np.abs(got - ref32).max(), np.abs(ref16 - ref32).max()
    c, b, v = np.unravel_index(np.abs(got - ref32).argmax(), got.shape)
    print(f"[{name} force_tc] |eng-ref32| = {e32:.3e} = {e32 / floor:.3f} x floor {floor:.3e}; largest at call {c}, "
          f"sequence {b}, logit {v}: engine {got[c, b, v]:.5f}, fp32 {ref32[c, b, v]:.5f}, fp16 {ref16[c, b, v]:.5f}; "
          f"that row's floor {np.abs(ref16[c, b] - ref32[c, b]).max():.3e}")
    assert np.isfinite(got).all()
    assert e16 <= 1e-3 or e32 <= MAX_FACTOR.get(name, 1.5) * floor, (e16, e32, floor)
    if kind == "llama":
        port = {}
        for dt in (torch.float32, torch.float16):
            port[dt] = PortModel(kind, args, sd_ref, dtype=dt)
            port[dt].record = []
            cases.run_schedule(port[dt], toks, plen, ndec)
        rec32, rec16 = port[torch.float32].record, port[torch.float16].record
        _band_report(f"{name} force_tc", a, rec32, rec16, calls, bsz, args["n_layers"])
        # the largest logit error split into what the final residual carries and what the head adds: the float64 head
        # (final RMSNorm and lm_head without any rounding) of the engine's and of both ports' last residual of that row
        sp, n = calls[c]
        L = args["n_layers"]
        W = _w_hat(eng.lm_head)[v].double()
        gamma = eng.final_norm.double()

        def head64(h):
            h = h.double().to(DEV)
            return float((h * gamma / torch.sqrt(h.pow(2).mean() + eng.cfg.norm_eps)) @ W)
        hs = dict(engine=a.hidden[(sp, L - 1, "block", b, n - 1)], port16=rec16[c]["h"][L - 1][b, n - 1],
                  port32=rec32[c]["h"][L - 1][b, n - 1])
        print(f"[{name} force_tc] that logit from the float64 head of each last residual: " + ", ".join(
            f"{k} {head64(h):.5f}" for k, h in hs.items()) + "; |engine - port16| of the residual "
            f"{float((hs['engine'].float() - hs['port16'].float()).abs().max()):.3e}")


def _llama_cfg(dim, n_heads, n_kv_heads, ffn, bits, max_seq_len):
    return EngineConfig(kind="llama", dim=dim, n_layers=1, n_heads=n_heads, n_kv_heads=n_kv_heads, ffn_hidden=ffn,
                        vocab_size=2048, max_seq_len=max_seq_len, bits=bits, group_size=0)


REAL_TC = {
    # name: (config, batch, prompt)
    "llama2_7b_w4": (lambda: _llama_cfg(4096, 32, None, 11008, 4, 320), 2, 300),
    "llama2_7b_w3": (lambda: _llama_cfg(4096, 32, None, 11008, 3, 288), 1, 257),   # w2: K 11008 ends in a 48-k block
    "llama2_13b_fp16": (lambda: _llama_cfg(5120, 40, None, 13824, 16, 96), 1, 64),
    # LLaMA-2-70B's D = 8192 norm depth and 64 / 8 heads; its FFN of 28672 is above the kernels' local limit of 16384 at
    # TP = 1, so the FFN is one rank's 14336 at TP = 2
    "llama2_70b_w4": (lambda: _llama_cfg(8192, 64, 8, 14336, 4, 64), 1, 40),
    "mixtral_8x7b_w4": (lambda: EngineConfig.from_model_args("mixtral", dict(MIXTRAL_WIDTH, max_seq_len=288), bits=4,
                                                             group_size=0), 1, 260),  # 512 slot rows in the first chunk
}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", list(REAL_TC))
def test_real_widths_tensor_core_one_layer(name):
    """One layer at real width, random packed weights (engine.load_random), a tensor-core prompt and 1 decode step."""
    make, bsz, plen = REAL_TC[name]
    torch.cuda.empty_cache()
    eng = DecodeEngine(make(), DEV).load_random(5)
    a = audit_schedule(eng, bsz, _calls(plen, 0, 1), f"{name} tc", tc=True)
    chunks = [min(256, plen - o) for o in range(0, plen, 256)]
    _tc_paths(a, [("tc", c) for c in chunks] * bsz + [("gemv", bsz)])
    del eng, a
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ forward_full --------
@pytest.mark.timeout(600)
@pytest.mark.parametrize("bsz,seqlen", [(3, 70), (34, 4)])
def test_forward_full_tiny_llama_w4(bsz, seqlen):
    """DecodeEngine.forward_full (Transformer.forward, MetaModel.compute_logits): the GEMV chunks with the logits of every
    row; batch 34 runs in sequence groups of 32 and 2 (t_max 32)."""
    eng = _eager(_llama_engine(dict(cases.TINY_LLAMA, max_seq_len=96), 4, 0))
    toks = weights.synthetic_tokens(bsz, seqlen, eng.cfg.vocab_size, seed=13)
    a = Audit(eng)
    a.run_full(toks, eng.forward_full)
    a.report(f"forward_full tiny llama w4 {bsz} x {seqlen}")


@pytest.mark.timeout(600)
def test_forward_full_tiny_mixtral_w4_dropin():
    """mixtral_b200.Transformer.forward -> (logits, {}) over batch 2 x 40 tokens, every launch audited."""
    from llama2_accessory_b200.model import mixtral_b200
    from test_dropin_gpu import _model
    args = dict(cases.TINY_MIXTRAL, max_seq_len=64)
    m = _model(mixtral_b200, args, weights.mixtral_state_dict(args, seed=0), 4, 0)
    eng = _eager(m.build_engine())
    toks = weights.synthetic_tokens(2, 40, args["vocab_size"], seed=13)

    def forward(t):
        out, aux = m.forward(t)
        assert aux == {}
        return out
    a = Audit(eng)
    a.run_full(toks, forward)
    a.report("forward_full tiny mixtral w4 drop-in 2 x 40")
