"""GPU: every launch DecodeEngine.forward_inference makes on the GEMV-chunk path, audited one at a time on the engine's own
buffers against float64.

The kernel modules test each kernel on inputs the test allocates; this module tests the glue between them.  The `ops`
entry points the engine calls (and the engine's `_step` and `_allreduce`) are wrapped.  For every launch the wrapper
synchronises, clones what the launch reads and snapshots every engine buffer (h[0], h[1], q, attn, o, f, act, xn, slot_w,
slot_e, act_slots, y_slot, logits_loc, kcache, vtcache, counters), runs the real launch, synchronises, and checks the
launch against float64 computed from its own inputs.  The inputs are teacher-forced, so an error is the launch's own.

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
  attn_decode      the float64 bound of test_attn_decode_gpu.py on the cache rows of the chunk's sequences; counters back
                   at zero
  moe_route        h_out bit for bit, xn_out one candidate, slot_expert / slot_weight a kernel_route outcome of the logit
                   window of its own xn_out (section B)
  moe_expert_ffn   section B ranges for act and the bound for y_slot, on every slot routed to a local expert
  moe_combine      bit for bit
  _head            the F32 bound, and its rows are the last token of every sequence (or every row of a decode step)
Every launch: no engine buffer changes outside the output elements its checker verified (the declared rows, and within
them the declared columns), and a launch kind without a checker fails.

The module also prints, per launch kind, the launches audited and the worst err / tol, and every routing decision that
differs from the route of the float64 logits of its own input, with the float64 score gap of the experts involved.
"""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import _cabi, kvlayout, ops, quant  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig  # noqa: E402
from oracle import cases, omniquant, weights  # noqa: E402
from oracle.numerics import (C_ACC, SILU_REL, TUNE_DEFAULTS, AttnRef, attn_host_split, fp16_sides,  # noqa: E402
                             gemv_check, gemv_tol, kernel_route, logit_window, qkv_from_y, route_check,
                             silu_mul_range, x_candidates)

DEV = "cuda"
BUFS = ("h0", "h1", "q", "attn", "o", "f", "act", "xn", "slot_w", "slot_e", "act_slots", "y_slot", "logits_loc",
        "kcache", "vtcache", "counters")
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
        self.queue, self.ctx = [], None
        self.layer, self.resid, self.delta = -1, None, None
        self.n_engine = 0          # launch_count increments inside audited engine launches
        self.start_pos = 0
        self.even = int(os.environ.get("B200_ATTN_EVEN", TUNE_DEFAULTS["B200_ATTN_EVEN"]))

    # ------------------------------------------------------------------------------------------ plumbing ---------
    def bufs(self):
        e = self.eng
        out = dict(h0=e.h[0], h1=e.h[1])
        for n in BUFS[2:]:
            t = getattr(e, n, None)
            if t is not None:
                out[n] = t
        return out

    def name(self, t):
        if t is None:
            return None
        for n, b in self.bufs().items():
            if t.data_ptr() == b.data_ptr() and t.dtype == b.dtype:
                return n
        return "other"

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
        assert {"embed", "gemv", "attn_decode", "moe_route", "moe_expert_ffn", "moe_combine"} <= set(names), names
        for n in names:
            self.real[n] = getattr(ops, n)
            setattr(ops, n, self._wrap(n, self.real[n]))
        real_step, eng = self.eng._step, self.eng
        eng._step = self._step_wrapper(real_step)
        eng._allreduce = self._allreduce
        try:
            yield self
        finally:
            for n in names:
                setattr(ops, n, self.real[n])
            del eng._step, eng._allreduce

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
            declared = check(before, *a, **kw)
            self.no_stray_writes(kind, before, declared)
        return launch

    def no_stray_writes(self, kind, before, declared):
        """declared: name -> n (rows [0, n) verified whole by the checker), (n, c) (only columns [0, c) of those rows
        verified: the rest of the rows must keep their bytes) or 'checked' (the whole buffer verified by the checker)."""
        for n, b in self.bufs().items():
            d = declared.get(n, 0)
            if d == "checked":
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
        assert self.name(t) in ("o", "f")
        self.no_stray_writes("allreduce", before, {})
        self.note("allreduce (TP = 1: no-op)", 0.0)

    def expect(self, toks, start_pos):
        """The _step calls forward_inference must make for tokens [bsz, seqlen] at start_pos (engine.py, GEMV path)."""
        e = self.eng
        bsz, seqlen = toks.shape
        tm, S = e.t_max, e.cache_seq
        self.start_pos = start_pos
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

    def _step_wrapper(self, real):
        def step(T, tokens_per_seq, max_kv_len, row0=0, want_logits=True, last_rows=None):
            assert self.queue, "a _step the schedule does not call for"
            e = self.queue.pop(0)
            rows = None if last_rows is None else last_rows.tolist()
            got = dict(T=T, tps=tokens_per_seq, kv=max_kv_len, row0=row0, want=want_logits, rows=rows)
            assert got == {k: e[k] for k in got}, ("_step arguments", got, {k: e[k] for k in got})
            self.ctx, self.layer = e, -1
            return real(T, tokens_per_seq, max_kv_len, row0=row0, want_logits=want_logits, last_rows=last_rows)
        return step

    # ------------------------------------------------------------------------------------------- checkers --------
    def check_embed(self, before, tokens, table, h, T, D, vocab):
        e, x = self.eng, self.ctx
        assert self.name(h) == "h0" and tokens.data_ptr() == e.tokens.data_ptr()
        assert T == x["T"] and torch.equal(e.tokens[:T].cpu(), x["tok"].cpu()), "tokens staged for the chunk"
        assert e.pos[:T].tolist() == x["pos"], "positions staged for the chunk"
        assert _same(h[:T], table[tokens[:T]]), "embed rows"
        self.resid, self.delta, self.layer = "h0", None, -1
        self.note("embed", 0.0)
        return {"h0": T}

    def _prologue(self, resid, delta, h_out, T):
        """The residual stream of an RMSNorm prologue: -> (h [T, K] the normalised rows, declared h_out rows)."""
        b = self.bufs()
        assert self.name(resid) == self.resid, ("resid", self.name(resid), self.resid)
        assert self.name(delta) == self.delta, ("delta", self.name(delta), self.delta)
        if delta is None:
            assert h_out is None
            return resid[:T].clone(), {}
        other = "h1" if self.resid == "h0" else "h0"
        assert self.name(h_out) == other, ("h_out", self.name(h_out))
        h = resid[:T] + delta[:T]
        assert _same(h_out[:T], h), (self.layer, "h_out != fp16(resid + delta)")
        self.resid = other
        return b[other][:T].clone(), {other: T}

    def _y_bound(self, y, h, gamma, eps, pl):
        """y [T, N] (fp16 or fp32) against float64 for the best rstd candidate of every row -> worst err / tol."""
        W, A = self.dense(pl)
        worst = 0.0
        for t in range(y.shape[0]):
            X = x_candidates(h[t], gamma, eps).double()
            Y, M = X @ W.T, X.abs() @ A.T
            r = ((y[t].double()[None] - Y).abs() / gemv_tol(Y, M)).amax(1)
            worst = max(worst, float(r.min()))
        assert worst <= 1.0, (self.layer, pl.N, pl.K, worst)
        return worst

    def _f16_relaunch(self, pl, T, resid, delta, gamma, eps):
        y = torch.empty(T, pl.N, dtype=torch.float16, device=DEV)
        n0 = ops.launch_count
        self.real["gemv"](pl, T, out=y, epilogue=ops.B200_EPI_F16, resid=resid, delta=delta, gamma=gamma, eps=eps)
        torch.cuda.synchronize()
        assert ops.launch_count == n0 + 1
        return y

    def check_gemv(self, before, lin, T, *, out, epilogue=ops.B200_EPI_F16, xin=None, resid=None, delta=None, h_out=None,
                   gamma=None, eps=1e-5, qkv=None, moe=None, **kw):
        e, x = self.eng, self.ctx
        assert moe is None and kw.get("ar") is None, "moe-slot / fused all-reduce gemv: no checker"
        if epilogue == ops.B200_EPI_QKV:
            return self._check_qkv(before, lin, T, out, resid, delta, h_out, gamma, eps, qkv)
        if epilogue == ops.B200_EPI_SILU:
            assert self.c.kind == "llama" and lin is e.layers[self.layer].w13 and self.name(out) == "act"
            rb, db = resid.clone(), delta.clone()
            h, decl = self._prologue(resid, delta, h_out, T)
            y = self._f16_relaunch(lin, T, rb, db, gamma, eps)
            r = self._y_bound(y, h, gamma, eps, lin)
            t = y.reshape(T, lin.N // 16, 2, 8)
            a, b = t[:, :, 0].reshape(T, -1).double(), t[:, :, 1].reshape(T, -1).double()
            sl = a / (1 + torch.exp(-a))
            sn, sa, sd = fp16_sides(sl)
            amb = sd <= SILU_REL * sl.abs()
            got = out[:T, :lin.N // 2].double()
            ok = (got == (sn * b).half().double()) | (amb & (got == (sa * b).half().double()))
            assert bool(ok.all()), (self.layer, "silu", int((~ok).sum()))
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
        W, A = self.dense(lin)
        xd = xin[:T, :lin.K].double()
        r, _, _ = gemv_check(out[:T], xd @ W.T, xd.abs() @ A.T, (kind, self.layer))
        self.note(kind, r)
        return {dst: T}

    def _check_qkv(self, before, lin, T, out, resid, delta, h_out, gamma, eps, qkv):
        e, x = self.eng, self.ctx
        self.layer += 1
        i, row0, tps = self.layer, x["row0"], x["tps"]
        lw = e.layers[i]
        assert lin is lw.wqkv and gamma is lw.attn_norm and self.name(out) == "q"
        assert qkv["tokens_per_seq"] == tps and qkv["pos"].data_ptr() == e.pos.data_ptr() and qkv["rope"] is e.rope
        assert qkv["kcache"].data_ptr() == e.kcache[i, row0].data_ptr(), ("K cache slice", i, row0)
        assert qkv["vtcache"].data_ptr() == e.vtcache[i, row0].data_ptr(), ("V cache slice", i, row0)
        rb, db = resid.clone(), None if delta is None else delta.clone()
        h, decl = self._prologue(resid, delta, h_out, T)
        y = self._f16_relaunch(lin, T, rb, db, gamma, eps)
        r = self._y_bound(y, h, gamma, eps, lin)
        nq, nkv = qkv["n_q_rows"], qkv["n_kv_rows"]
        pos = x["pos"]
        q, k, v = qkv_from_y(y, e.rope, pos, nq, nkv)
        assert _same(out[:T], q), (i, "q != RoPE(y)")
        kc = kvlayout.k_from_engine(before["kcache"][i])
        vc = kvlayout.v_from_engine(before["vtcache"][i])
        for t in range(T):
            b = row0 + t // tps
            kc[b, :, pos[t]] = k[t].view(-1, 128)
            vc[b, :, pos[t]] = v[t].view(-1, 128)
        kexp, vexp = before["kcache"].clone(), before["vtcache"].clone()
        kexp[i], vexp[i] = kvlayout.k_to_engine(kc), kvlayout.v_to_engine(vc)
        assert _same(e.kcache, kexp), (i, row0, "K cache: a slot other than (row0 + t // tps, pos[t]) or a wrong value")
        assert _same(e.vtcache, vexp), (i, row0, "V cache: a slot other than (row0 + t // tps, pos[t]) or a wrong value")
        self.note("gemv QKV", r)
        return dict(decl, q=T, kcache="checked", vtcache="checked")

    def check_attn_decode(self, before, q, kcache, vtcache, pos, out, *, T, Hq, Hkv, cache_seq, tokens_per_seq, max_kv_len,
                          ws=None, counters=None, n_split=0, **kw):
        e, x = self.eng, self.ctx
        i, row0 = self.layer, x["row0"]
        assert (self.name(q), self.name(out), self.name(counters)) == ("q", "attn", "counters")
        assert pos.data_ptr() == e.pos.data_ptr() and T == x["T"] and tokens_per_seq == x["tps"]
        assert max_kv_len == x["kv"] and (Hq, Hkv, cache_seq) == (e.Hq, e.Hkv, e.cache_seq)
        assert kcache.data_ptr() == e.kcache[i, row0].data_ptr() and vtcache.data_ptr() == e.vtcache[i, row0].data_ptr()
        nseq = -(-T // tokens_per_seq)
        kc = kvlayout.k_from_engine(kcache[:nseq])
        vc = kvlayout.v_from_engine(vtcache[:nseq])
        ref = AttnRef(q[:T].view(T, Hq, 128), kc, vc, x["pos"], tokens_per_seq)
        n_launched, chunk = attn_host_split(max_kv_len, n_split)
        r = ref.ratio(out[:T].view(T, Hq, 128), n_launched, chunk, self.even)
        assert r <= 1.0, (i, "attention", r)
        assert int(counters.abs().sum()) == 0, "attention counters not reset"
        self.note("attn_decode", r)
        return {"attn": T}

    def check_moe_route(self, before, *, T, D, E, topk, resid, delta, h_out, gamma, eps, gate_w, xn_out, slot_weight,
                        slot_expert, **kw):
        e, x = self.eng, self.ctx
        i, k = self.layer, topk
        lw = e.layers[i]
        assert gate_w is lw.gate and gamma is lw.ffn_norm
        assert (self.name(xn_out), self.name(slot_weight), self.name(slot_expert)) == ("xn", "slot_w", "slot_e")
        h, decl = self._prologue(resid, delta, h_out, T)
        xn = xn_out[:T]
        for t in range(T):
            X = x_candidates(h[t], gamma, eps)
            assert bool((_raw(X) == _raw(xn[t])[None]).all(1).any()), (i, t, "xn_out is no candidate of the rstd window")
        se, sw = slot_expert[:T * k].view(T, k), slot_weight[:T * k].view(T, k)
        matched, window, skipped = route_check(xn, gate_w, sw, se, k)
        assert skipped == 0 and matched + window == T
        # the float64 route of the same input: logits rounded to nearest fp16, then the kernel's routing rule
        L, R = logit_window(xn, gate_w)
        near = fp16_sides(L)[0]
        idx64, _ = kernel_route(near.half().cpu(), k)
        p64 = torch.softmax(L, -1).cpu()
        se_c = se.cpu().long()
        for t in torch.nonzero((idx64 != se_c).any(1)).reshape(-1).tolist():
            j = int(torch.nonzero(idx64[t] != se_c[t])[0])
            a, b = int(se_c[t, j]), int(idx64[t, j])
            self.flips.append(dict(start_pos=self.start_pos, layer=i, seq=x["seq"][t], pos=x["pos"][t],
                                   kernel=se_c[t].tolist(), float64=idx64[t].tolist(),
                                   gap=float(p64[t, a] - p64[t, b]), logit_gap=float(L[t, a] - L[t, b]),
                                   window=float(R[t, a] + R[t, b])))
        Lc = L.cpu()
        self.ties += sum(int(Lc[t].unique().numel() < Lc.shape[1]) for t in range(T))
        self.routed += T
        self.note("moe_route", 0.0)
        return dict(decl, xn=T, slot_w=T * k, slot_e=T * k)

    def check_moe_expert_ffn(self, before, w13, w2, *, T, D, F, topk, e_first, xn, slot_expert, act, y_slot, **kw):
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
            "y_slot", "slot_w", "slot_e", "f")
        acc = torch.zeros(T, D, device=DEV)
        for j in range(topk):
            sl = torch.arange(T, device=DEV) * topk + j
            local = (slot_expert[sl] >= e_first) & (slot_expert[sl] < e_first + e_count)
            prod = (y_slot[sl].float() * slot_weight[sl].float()[:, None]).half().float()
            acc = acc + torch.where(local[:, None], prod, torch.zeros_like(prod))
        assert _same(out[:T], acc.half()), (self.layer, "moe_combine")
        self.delta = "f"
        self.note("moe_combine", 0.0)
        return {"f": T}

    # ------------------------------------------------------------------------------------------ running ----------
    def run(self, toks, calls):
        """calls: [(start_pos, length)] in order over toks [bsz, *] (CPU)."""
        with self.installed():
            lc0, n0 = ops.launch_count, self.n_engine
            for sp, n in calls:
                chunk = toks[:, sp:sp + n].contiguous()
                self.expect(chunk, sp)
                assert torch.isfinite(self.eng.forward_inference(chunk.to(DEV), sp)).all()
                assert not self.queue, "forward_inference made fewer _step calls than its schedule"
            checker_launches = ops.launch_count - lc0 - (self.n_engine - n0)
        assert checker_launches == self.stats.get("gemv QKV", [0])[0] + self.stats.get("gemv SILU (w13)", [0])[0], \
            "a launch outside the audited entry points"

    def report(self, label):
        lines = [f"\n[audit {label}]"]
        for k, (n, w) in sorted(self.stats.items()):
            lines.append(f"  {k:40s} {n:6d} launches, worst err/tol {w:.3f}")
        if "moe_route" in self.stats:
            lines.append(f"  tokens routed with two exactly equal gate logits: {self.ties}")
        lines.append(f"  routing decisions differing from the float64 route of their own input: {len(self.flips)}")
        for f in self.flips:
            lines.append(f"    start {f['start_pos']} layer {f['layer']} seq {f['seq']} pos {f['pos']}: kernel {f['kernel']} "
                         f"float64 {f['float64']}, float64 score gap {f['gap']:.3e}, logit gap {f['logit_gap']:.3e} "
                         f"(window {f['window']:.3e})")
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


def _eager(eng):
    eng.use_graph, eng.use_prefill_tc = False, False
    return eng


def _calls(p0, p1, ndec):
    return [(0, p0)] + ([(p0, p1)] if p1 else []) + [(p0 + p1 + j, 1) for j in range(ndec)]


def audit_schedule(eng, bsz, calls, label, seed=11):
    """Run `calls` on the eager GEMV-chunk path with every launch audited -> the Audit."""
    end = max(sp + n for sp, n in calls)
    toks = weights.synthetic_tokens(bsz, end, eng.cfg.vocab_size, seed=seed)
    a = Audit(_eager(eng))
    a.run(toks, calls)
    a.report(label)
    return a


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
