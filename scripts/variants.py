"""One process, many tuning variants of the bs = 1 decode step (LLaMA2-7B W4 ctx 2048): tokens/s of the graph-replayed greedy
loop per variant and, for variants flagged `tl`, the in-kernel %globaltimer timeline of layer 15.
Usage: python scripts/variants.py [spec-file]   (spec = python list of (label, {knob: value}, want_timeline))"""
import os, sys, json, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import torch
import llama2_accessory_b200 as pkg
pkg.build()
from llama2_accessory_b200 import _cabi
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig

DEFAULTS = {"B200_PF_KB": 96, "B200_PF_KV": 1, "B200_SELF_PF_KB": 0, "B200_PF_EARLY": 0, "B200_ATTN_MAX_SPLIT": 16,
            "B200_GEMV_RING_KB": 128, "B200_QKV_RING_KB": 0, "B200_ATTN_DEFER_MERGE": 0,
            "B200_EPI_WARPS4": 0, "B200_KEEP_CONST": 1, "B200_CONST_PF": 1, "B200_ATTN_EVEN": 0,
            "B200_G1_HOLD_SLOTS": 0, "B200_G1_DBG": 0, "B200_G1_WARM": 0, "B200_STREAM_EF": 1, "B200_KV_EF": 1}
SPEC = [
    ("A default", {}, True),
    ("B PF_KV=0", {"B200_PF_KV": 0}, True),
    ("C SELF_PF", {"B200_SELF_PF_KB": 4096}, False),
    ("D SELF_PF+EARLY", {"B200_SELF_PF_KB": 4096, "B200_PF_EARLY": 1}, False),
    ("E SELF_PF+EARLY+next full", {"B200_SELF_PF_KB": 4096, "B200_PF_EARLY": 1, "B200_PF_KB": 100000}, True),
    ("F E+PF_KV=0", {"B200_SELF_PF_KB": 4096, "B200_PF_EARLY": 1, "B200_PF_KB": 100000, "B200_PF_KV": 0}, True),
    ("G SELF_PF+PF_KV=0", {"B200_SELF_PF_KB": 4096, "B200_PF_KV": 0}, True),
    ("H SELF_PF+EARLY+512KB", {"B200_SELF_PF_KB": 4096, "B200_PF_EARLY": 1, "B200_PF_KB": 512}, False),
    ("I SELF_PF+EARLY+512KB+PF_KV=0", {"B200_SELF_PF_KB": 4096, "B200_PF_EARLY": 1, "B200_PF_KB": 512, "B200_PF_KV": 0}, False),
    ("J EARLY only", {"B200_PF_EARLY": 1}, False),
    ("K next full, late", {"B200_PF_KB": 100000}, False),
]
if len(sys.argv) > 1:
    SPEC = eval(open(sys.argv[1]).read())
MODEL = dict(dim=4096, n_layers=32, n_heads=32, n_kv_heads=None, multiple_of=256, ffn_dim_multiplier=None,
             norm_eps=1e-5, rope_theta=10000.0, vocab_size=32000, max_seq_len=2048 + 352)
CTX, BSZ, K, W = 2048, 1, int(os.environ.get("STEPS", "64")), 40
lib = _cabi.lib()
eng = DecodeEngine(EngineConfig.from_model_args("llama", MODEL, bits=4, group_size=0), "cuda")
eng.load_random(0)
eng.allocate_kv_cache(BSZ)
eng.fill_kv_cache_noise()
NROW = 400
tl = torch.zeros((NROW, 8), dtype=torch.int64, device="cuda")
names = ["qkv", "attn", "wo", "w13", "w2"]


def set_knobs(kv):
    for k, v in DEFAULTS.items():
        lib.b200_tune(k.encode(), int(kv.get(k, v)))
    for k, v in kv.items():
        if k not in DEFAULTS:
            lib.b200_tune(k.encode(), int(v))


def timeline():
    eng.tokens[:BSZ].fill_(5); eng.pos[:BSZ].fill_(CTX)
    eng._step(BSZ, 1, eng.cache_seq); torch.cuda.synchronize()
    lib.b200_timeline(C.c_void_p(tl.data_ptr()), NROW)
    g, n = eng.capture_greedy_loop(BSZ)
    lib.b200_timeline(None, 0)
    for _ in range(4):
        tl.zero_(); tl[:, 0] = torch.iinfo(torch.int64).max
        g.replay()
    torch.cuda.synchronize()
    t = tl.cpu()
    used = [i for i in range(NROW) if t[i, 3] > 0]
    rows = t[used].tolist()
    rows = rows[-161:] if len(rows) > 161 else rows
    t0 = min(r[0] for r in rows)
    out = [f"  rows={len(rows)} step span={(max(r[3] for r in rows) - t0) / 1000:.1f} us   (kern: start | dep-wait xstage mmaend end, us from own first-CTA start | gap to prev end)"]
    prev_end = None
    for j, r in enumerate(rows):
        L, k = divmod(j, 5)
        if L == 15 or j >= 160:
            nm = names[k] if j < 160 else "head"
            gap = (r[0] - prev_end) / 1000 if prev_end else 0
            w = (r[4] - r[0]) / 1000 if r[4] else float("nan")
            out.append(f"  {L:3d} {nm:5s} {(r[0]-t0)/1000:8.2f} | {w:6.2f} {(r[1]-r[0])/1000:6.2f} {(r[2]-r[0])/1000:6.2f} {(r[3]-r[0])/1000:6.2f} | {gap:6.2f}")
        prev_end = r[3]
    per = {}
    for j, r in enumerate(rows[:160]):
        per.setdefault(names[j % 5], []).append((r[3] - r[0]) / 1000)
    out.append("  avg dur: " + "  ".join(f"{k} {sum(v)/len(v):.2f}" for k, v in per.items()))
    # layer period from qkv start to next qkv start, averaged over layers 4..28
    st = [rows[5 * L][0] for L in range(32)]
    out.append(f"  layer period (avg of layers 4..27): {(st[28] - st[4]) / 24 / 1000:.2f} us")
    return "\n".join(out)


for label, kv, want_tl in SPEC:
    try:
        set_knobs(kv)
        eng._graphs.clear()
        g, n = eng.capture_greedy_loop(BSZ)
        eng.tokens[:BSZ].fill_(1234); eng.pos[:BSZ].fill_(CTX)
        for _ in range(W):
            g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(K):
            g.replay()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / K
        print(f"== {label}: {1000.0 / ms:8.1f} tok/s  {ms:.4f} ms/step  knobs={json.dumps(kv)}", flush=True)
        if want_tl:
            print(timeline(), flush=True)
    except Exception as ex:  # keep going: one bad variant must not cost the whole GPU call
        print(f"== {label}: FAILED {type(ex).__name__}: {ex}", flush=True)
        torch.cuda.synchronize()
