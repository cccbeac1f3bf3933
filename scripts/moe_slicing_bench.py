"""Whole experts per rank (mixtral) against every expert sliced over the ranks (mixtral_sparse), timed on ONE GPU.

  python scripts/moe_slicing_bench.py [--steps 40] [--rounds 3] [--prompt 2048]   -> JSON lines on stdout

1. C4 decode step: Mixtral-8x7B, per-channel W4, bs 16, context 4096, TP 4.  Every rank's shard is timed on its own with
   the collectives skipped (DecodeEngine.shard_only), base and sliced built from the same seed (same embedding, router
   and KV-cache noise, so the same tokens reach the routers).  A base rank holds 2 whole experts and streams the ones the
   router picks; a sliced rank holds a quarter of all 8 and streams the quarter of each picked expert.  Reported: every
   rank's median step time and the maximum over ranks (the rank a multi-GPU step would wait for).  These are one shard at
   a time on one GPU: without the all-reduces, and with each rank's own partial sums feeding its router.  They are not
   a multi-GPU measurement, and no multi-GPU number follows from them.
2. A 2048-token TP = 1 prompt (tensor-core path), base against sparse, alternating in one process: at TP 1 the two
   engines differ only in the router's score rule.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import llama2_accessory_b200 as pkg  # noqa: E402

MIX = dict(dim=4096, n_layers=32, n_heads=32, n_kv_heads=8, vocab_size=32000, hidden_dim=14336, norm_eps=1e-5,
           rope_theta=1e6, moe=dict(num_experts=8, num_experts_per_tok=2))


def card():
    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001 -- the number is still reported, labelled without the limit
        out["power_limit"] = f"unknown ({type(e).__name__})"
    return out


def _engine(kind, tp, rank, bsz, max_seq):
    from llama2_accessory_b200.engine import DecodeEngine, EngineConfig
    cfg = EngineConfig.from_model_args(kind, dict(MIX, max_seq_len=max_seq, max_batch_size=max(32, bsz)), bits=4,
                                       tp_rank=rank, tp_world=tp)
    eng = DecodeEngine(cfg, "cuda")
    eng.shard_only = tp > 1
    return eng.load_random(seed=0)


def decode(args):
    bsz, ctx, tp = 16, 4096, 4
    max_seq = (ctx + 2 * args.rounds * (args.steps + 8) + 64 + 31) // 32 * 32
    res = {"what": "C4 decode step, one TP-4 rank's shard at a time on one GPU (collectives skipped)",
           "model": "Mixtral-8x7B W4 per-channel", "bsz": bsz, "ctx": ctx, "tp": tp, "ranks": {}}
    for r in range(tp):
        runs = {}
        for kind in ("mixtral", "mixtral_sparse"):
            eng = _engine(kind, tp, r, bsz, max_seq)
            eng.allocate_kv_cache(bsz)
            eng.fill_kv_cache_noise(0.5, seed=1)
            graph, _ = eng.capture_greedy_loop(bsz)
            eng.tokens[:bsz].fill_(1234)
            eng.pos[:bsz].fill_(ctx)
            for _ in range(8):
                graph.replay()
            runs[kind] = dict(eng=eng, graph=graph, ms=[])
        for _ in range(args.rounds):  # alternate base / sliced
            for kind, st in runs.items():
                torch.cuda.synchronize()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
                ev[0].record()
                for i in range(args.steps):
                    st["graph"].replay()
                    ev[i + 1].record()
                torch.cuda.synchronize()
                st["ms"] += [ev[i].elapsed_time(ev[i + 1]) for i in range(args.steps)]
        res["ranks"][r] = {}
        for kind, st in runs.items():
            ms = sorted(st["ms"])
            res["ranks"][r][kind] = {"p50_ms": ms[len(ms) // 2], "p90_ms": ms[int(len(ms) * 0.9)],
                                     "weight_bytes": st["eng"].step_bytes(bsz, ctx)["weights"]}
        del runs
        torch.cuda.empty_cache()
    for kind in ("mixtral", "mixtral_sparse"):
        res[f"max_over_ranks_p50_ms_{kind}"] = max(v[kind]["p50_ms"] for v in res["ranks"].values())
    return res


def prompt(args):
    from llama2_accessory_b200.engine import EngineConfig  # noqa: F401
    n = args.prompt
    engs = {k: _engine(k, 1, 0, 1, n + 64) for k in ("mixtral", "mixtral_sparse")}
    toks = torch.randint(1, 32000, (1, n), generator=torch.Generator().manual_seed(0)).cuda()
    ms = {k: [] for k in engs}
    for k, e in engs.items():  # warm-up
        e.forward_inference(toks, 0)
    for _ in range(args.rounds):
        for k, e in engs.items():
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            e.forward_inference(toks, 0)
            b.record()
            torch.cuda.synchronize()
            ms[k].append(a.elapsed_time(b))
    assert all(e.prefill_tc_supported() for e in engs.values())
    return {"what": f"{n}-token prompt, TP 1, tensor-core path, alternating", "model": "Mixtral-8x7B W4 per-channel",
            **{f"{k}_ms": sorted(v) for k, v in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--prompt", type=int, default=2048)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU: this script only measures")
    pkg.build()
    c = card()
    t0 = time.time()
    print(json.dumps({**c, **decode(args)}), flush=True)
    torch.cuda.empty_cache()
    print(json.dumps({**c, **prompt(args), "wall_s": time.time() - t0}), flush=True)


if __name__ == "__main__":
    main()
