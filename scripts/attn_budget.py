"""Attention's share of the bs = 1 decode step that bench.py measures (LLaMA2-7B W4A16 per-channel, ctx 2048).

Three CUDA graphs on bench.py's model, weights, KV-cache noise and start position:
  step      the captured greedy step (all launches, as bench.py replays it)
  no_attn   the same step with the 32 attention launches left out (GEMVs + head only; its outputs are meaningless)
  attn      the 32 attention launches alone, back to back, with the step's arguments
Each is timed with CUDA events over --steps replays after --warmup, the three alternating for --rounds rounds; the
median round is reported.  attention's marginal time is step - no_attn, and its effective rate is the K/V bytes one
step reads (2 * layers * kv_len * Hkv * 128 * 2) over that time.

    python scripts/attn_budget.py [--steps 128] [--warmup 16] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (MODEL, CTX, BSZ of the benchmarked workload)


def gpu_info():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        pl, mx = r.stdout.strip().split(", ")[:2]
        info.update(power_limit_w=float(pl), sm_max_mhz=float(mx))
    except Exception as e:  # the timings stand without it; say why it is missing
        info["nvidia_smi"] = f"unavailable ({type(e).__name__})"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "attn_budget.py times kernels on the GPU"
    import llama2_accessory_b200 as pkg
    pkg.build()
    from llama2_accessory_b200 import ops
    from llama2_accessory_b200.engine import DecodeEngine, EngineConfig

    K, W = args.steps, max(args.warmup, 3)
    bsz, ctx = bench.BSZ, bench.CTX
    max_seq = (ctx + 2 * (K + W) + 64 + 31) // 32 * 32  # bench.py's cache size, so the split schedule is the same
    eng = DecodeEngine(EngineConfig.from_model_args("llama", dict(bench.MODEL, max_seq_len=max_seq), bits=4, group_size=0),
                       "cuda:0")
    eng.load_random(seed=0)
    eng.allocate_kv_cache(bsz)
    eng.fill_kv_cache_noise(0.5, seed=1)

    with torch.inference_mode():
        step, n_step = eng.capture_greedy_loop(bsz)
        launch = ops.attn_decode
        ops.attn_decode = lambda *a, **k: None
        try:
            no_attn, n_no_attn = eng.capture_greedy_loop(bsz)
        finally:
            ops.attn_decode = launch

        n_split = ops.attn_split(bsz, eng.Hkv, eng.cache_seq)
        eng._ensure_ws(bsz, n_split)

        def attn_only():
            for i, lw in enumerate(eng.layers):
                pf = (lw.wo.qweight, lw.wo.qweight.numel(), lw.wo.N // 16) if eng.prefetch_bytes else None
                ops.attn_decode(eng.q, eng.kcache[i], eng.vtcache[i], eng.pos, eng.attn, T=bsz, Hq=eng.Hq, Hkv=eng.Hkv,
                                cache_seq=eng.cache_seq, tokens_per_seq=1, max_kv_len=eng.cache_seq, ws=eng.ws,
                                counters=eng.counters, n_split=n_split, use_pdl=eng.use_pdl, prefetch=pf)
        attn_only()
        torch.cuda.synchronize()
        attn = torch.cuda.CUDAGraph()
        with torch.cuda.graph(attn):
            attn_only()

    def timed(g, advancing):
        eng.tokens[:bsz].fill_(1234)
        eng.pos[:bsz].fill_(ctx if advancing else ctx + W + K // 2)
        for _ in range(W):
            g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(K):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / K

    runs = {"step": [], "no_attn": [], "attn": []}
    clocks = bench.ClockSampler(0)
    for _ in range(args.rounds):
        runs["step"].append(timed(step, True))
        runs["no_attn"].append(timed(no_attn, True))
        runs["attn"].append(timed(attn, False))
    clk = clocks.stop()

    ms = {k: statistics.median(v) for k, v in runs.items()}
    kv_bytes = eng.step_bytes(bsz, ctx + W + K // 2)["kv"]  # bench.py's mid-window kv length
    marginal = ms["step"] - ms["no_attn"]
    print(json.dumps({
        "workload": bench.WORKLOAD, "gpu": gpu_info(), "clocks": clk, "steps": K, "warmup": W, "rounds": args.rounds,
        "n_split": n_split, "launches": {"step": n_step, "no_attn": n_no_attn, "attn": len(eng.layers)},
        "ms_per_step": {k: round(v, 4) for k, v in ms.items()},
        "ms_per_step_all_rounds": {k: [round(x, 4) for x in v] for k, v in runs.items()},
        "attn_kv_bytes_per_step": kv_bytes,
        "attn_marginal_ms": round(marginal, 4),
        "attn_marginal_tb_s": round(kv_bytes / (marginal * 1e-3) / 1e12, 3),
        "attn_alone_us_per_launch": round(1000.0 * ms["attn"] / len(eng.layers), 2),
        "attn_alone_tb_s": round(kv_bytes / (ms["attn"] * 1e-3) / 1e12, 3),
    }), flush=True)


if __name__ == "__main__":
    main()
