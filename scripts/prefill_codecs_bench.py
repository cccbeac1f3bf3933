"""Prompt (prefill) latency of the tensor-core path against the GEMV chunks for per-channel W3 and fp16 linears.

    python scripts/prefill_codecs_bench.py [--runs 3] [--out result.json]

  - LLaMA-2-7B full depth, TP = 1, bs = 1, random packed weights, W3 per-channel and fp16 linears: prompts of 33 / 128 /
    512 / 2048 tokens (W3 also 40 / 48 / 64 / 96), each timed from its first launch to a device synchronise, the two
    paths alternating in one process after a warm-up of every shape; best of --runs.
  - The per-rank linears of LLaMA-2-70B at TP = 8 (W3), timed alone: one 256-token GEMM launch against the eight 32-token
    GEMV launches the chunked path spends on the same tokens (CUDA events around 20 repetitions).  A 70B model does not
    fit one engine at TP = 1, and an engine that holds only its own shard does not take the tensor-core path.
The card name, power limit and max SM clock are printed with the numbers.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from prefill_bench import LLAMA7B, PROMPTS, card, timed_prompt  # noqa: E402

CROSSOVER = (40, 48, 64, 96)  # W3 prompts just above one 32-token chunk, where the two paths are closest
R70_TP8 = {"wqkv": (1280, 8192), "wo": (8192, 1024), "w13": (7168, 8192), "w2": (8192, 3584)}  # (N, K) of one rank


def engine(bits, max_seq_len):
    from llama2_accessory_b200.engine import DecodeEngine, EngineConfig
    cfg = EngineConfig.from_model_args("llama", dict(LLAMA7B, max_seq_len=max_seq_len), bits=bits, group_size=0)
    eng = DecodeEngine(cfg, "cuda:0")
    eng.load_random(seed=0)
    assert eng.prefill_tc_supported(), f"per-channel bits {bits} with 128-row tiles: the tensor-core path must apply"
    return eng


def prompts(bits, runs, g, lengths=PROMPTS):
    import torch
    eng = engine(bits, 2048 + 64)
    toks = {n: torch.randint(1, LLAMA7B["vocab_size"], (1, n), device="cuda:0", generator=g) for n in lengths}
    for n in lengths:  # warm-up of every shape on both paths
        for tc in (True, False):
            eng.use_prefill_tc = tc
            eng.forward_inference(toks[n], 0)
    torch.cuda.synchronize()
    res = {}
    for n in lengths:
        t = {True: [], False: []}
        for _ in range(runs):
            for tc in (True, False):
                eng.use_prefill_tc = tc
                t[tc].append(timed_prompt(eng, toks[n]))
        res[n] = dict(tc_ms=t[True], gemv_ms=t[False], speedup=min(t[False]) / min(t[True]))
        print(f"7B {'W3' if bits == 3 else 'fp16'} prompt {n:5d}: tensor cores {min(t[True]):8.2f} ms  "
              f"GEMV chunks {min(t[False]):8.2f} ms  x{res[n]['speedup']:.2f}  "
              f"(runs: {['%.2f' % v for v in t[True]]} / {['%.2f' % v for v in t[False]]})", flush=True)
    del eng
    torch.cuda.empty_cache()
    return res


def rank_linears(runs, g, reps=20):
    """70B TP = 8 rank, W3: 256 tokens as one GEMM launch vs eight 32-token GEMV launches, per linear."""
    import torch
    from llama2_accessory_b200 import ops
    from llama2_accessory_b200.quant import random_packed
    res = {}
    for name, (N, K) in R70_TP8.items():
        pl = random_packed(3, N, K, 0, "cuda:0", seed=N + K)
        x = torch.randn(256, K, device="cuda:0", generator=g).half()
        out = torch.empty(256, N, device="cuda:0", dtype=torch.float16)

        def tc():
            ops.prefill_gemm_w4(pl, x, out, 256)

        def gemv():
            for t0 in range(0, 256, 32):
                ops.gemv(pl, 32, xin=x[t0:t0 + 32], out=out[t0:t0 + 32])
        t = {}
        for label, fn in (("tc", tc), ("gemv", gemv)):
            fn()
        torch.cuda.synchronize()
        for label, fn in (("tc", tc), ("gemv", gemv)) * runs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            e1.synchronize()
            t.setdefault(label, []).append(e0.elapsed_time(e1) / reps * 1e3)
        res[name] = dict(N=N, K=K, tc_us=t["tc"], gemv_us=t["gemv"], speedup=min(t["gemv"]) / min(t["tc"]))
        print(f"70B TP=8 rank W3 {name:4s} {N:5d} x {K:5d}, 256 tokens: one GEMM {min(t['tc']):8.1f} us  "
              f"8 GEMV launches {min(t['gemv']):8.1f} us  x{res[name]['speedup']:.2f}", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "timings need a GPU"
    torch.cuda.set_device(0)
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, max SM clock {info['sm_max_clock']}", flush=True)
    g = torch.Generator(device="cuda:0").manual_seed(1)
    t0 = time.time()
    res = dict(card=info, llama7b_w3=prompts(3, args.runs, g, PROMPTS + CROSSOVER),
               llama7b_fp16=prompts(16, args.runs, g), llama70b_tp8_rank_w3=rank_linears(args.runs, g))
    res["wall_s"] = time.time() - t0
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
