"""Time of one b200_sample_top_p call across the vocabulary sizes users serve, on both of its kernels.

    python scripts/sample_bench.py [--reps 200] [--out result.json]

V = 32000 (LLaMA-2) and 57856 run the shared-memory kernel (bisection over the probabilities held on chip); 57857,
103168 (InternLM-7B / -20B) and 256000 run the large-vocabulary kernel (radix descent over the logits row re-read from
L2).  T = 1 and 32 rows, logits ~ N(0, 2.5^2), temperature 0.8, top_p 0.9 and 1.0 (1.0: no threshold search).  Each
figure is CUDA-event time over one replay of a CUDA graph holding --reps calls, so host enqueue cost is excluded; best
of 5 replays after a warm-up replay.  The card name, power limit and max SM clock are printed with the numbers.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from prefill_bench import card  # noqa: E402

VOCABS = (32000, 57856, 57857, 103168, 256000)


def time_call(V, T, top_p, reps):
    import torch
    from llama2_accessory_b200 import ops
    g = torch.Generator(device="cuda:0").manual_seed(V + T)
    logits = torch.randn(T, V, device="cuda:0", generator=g) * 2.5
    u = torch.rand(T, device="cuda:0", generator=g)
    out = torch.empty(T, dtype=torch.int64, device="cuda:0")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ops.sample_top_p(logits, u, out, T, V, 0.8, top_p)  # first launch outside the capture
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(reps):
                ops.sample_top_p(logits, u, out, T, V, 0.8, top_p)
    torch.cuda.synchronize()
    graph.replay()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        graph.replay()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b) * 1e3 / reps)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "sample_bench times the GPU; there is no CPU measurement"
    import llama2_accessory_b200 as pkg
    pkg.build()
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, max SM clock {info['sm_max_clock']}", flush=True)
    res = []
    for V in VOCABS:
        for T in (1, 32):
            for top_p in (0.9, 1.0):
                us = time_call(V, T, top_p, args.reps)
                kernel = "shared-memory bisection" if V * 4 + 1024 <= 227 * 1024 else "radix over L2"
                res.append(dict(V=V, T=T, top_p=top_p, us=us, kernel=kernel))
                print(f"V {V:6d}  T {T:2d}  top_p {top_p:.1f}  {us:8.1f} us/call  ({kernel})", flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=info, results=res), f, indent=1)


if __name__ == "__main__":
    main()
