"""Prompt (prefill) latency of Mixtral-8x7B W4 per-channel on one GPU: the tensor-core path (grouped wgmma GEMM over each
layer's routed experts, b200_prefill_moe_gemm_w4) against the GEMV chunks (32 / top-k = 16 tokens per chunk, every chunk
streams nearly all expert weights), plus a LLaMA-2-7B 2048-token control.

    python scripts/prefill_bench.py [--runs 3] [--out result.json]

Full depth, TP = 1, bs = 1, random packed weights (about 23 GB for Mixtral).  Each prompt is timed from its first launch
to a device synchronise, the two paths alternating in one process, after a warm-up of every shape.  A second pass records
the grouped GEMM with torch.profiler (a separate pass: tracing slows the host) and reports per launch its time, the bytes
it must move (weights of the experts that got a slot, activations in, outputs out) and the FLOPs of its slots, against the
H100 SXM data-sheet peaks (3.35 TB/s HBM3, 989 TFLOP/s dense fp16) -- the larger of the two least times names the bound.
The card name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12
FP16_PEAK = 989e12
MIXTRAL = dict(dim=4096, n_layers=32, n_heads=32, n_kv_heads=8, hidden_dim=14336, vocab_size=32000, norm_eps=1e-5,
               rope_theta=1e6, max_batch_size=1, moe=dict(num_experts=8, num_experts_per_tok=2))
LLAMA7B = dict(dim=4096, n_layers=32, n_heads=32, n_kv_heads=None, multiple_of=256, ffn_dim_multiplier=None, norm_eps=1e-5,
               rope_theta=10000.0, vocab_size=32000, max_batch_size=1)
PROMPTS = (33, 128, 512, 2048)


def card():
    import torch
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ""
    parts = [p.strip() for p in line.split(",")] if line else []
    return dict(name=torch.cuda.get_device_name(0), power_limit=parts[1] if len(parts) > 1 else "unknown",
                sm_max_clock=parts[2] if len(parts) > 2 else "unknown")


def timed_prompt(eng, toks):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng.forward_inference(toks, 0)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def engine(kind, margs, max_seq_len):
    from llama2_accessory_b200.engine import DecodeEngine, EngineConfig
    cfg = EngineConfig.from_model_args(kind, dict(margs, max_seq_len=max_seq_len), bits=4, group_size=0)
    eng = DecodeEngine(cfg, "cuda:0")
    eng.load_random(seed=0)
    assert eng.prefill_tc_supported(), "per-channel W4 with 128-row tiles: the tensor-core path must apply"
    return eng


def grouped_gemm_profile(eng, toks):
    """torch.profiler pass over one prompt: every b200_prefill_moe_gemm_w4 launch with its bytes and FLOPs."""
    import torch
    from llama2_accessory_b200 import ops
    c = eng.cfg
    k = c.experts_per_tok
    launches = []  # per launch, in enqueue order: (proj, n_slots, bytes, flops), counts read back after the pass
    orig = ops.prefill_moe_gemm_w4

    def spy(experts, x, out, *, slot_expert, n_slots, src_div, e_first):
        orig(experts, x, out, slot_expert=slot_expert, n_slots=n_slots, src_div=src_div, e_first=e_first)
        counts = torch.bincount(slot_expert[:n_slots].long() - e_first, minlength=len(experts))[:len(experts)]
        launches.append((experts, counts.clone(), src_div, n_slots))
    ops.prefill_moe_gemm_w4 = spy
    try:
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            eng.forward_inference(toks, 0)
            torch.cuda.synchronize()
    finally:
        ops.prefill_moe_gemm_w4 = orig
    from torch.autograd import DeviceType
    times = [e.time_range.elapsed_us() for e in prof.events()  # us, in launch order
             if e.device_type == DeviceType.CUDA and "prefill_moe_gemm_w4_kernel" in e.name]
    assert len(times) == len(launches), (len(times), len(launches))
    rows = []
    for (experts, counts, src_div, n_slots), us in zip(launches, times):
        counts = counts.cpu().tolist()
        N, K = experts[0].N, experts[0].K
        used = [i for i, n in enumerate(counts) if n]
        wbytes = sum(experts[i].nbytes for i in used)
        slots = sum(counts)
        xbytes = ((n_slots - 1) // src_div + 1) * K * 2 if src_div > 1 else slots * K * 2
        byts = wbytes + xbytes + slots * N * 2
        flops = 2.0 * slots * N * K
        t_mem, t_cmp = byts / HBM_PEAK, flops / FP16_PEAK
        rows.append(dict(proj="w13" if src_div > 1 else "w2", N=N, K=K, slots=slots, experts_used=len(used), us=us,
                         bytes=byts, flops=flops, tbps=byts / (us * 1e-6) / 1e12, tflops=flops / (us * 1e-6) / 1e12,
                         bound="HBM" if t_mem >= t_cmp else "tensor-core", frac_of_bound=max(t_mem, t_cmp) / (us * 1e-6)))
    return rows


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
    res = dict(card=info, mixtral={}, profile=None, llama7b=None)

    eng = engine("mixtral", MIXTRAL, 2048 + 64)
    g = torch.Generator(device="cuda:0").manual_seed(1)
    toks = {n: torch.randint(1, MIXTRAL["vocab_size"], (1, n), device="cuda:0", generator=g) for n in PROMPTS}
    for n in PROMPTS:  # warm-up of every shape on both paths
        for tc in (True, False):
            eng.use_prefill_tc = tc
            eng.forward_inference(toks[n][:, :min(n, 300)], 0)
    torch.cuda.synchronize()
    for n in PROMPTS:
        t = {True: [], False: []}
        for _ in range(args.runs):
            for tc in (True, False):
                eng.use_prefill_tc = tc
                t[tc].append(timed_prompt(eng, toks[n]))
        res["mixtral"][n] = dict(tc_ms=t[True], gemv_ms=t[False], speedup=min(t[False]) / min(t[True]))
        print(f"mixtral prompt {n:5d}: tensor cores {min(t[True]):8.2f} ms  GEMV chunks {min(t[False]):8.2f} ms  "
              f"(runs: {['%.2f' % v for v in t[True]]} / {['%.2f' % v for v in t[False]]})", flush=True)

    eng.use_prefill_tc = True
    rows = grouped_gemm_profile(eng, toks[2048])
    res["profile"] = rows
    for proj in ("w13", "w2"):
        r = [x for x in rows if x["proj"] == proj]
        us = sorted(x["us"] for x in r)
        full = [x for x in r if x["slots"] == 512]
        print(f"grouped {proj}: {len(r)} launches, median {us[len(us) // 2]:.1f} us, "
              f"256-token chunks: {sum(x['tbps'] for x in full) / max(1, len(full)):.2f} TB/s, "
              f"{sum(x['tflops'] for x in full) / max(1, len(full)):.0f} TFLOP/s, bound {full[0]['bound'] if full else '-'}, "
              f"{sum(x['frac_of_bound'] for x in full) / max(1, len(full)):.2f} of that bound", flush=True)
    del eng
    torch.cuda.empty_cache()

    eng = engine("llama", LLAMA7B, 2048 + 64)
    p = torch.randint(1, LLAMA7B["vocab_size"], (1, 2048), device="cuda:0", generator=g)
    eng.forward_inference(p[:, :256], 0)
    ts = [timed_prompt(eng, p) for _ in range(args.runs)]
    res["llama7b"] = dict(prompt=2048, tc_ms=ts)
    print(f"llama-2-7b prompt 2048: tensor cores {min(ts):.2f} ms (runs: {['%.2f' % v for v in ts]})", flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "profile"}))


if __name__ == "__main__":
    main()
