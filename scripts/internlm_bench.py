"""InternLM-7B W4A16 at bs = 1, context 2048, random weights: decode tokens/s and the time of a 2048-token prompt, with the
Wqkv / out_proj bias epilogues on and off in the same engine (alternated), beside the card's name and power limit.

    python scripts/internlm_bench.py [--steps 200] [--rounds 5] [--out internlm_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig  # noqa: E402

INTERNLM_7B = dict(num_layers=32, hidden_size=4096, num_attention_heads=32, mlp_ratio=8 / 3, multiple_of=256,
                   layer_norm_epsilon=1e-6, vocab_size=103168, rope_theta=10000, max_seq_len=2048, max_batch_size=1)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg.build()
    eng = DecodeEngine(EngineConfig.from_model_args("internlm", INTERNLM_7B, bits=4), "cuda").load_random(seed=0)
    biases = [(lw.bqkv, lw.bo) for lw in eng.layers]

    def set_bias(on):
        for lw, (bq, bo) in zip(eng.layers, biases):
            lw.bqkv, lw.bo = (bq, bo) if on else (None, None)
        eng._graphs.clear()

    eng.allocate_kv_cache(1)
    eng.fill_kv_cache_noise()
    tok = torch.ones(1, dtype=torch.int64, device="cuda")
    prompt = torch.randint(1, 103168, (1, 2048), generator=torch.Generator().manual_seed(0)).cuda()
    res = {"on": {"decode_ms": [], "prompt_ms": []}, "off": {"decode_ms": [], "prompt_ms": []}}
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    for r in range(a.rounds + 1):  # round 0 warms up (graph capture, cudaFuncSetAttribute)
        for tag in ("on", "off"):
            set_bias(tag == "on")
            e0, e1 = ev(), ev()
            eng.forward_inference(prompt, 0)
            torch.cuda.synchronize()
            e0.record()
            eng.forward_inference(prompt, 0)
            e1.record()
            torch.cuda.synchronize()
            pm = e0.elapsed_time(e1)
            eng.fill_kv_cache_noise()
            for _ in range(3):
                eng.decode_step(tok, 2040)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.steps):
                eng.decode_step(tok, 2040)  # attention over 2041 cache rows
            e1.record()
            torch.cuda.synchronize()
            if r:
                res[tag]["decode_ms"].append(e0.elapsed_time(e1) / a.steps)
                res[tag]["prompt_ms"].append(pm)
    out = {"model": "InternLM-7B W4A16 (per-channel), random weights", "bs": 1, "ctx": 2048, "card": card(),
           "steps": a.steps, "rounds": a.rounds, "step_bytes": eng.step_bytes(1, 2048)}
    for tag in ("on", "off"):
        d = sorted(res[tag]["decode_ms"])
        p = sorted(res[tag]["prompt_ms"])
        out[f"bias_{tag}"] = {"decode_ms_median": d[len(d) // 2], "decode_tok_s": 1000.0 / d[len(d) // 2],
                              "decode_ms_all": d, "prompt2048_ms_median": p[len(p) // 2], "prompt2048_ms_all": p}
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(out, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
