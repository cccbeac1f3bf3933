"""Per-rank decode-step timing of the SURVEY.md section-8 configurations on ONE GPU.

For a TP > 1 configuration this times ONE rank's shard (its weights, its KV heads) with the collectives
skipped (engine.shard_only) -- the HBM work of a rank, i.e. the per-GPU roofline fraction, NOT the multi-GPU
tokens/s (the all-reduces are missing).  TP = 1 rows are real end-to-end decode numbers.

  python scripts/shape_bench.py [name ...]      -> one JSON line per configuration (stdout)

Under torch.distributed.run with N ranks (python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1
scripts/shape_bench.py C5_70B_W3_tp8rank) the configurations whose TP size equals N run for real: every rank holds its
shard, the collectives run (NCCL all-reduce at T > 1, the fused LL exchange at T = 1), the step time is the maximum over
ranks and the tokens/s are the whole job's.  (Written after the round's GPU budget was spent: this mode has not been run.)
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import llama2_accessory_b200 as pkg  # noqa: E402

L7 = dict(dim=4096, n_layers=32, n_heads=32, vocab_size=32000, multiple_of=256, norm_eps=1e-5)
L13 = dict(dim=5120, n_layers=40, n_heads=40, vocab_size=32000, multiple_of=256, norm_eps=1e-5)
L70 = dict(dim=8192, n_layers=80, n_heads=64, n_kv_heads=8, vocab_size=32000, multiple_of=4096,
           ffn_dim_multiplier=1.3, norm_eps=1e-5)
MIX = dict(dim=4096, n_layers=32, n_heads=32, n_kv_heads=8, vocab_size=32000, hidden_dim=14336, norm_eps=1e-5,
           rope_theta=1e6, moe=dict(num_experts=8, num_experts_per_tok=2))

#            name              kind       args bits gs  bsz  ctx   tp
CONFIGS = [
    ("C2_7B_W4",            "llama",   L7,  4,   0,   1,  2048, 1),
    ("C2_7B_W4g128",        "llama",   L7,  4, 128,   1,  2048, 1),
    ("7B_W3",               "llama",   L7,  3,   0,   1,  2048, 1),
    ("7B_W2g64",            "llama",   L7,  2,  64,   1,  2048, 1),
    ("7B_W4_bs8",           "llama",   L7,  4,   0,   8,  2048, 1),
    ("7B_W4_bs32",          "llama",   L7,  4,   0,  32,  2048, 1),
    ("C3_13B_W4_tp2rank",   "llama",   L13, 4,   0,  32,  4096, 2),
    ("C4_mixtral_W4_tp4rank", "mixtral", MIX, 4,  0,  16,  4096, 4),
    ("C5_70B_W3_tp8rank",   "llama",   L70, 3,   0,   8,  8192, 8),
    ("70B_W3_bs1_tp8rank",  "llama",   L70, 3,   0,   1,  8192, 8),
]


def peak_gbs():
    try:
        d = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
        for k in ("hbm_gbs", "hbm_copy_gbs", "hbm_gb_s"):
            if k in d:
                return float(d[k])
    except Exception:
        pass
    return 6572.5


def run(name, kind, margs, bits, gs, bsz, ctx, tp, steps=48, warmup=8, rank=0, world=1, local=0, group=None):
    from llama2_accessory_b200.engine import DecodeEngine, EngineConfig
    real = world > 1  # every rank of the TP group is a process: collectives on
    max_seq = (ctx + 2 * (steps + warmup) + 64 + 31) // 32 * 32
    cfg = EngineConfig.from_model_args(kind, dict(margs, max_seq_len=max_seq, max_batch_size=max(32, bsz)), bits=bits,
                                       group_size=gs, tp_rank=rank if real else 0, tp_world=tp)
    eng = DecodeEngine(cfg, f"cuda:{local}", group=group)
    eng.shard_only = tp > 1 and not real
    eng.load_random(seed=0)
    eng.allocate_kv_cache(bsz)
    eng.fill_kv_cache_noise(0.5, seed=1)
    graph, launches = eng.capture_greedy_loop(bsz)
    eng.tokens[:bsz].fill_(1234)
    eng.pos[:bsz].fill_(ctx)
    for _ in range(warmup):
        graph.replay()
    if real:
        torch.distributed.barrier()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    ev[0].record()
    for i in range(steps):
        graph.replay()
        ev[i + 1].record()
    if real:
        torch.distributed.barrier()
    torch.cuda.synchronize()
    per = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(steps))
    p50 = per[steps // 2]
    if real:  # the job's step time is the slowest rank's
        t = torch.tensor([p50, per[int(steps * 0.9)]], device=f"cuda:{local}", dtype=torch.float64)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        p50, per[int(steps * 0.9)] = float(t[0]), float(t[1])
    sb = eng.step_bytes(bsz, ctx + warmup + steps // 2)
    if kind == "mixtral":  # only the experts actually selected are read; report the upper bound (all local experts)
        sb["note"] = "weights = all local experts (upper bound on bytes actually read)"
    gbs = sb["total"] / (p50 / 1e3) / 1e9
    pk = peak_gbs()
    out = {"name": name, "kind": kind, "bits": bits, "group_size": gs, "bsz": bsz, "ctx": ctx, "tp_rank_of": tp,
           "collectives": ("real (all ranks running)" if real else "skipped (single-rank shard)") if tp > 1 else "none needed",
           "n_gpus": world, "p50_ms_per_step": p50, "p90_ms_per_step": per[int(steps * 0.9)],
           ("tokens_per_s_whole_job" if real else "tokens_per_s_this_rank"): bsz / (p50 / 1e3),
           "launches_per_step": launches, "step_bytes": sb, "achieved_gbs": gbs, "frac_of_measured_peak": gbs / pk,
           "frac_of_8TBps": gbs / 8000.0}
    del graph, eng
    torch.cuda.empty_cache()
    return out


def main():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    group = None
    torch.cuda.set_device(local)
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
        group = torch.distributed.group.WORLD
    pkg.build()
    want = set(sys.argv[1:])
    for c in CONFIGS:
        if want and c[0] not in want:
            continue
        if world > 1 and c[7] != world:  # under N ranks only the TP = N configurations make sense
            continue
        t0 = time.time()
        try:
            r = run(*c, rank=rank, world=world, local=local, group=group)
            r["wall_s"] = time.time() - t0
        except Exception as e:  # keep going: one bad shape must not lose the others
            r = {"name": c[0], "error": f"{type(e).__name__}: {e}"}
            if world > 1:
                raise  # a rank that dropped out would leave the others waiting in a collective
        if rank == 0:
            print(json.dumps(r), flush=True)
    if world > 1:
        torch.cuda.synchronize()
        torch.distributed.barrier()
        sys.stdout.flush()
        os._exit(0)  # NCCL communicators referenced by captured graphs can hang destroy_process_group()


if __name__ == "__main__":
    main()
