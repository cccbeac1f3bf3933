"""GPU: parity at the layer widths of the other BASELINE.json configurations (VERDICT r01 item 2) -- two full blocks +
lm_head each, against the UNMODIFIED reference Transformer (oracle/_ref; the bit-pinned port if absent) run on the same
GPU in fp32 and in fp16 on the identical OmniQuant fake-quantised weights:

  C1 width  LLaMA2-7B    D 4096, 32 heads, F 11008, fp16 weights (no quantiser: BASELINE.json's first configuration, "fp16 single
                         forward seq=128 bs=1"), prompt 128 through the fp16 GEMV family in 32-token chunks + 4 decode steps
  C3 width  LLaMA2-13B   D 5120, 40 heads, F 13824, W4 per-channel, bs 1, prefill 128 (wgmma GEMM) + 8 decode steps
                         (integer-path GEMV at K = 5120 / 13824)
  C5 width  LLaMA2-70B   D 8192, 64 query / 8 kv heads (n_rep 8), W3 per-channel (native 3-bit layout), bs 4, prefill 24
                         (chunked GEMV path, token-group split) + 4 batched decode steps.  F = 14336 = the FFN width of
                         one rank at TP = 2 (28672 / 2): the GEMV kernels stage one token's activations in shared memory
                         and take K <= 16384, i.e. the 70B model runs at TP >= 2 (BASELINE C5 is TP = 8), and the
                         unmodified reference Transformer cannot be built with a rank's head count, so the test model
                         keeps all 64 heads and takes the rank's FFN width

The full-depth LLaMA2-7B case is tests/test_parity_7b_gpu.py.  Numbers land in PARITY_r02.json.  Asserted rule as for the
other cases (e16 <= 1e-3 or e32 <= RULE_FACTOR * floor or same rms accuracy), with an absolute allowance of two fp16 ulps
of the largest logit for these two-block models, whose own fp16 noise floor is a single rounding step.
"""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig  # noqa: E402
from oracle import big_model, weights  # noqa: E402

RULE_FACTOR = float(os.environ.get("B200_PARITY_FACTOR", "1.5"))

WIDTHS = {
    "C1_width_llama2_7b_fp16": dict(
        args=dict(dim=4096, n_layers=2, n_heads=32, n_kv_heads=None, multiple_of=256, ffn_dim_multiplier=None,
                  norm_eps=1e-5, rope_theta=10000.0, vocab_size=32000, max_seq_len=160, max_batch_size=1),
        bits=0, gs=0, bsz=1, plen=128, ndec=4),
    "C3_width_llama2_13b_w4": dict(
        args=dict(dim=5120, n_layers=2, n_heads=40, n_kv_heads=None, multiple_of=256, ffn_dim_multiplier=None,
                  norm_eps=1e-5, rope_theta=10000.0, vocab_size=32000, max_seq_len=192, max_batch_size=1),
        bits=4, gs=0, bsz=1, plen=128, ndec=8),
    "C5_width_llama2_70b_w3": dict(
        args=dict(dim=8192, n_layers=2, n_heads=64, n_kv_heads=8, multiple_of=256, ffn_dim_multiplier=0.65,
                  norm_eps=1e-5, rope_theta=10000.0, vocab_size=32000, max_seq_len=64, max_batch_size=4),
        bits=3, gs=0, bsz=4, plen=24, ndec=4),
}


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _schedule(model, toks, plen, ndec):
    outs = [model.forward_inference(toks[:, :plen], 0).float().cpu().clone()]
    for j in range(ndec):
        outs.append(model.forward_inference(toks[:, plen + j:plen + j + 1], plen + j).float().cpu().clone())
    return torch.stack(outs).numpy()


def reference_runs(args, bits, gs, toks, plen, ndec, device):
    """-> (ref32, ref16, kind, fp16 tensors for the engine, quant records): the reference model built once in fp32 on
    `device` (every fp16 / fake-quantised fp16 weight is exact in fp32), run, converted to fp16 in place and run again.
    Quantised models hand the engine their (q, scale, zero) records + the small unquantised tensors; bits = 0 (fp16
    linears) hands it the whole fp16 state dict."""
    model, kind, recs = big_model.build(args, bits=bits, group_size=gs, dtype=torch.float32, device=device,
                                        prep_device=device, want_records=True)
    small = ("tok_embeddings.weight", "norm.weight", "output.weight")
    with torch.inference_mode():
        ref32 = _schedule(model, toks.to(device), plen, ndec)
        if kind == "reference":
            model._destroy_kv_cache()
            model.half()
            ref16 = _schedule(model, toks.to(device), plen, ndec)
            sd_small = {k: v.detach().to(torch.float16).cpu() for k, v in model.state_dict().items()
                        if not bits or k in small or k.endswith("_norm.weight")}
        else:
            from oracle.llama_port import PortModel
            sd16 = {k: v.to(torch.float16) for k, v in model.sd.items()}
            ref16 = _schedule(PortModel("llama", args, sd16, dtype=torch.float16), toks.to(device), plen, ndec)
            sd_small = {k: v.cpu() for k, v in sd16.items() if not bits or k in small or k.endswith("_norm.weight")}
    del model
    return ref32, ref16, kind, sd_small, recs


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", list(WIDTHS))
def test_two_blocks_at_baseline_config_width(name):
    w = WIDTHS[name]
    args, bits, gs, bsz, plen, ndec = w["args"], w["bits"], w["gs"], w["bsz"], w["plen"], w["ndec"]
    torch.cuda.empty_cache()  # earlier tests of the session leave blocks cached in the allocator
    if torch.cuda.mem_get_info()[0] < 40e9:
        pytest.skip("needs ~30 GB of free HBM for the fp32 reference next to the engine")
    toks = weights.synthetic_tokens(bsz, plen + ndec, args["vocab_size"], seed=11)
    ref32, ref16, kind, sd_small, recs = reference_runs(args, bits, gs, toks, plen, ndec, "cuda")
    torch.cuda.empty_cache()
    eng = DecodeEngine(EngineConfig.from_model_args("llama", args, bits=bits or 16, group_size=gs), "cuda")
    eng.load_master_state_dict(sd_small, quant_records={k: dict(q=r["q"], scale=r["scale"], zero=r["zero"],
                                                                group_size=r["group_size"]) for k, r in recs.items()} if bits else None)
    got = _schedule(eng, toks.cuda(), plen, ndec)
    assert got.shape == ref32.shape and np.isfinite(got).all()
    e16, e32, floor = np.abs(got - ref16).max(), np.abs(got - ref32).max(), np.abs(ref16 - ref32).max()
    absmax = float(np.abs(ref32).max())
    rms32 = float(np.sqrt(np.mean((got - ref32) ** 2)))
    rms_floor = float(np.sqrt(np.mean((ref16 - ref32) ** 2)))
    agree = float((got.argmax(-1) == ref32.argmax(-1)).mean())
    agree16 = float((ref16.argmax(-1) == ref32.argmax(-1)).mean())
    top2 = np.sort(ref32, axis=-1)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 4 * floor
    ulp = 2.0 ** (math.floor(math.log2(max(absmax, 1e-3))) - 10)  # fp16 spacing at the largest logit
    print(f"\n[{name}, {kind}] |eng-ref16|={e16:.3e} |eng-ref32|={e32:.3e} floor={floor:.3e} rms {rms32:.3e}/{rms_floor:.3e} "
          f"argmax eng/ref16 vs ref32 = {agree:.3f}/{agree16:.3f} absmax={absmax:.2f}")
    from conftest import record_parity
    record_parity(name, e16=e16, e32=e32, floor=floor, rms32=rms32, rms_floor=rms_floor,
                  strict_pass=bool(e16 <= 1e-3 or e32 <= floor), absmax=absmax, argmax_agree=agree,
                  argmax_agree_ref16=agree16, rule_factor=RULE_FACTOR, bits=bits, bsz=bsz, prefill=plen, decode=ndec,
                  prefill_path="wgmma GEMM" if (eng.prefill_tc_supported() and plen > 32) else "GEMV chunks",
                  source=f"{kind} on the GPU (fp32 / fp16), identical fake-quantised weights, 2 blocks + lm_head")
    assert (e16 <= 1e-3 or e32 <= RULE_FACTOR * floor or (rms32 <= 1.02 * rms_floor and e32 <= 1.25 * floor)
            or e32 <= 2.05 * ulp), (name, e16, e32, floor, rms32, rms_floor, ulp)
    if clear.any():
        assert (got.argmax(-1)[clear] == ref32.argmax(-1)[clear]).all()
