"""GPU: full-depth parity on BASELINE.json's headline model -- LLaMA2-7B (32 layers, D = 4096, F = 11008), OmniQuant
W4A16 per-channel, prefill 128 + 16 single-token decode steps (SURVEY.md 8d schedule) -- against the UNMODIFIED
reference Transformer (accessory/model/LLM/llama.py, staged under oracle/_ref; the bit-pinned port if absent) run on
the same GPU in fp32 and in fp16 on the identical fake-quantised weights.  Decode steps go through the persistent
whole-step kernel, the prefill through the batched kernels.  Numbers land in PARITY_r02.json.
"""
import os
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig  # noqa: E402
from oracle import big_model, weights  # noqa: E402

ARGS_7B = dict(dim=4096, n_layers=32, n_heads=32, n_kv_heads=None, multiple_of=256, ffn_dim_multiplier=None,
               norm_eps=1e-5, rope_theta=10000.0, vocab_size=32000, max_seq_len=256, max_batch_size=1)
RULE_FACTOR = float(os.environ.get("B200_PARITY_FACTOR", "1.5"))


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _schedule(model, toks, plen, ndec):
    outs = [model.forward_inference(toks[:, :plen], 0).float().cpu()]
    for j in range(ndec):
        outs.append(model.forward_inference(toks[:, plen + j:plen + j + 1], plen + j).float().cpu())
    return torch.stack(outs).numpy()


@pytest.mark.timeout(900)
def test_llama2_7b_w4_full_depth_prefill128_decode16():
    if torch.cuda.mem_get_info()[0] < 70e9:
        pytest.skip("needs ~60 GB of free HBM for the fp32 reference next to the engine")
    n_layers = int(os.environ.get("B200_PARITY_LAYERS", "32"))
    args = dict(ARGS_7B, n_layers=n_layers)
    plen, ndec = 128, 16
    toks = weights.synthetic_tokens(1, plen + ndec, args["vocab_size"])
    t0 = time.time()
    # reference model on the GPU in fp32 (every fake-quantised fp16 weight is exact in fp32), then the same in fp16
    model, kind, recs = big_model.build(args, bits=4, group_size=0, dtype=torch.float32, device="cuda", prep_device="cuda",
                                        want_records=True)
    t1 = time.time()
    with torch.inference_mode():
        ref32 = _schedule(model, toks.cuda(), plen, ndec)
        if kind == "reference":
            model._destroy_kv_cache()
            model.half()
            model.freqs_cis = model.freqs_cis  # complex64 table is dtype independent
            ref16 = _schedule(model, toks.cuda(), plen, ndec)
            sd_small = {k: v.detach().to(torch.float16).cpu() for k, v in model.state_dict().items()
                        if k in ("tok_embeddings.weight", "norm.weight", "output.weight") or k.endswith("_norm.weight")}
        else:
            sd16 = {k: v.to(torch.float16) for k, v in model.sd.items()}
            from oracle.llama_port import PortModel
            m16 = PortModel("llama", args, sd16, dtype=torch.float16)
            ref16 = _schedule(m16, toks.cuda(), plen, ndec)
            sd_small = {k: v.cpu() for k, v in sd16.items()
                        if k in ("tok_embeddings.weight", "norm.weight", "output.weight") or k.endswith("_norm.weight")}
            del m16, sd16
    del model
    torch.cuda.empty_cache()
    t2 = time.time()
    eng = DecodeEngine(EngineConfig.from_model_args("llama", args, bits=4, group_size=0), "cuda")
    eng.load_master_state_dict(sd_small, quant_records={k: dict(q=r["q"], scale=r["scale"], zero=r["zero"],
                                                                group_size=r["group_size"]) for k, r in recs.items()})
    decode_path = ("persistent dataflow kernel" if (eng.mega_supported(1) and eng.mega_dataflow) else
                   "persistent barrier kernel" if eng.mega_supported(1) else "separate kernels")
    t3 = time.time()
    got = _schedule(eng, toks.cuda(), plen, ndec)
    t4 = time.time()
    e16, e32, floor = np.abs(got - ref16).max(), np.abs(got - ref32).max(), np.abs(ref16 - ref32).max()
    agree = float((got.argmax(-1) == ref32.argmax(-1)).mean())
    agree16 = float((ref16.argmax(-1) == ref32.argmax(-1)).mean())
    print(f"\n[7B W4 x{n_layers} layers, {kind}] |eng-ref16|={e16:.3e} |eng-ref32|={e32:.3e} |ref16-ref32|={floor:.3e} "
          f"argmax eng/ref16 vs ref32 = {agree:.3f}/{agree16:.3f} absmax={np.abs(ref32).max():.2f} "
          f"decode: {decode_path} (build ref {t1 - t0:.0f}s, ref runs {t2 - t1:.0f}s, engine load {t3 - t2:.0f}s, engine run {t4 - t3:.1f}s)")
    rms32 = float(np.sqrt(np.mean((got - ref32) ** 2)))
    rms_floor = float(np.sqrt(np.mean((ref16 - ref32) ** 2)))
    from conftest import record_parity
    record_parity(f"C2_llama2_7b_w4_{n_layers}layers_prefill{plen}_decode{ndec}", e16=e16, e32=e32, floor=floor,
                  rms32=rms32, rms_floor=rms_floor, strict_pass=bool(e16 <= 1e-3 or e32 <= floor),
                  absmax=np.abs(ref32).max(), argmax_agree=agree, argmax_agree_ref16=agree16, rule_factor=RULE_FACTOR,
                  decode_path=decode_path, prefill_path="wgmma GEMM" if eng.prefill_tc_supported() else "GEMV chunks",
                  source=f"{kind} on the GPU (fp32 / fp16), identical fake-quantised weights")
    assert np.isfinite(got).all()
    assert (e16 <= 1e-3 or e32 <= RULE_FACTOR * floor
            or (rms32 <= 1.02 * rms_floor and e32 <= 1.25 * floor)), (e16, e32, floor, rms32, rms_floor)
    assert agree >= agree16 - 1e-9 or agree >= 0.9
