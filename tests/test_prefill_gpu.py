"""GPU: the wgmma W4A16 prefill GEMM (csrc/prefill.cu) and the prompt path built on it, through the C-ABI.

GEMM checker: F.linear(x, w_hat) in fp32 with w_hat = fp16(fp16(q - z) * s16) -- the reference's fake-quantised weight,
which the kernel reproduces bit for bit before the tensor cores multiply it; tolerance = fp16 rounding of the output.
Prompt checker: the CPU port (bit-pinned to the unmodified reference) in fp32 / fp16 on 128- and 300-token prompts.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import ops, quant  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig  # noqa: E402
from oracle import cases, omniquant, weights  # noqa: E402
from oracle.llama_port import PortModel  # noqa: E402

DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


@pytest.mark.timeout(180)
@pytest.mark.parametrize("N,K,T", [(128, 64, 1), (128, 256, 16), (256, 512, 77), (4096, 4096, 256), (1024, 11008, 300),
                                   (384, 1536, 513)])
def test_prefill_gemm_w4_matches_fake_quantised_linear(N, K, T):
    g = torch.Generator().manual_seed(N + K + T)
    w = ((torch.rand(N, K, generator=g) * 2 - 1) / math.sqrt(K)).half()
    q, s, z, gg = quant.quantize_weight(w, 4, 0)
    pl = quant.pack_quantized(q, s, z, 4, 0, DEV)
    w_hat = quant.dequantize(q, s, z, gg).to(DEV)
    x = torch.randn(T, K, generator=g).half().to(DEV)
    out = torch.full((T, N), float("nan"), dtype=torch.float16, device=DEV)
    ops.prefill_gemm_w4(pl, x, out, T)
    torch.cuda.synchronize()
    ref = F.linear(x.float(), w_hat.float())
    assert torch.isfinite(out).all()
    err = (out.float() - ref).abs().max().item()
    assert err <= 2.0 ** -10 * ref.abs().max().item() + 1e-4, err  # one fp16 ulp of the largest output


@pytest.mark.timeout(300)
@pytest.mark.parametrize("plen", [128, 300])
def test_long_prompt_through_tensor_core_prefill_matches_port(plen):
    args = dict(cases.TINY_LLAMA, max_seq_len=640)
    sd = weights.llama_state_dict(args, seed=0)
    sd_ref, recs = omniquant.fake_quantize_state_dict(sd, 4, 0)
    ndec = 3
    toks = weights.synthetic_tokens(2, plen + ndec, args["vocab_size"], seed=7)
    ref32 = cases.run_schedule(PortModel("llama", args, sd_ref, dtype=torch.float32), toks, plen, ndec).numpy()
    ref16 = cases.run_schedule(PortModel("llama", args, sd_ref, dtype=torch.float16), toks, plen, ndec).numpy()
    floor = np.abs(ref16 - ref32).max()
    got = {}
    for tc in (True, False):
        eng = DecodeEngine(EngineConfig.from_model_args("llama", args, bits=4, group_size=0), DEV)
        eng.use_prefill_tc = tc
        eng.load_master_state_dict(sd, quant_records=recs)
        assert eng.prefill_tc_supported() == tc
        tk = toks.cuda()
        outs = [eng.forward_inference(tk[:, :plen], 0).float().cpu().clone()]
        for j in range(ndec):
            outs.append(eng.forward_inference(tk[:, plen + j:plen + j + 1], plen + j).float().cpu().clone())
        got[tc] = torch.stack(outs).numpy()
        e32, e16 = np.abs(got[tc] - ref32).max(), np.abs(got[tc] - ref16).max()
        print(f"\\n[prefill {plen} tc={tc}] |eng-ref16|={e16:.3e} |eng-ref32|={e32:.3e} floor={floor:.3e}")
        from conftest import record_parity
        record_parity(f"tiny_llama_w4_prefill{plen}_{'wgmma' if tc else 'gemv_chunks'}", e16=e16, e32=e32, floor=floor,
                      strict_pass=bool(e16 <= 1e-3 or e32 <= floor), source="oracle port fp16 / fp32 on the CPU")
        assert np.isfinite(got[tc]).all()
        assert e16 <= 1e-3 or e32 <= 1.5 * floor, (e16, e32, floor)
    assert np.abs(got[True] - got[False]).max() <= 4e-3
