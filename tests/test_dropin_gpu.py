"""GPU: the drop-in surface -- `llama_type` modules (ModelArgs / Transformer.forward_inference) and the
fairscale-style layers + quantize_omni operator hook -- against the oracle."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import parallel_layers as pl  # noqa: E402
from llama2_accessory_b200.model import llama_b200, mixtral_b200  # noqa: E402
from oracle import cases, omniquant  # noqa: E402
from oracle.llama_port import PortModel  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _model(mod, args, sd, wbits, gs):
    fields = mod.ModelArgs.__dataclass_fields__
    a = mod.ModelArgs(**{k: v for k, v in args.items() if k in fields}, wbits=wbits, group_size=gs)
    with torch.device("cuda"):
        old = torch.get_default_dtype()
        torch.set_default_dtype(torch.float16)
        try:
            m = mod.Transformer(a)
        finally:
            torch.set_default_dtype(old)
    missing, unexpected = m.load_state_dict({k: v.cuda() for k, v in sd.items()}, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    return m.eval()


@pytest.mark.parametrize("name,mod", [("llama_w4", llama_b200), ("mixtral_w4", mixtral_b200)])
def test_transformer_dropin_forward_inference(name, mod):
    """Checkpoint-shaped state dict (the reference's keys) -> Transformer -> forward_inference, vs the port
    run on the fake-quantised weights.  The module quantises its own (rank-local) shards, which at TP=1 is the
    same min/max quantisation the oracle applied."""
    kind, args, bits, gs, bsz, plen, ndec = cases.CASES[name]
    kind, args, sd, sd_ref, recs, toks = cases.build_case(name)
    m = _model(mod, args, sd, bits, gs)
    assert hasattr(m, "layers") and m.image_words == 0
    tk = toks.cuda()
    got = [m.forward_inference(tk[:, :plen], 0).float().cpu()]
    for j in range(ndec):
        got.append(m.forward_inference(tk[:, plen + j:plen + j + 1], plen + j).float().cpu())
    got = torch.stack([g.clone() for g in got]).numpy()
    port = PortModel(kind, args, sd_ref, dtype=torch.float32)
    ref = cases.run_schedule(port, toks, plen, ndec).numpy()
    assert got.shape == ref.shape and got.dtype == np.float32
    assert np.abs(got - ref).max() <= 3e-3
    m._destroy_kv_cache()
    assert m.engine.kcache is None


def test_transformer_full_forward_matches_port():
    """Transformer.forward (full-sequence logits, MetaModel.compute_logits) of LLaMA W4 and Mixtral W4 (which returns
    (logits, {})) at every position, against the port's last-position logits of every prefix: within 3e-3 of the fp32
    port (LLaMA), and within the floor rule of test_prefill_gpu.py (e16 <= 1e-3 or e32 <= 1.5 x |ref16 - ref32|)."""
    for name, mod in (("llama_w4", llama_b200), ("mixtral_w4", mixtral_b200)):
        kind, args, sd, sd_ref, recs, toks = cases.build_case(name)
        n = toks.shape[1]
        m = _model(mod, args, sd, 4, 0)
        out = m.forward(toks.cuda())
        if kind == "mixtral":
            out, aux = out
            assert aux == {}
        assert out.shape == (toks.shape[0], n, args["vocab_size"]) and out.dtype == torch.float16
        got = out.float().cpu().permute(1, 0, 2)
        refs = {dt: PortModel(kind, args, sd_ref, dtype=dt) for dt in (torch.float32, torch.float16)}
        ref32, ref16 = (torch.stack([refs[dt].forward_inference(toks[:, :p], 0).float() for p in range(1, n + 1)])
                        for dt in (torch.float32, torch.float16))
        e32, e16 = (got - ref32).abs().max().item(), (got - ref16).abs().max().item()
        floor = (ref16 - ref32).abs().max().item()
        print(f"\n[{name} forward, {n} positions] e32 {e32:.3e} e16 {e16:.3e} floor {floor:.3e}")
        assert torch.isfinite(got).all()
        if kind == "llama":
            assert e32 <= 3e-3
        assert e16 <= 1e-3 or e32 <= 1.5 * floor, (name, e16, e32, floor)


def test_parallel_layers_and_quantize_omni_operator_hook():
    """quant.py:95-163 mechanics: quanted_layer attached, weight deleted, forward = W-bit GEMV."""
    torch.manual_seed(0)

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.up = pl.ColumnParallelLinear(512, 256, bias=False, gather_output=False, init_method=None)
            self.down = pl.RowParallelLinear(256, 512, bias=False, input_is_parallel=True, init_method=None)
            self.lora_up = torch.nn.Linear(512, 8, bias=False)

        def forward(self, x):
            return self.down(self.up(x))

    with torch.device("cuda"):
        blk = Block().half()
    with torch.no_grad():
        blk.up.weight.uniform_(-0.05, 0.05)
        blk.down.weight.uniform_(-0.05, 0.05)
    wu, wd = blk.up.weight.detach().clone(), blk.down.weight.detach().clone()
    x = torch.randn(3, 5, 512, device="cuda").half()
    y16 = blk(x)  # un-quantised: fp16 GEMV kernel
    ref16 = F.linear(F.linear(x.float(), wu.float()).half().float(), wd.float())
    assert (y16.float() - ref16).abs().max() <= 2e-2 * ref16.abs().max()
    pl.quantize_omni(blk, wbits=4, group_size=128)
    assert blk.up.weight is None and isinstance(blk.up.quanted_layer, pl.B200Linear)
    assert blk.lora_up.weight is not None  # "lora" names are skipped (quant.py:102-106)
    yq = blk(x)
    ru = omniquant.quantize_weight(wu.cpu(), 4, 128)["w_hat"].cuda().float()
    rd = omniquant.quantize_weight(wd.cpu(), 4, 128)["w_hat"].cuda().float()
    refq = F.linear(F.linear(x.float(), ru).half().float(), rd)
    assert (yq.float() - refq).abs().max() <= 2e-2 * refq.abs().max()
