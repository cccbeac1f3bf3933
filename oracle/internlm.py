"""ORACLE TEST INFRASTRUCTURE: InternLM (accessory/model/LLM/internlm.py) -- a CPU port of its inference path, its small
parity cases and its state-dict layout.

The model is the LLaMA MHA block with four differences that matter to inference:
  * one fused ``mixer.Wqkv`` [3D, D] with a bias, split as ``(three h d)``: F.linear(x, W, b), one fp16 rounding;
  * ``mixer.out_proj`` with a bias that RowParallelLinear adds to the fp16 output after the all-reduce: fp16(fp16(acc) + b);
  * RoPE pairs element i with i + hd/2 and returns the rotated pairs interleaved (internlm.py:31-40);
  * MLP names: ``mlp.w1`` gate [F, D], ``mlp.w2`` up [F, D], ``mlp.w3`` down [D, F]; F = multiple_of * ceil(int(D * mlp_ratio)
    / multiple_of); the norms read ``layer_norm_epsilon``.
The port keeps the module's GEMM shapes (one [3D, D] product for q, k and v), so on one host it reproduces the unmodified
module bit for bit in fp16 and fp32 (tests/test_internlm_cpu.py).  oracle/make_golden_internlm.py writes
tests/golden/internlm_*.npz from the module itself.
"""
import contextlib
import io
import os

import torch
import torch.nn.functional as F

from . import omniquant, weights
from .cases import run_schedule
from .llama_port import causal_mask, precompute_freqs_cis, rmsnorm

TINY_INTERNLM = dict(num_layers=2, hidden_size=256, num_attention_heads=2, mlp_ratio=8 / 3, multiple_of=256,
                     layer_norm_epsilon=1e-5, norm_type="rmsnorm", use_swiglu=True, rope_theta=10000, vocab_size=1024,
                     max_seq_len=64, max_batch_size=4)

# name -> (args, bits (0 = fp16 weights), group_size, bsz, prefill_len, n_decode)
CASES = {
    "internlm_fp16":    (TINY_INTERNLM, 0, 0, 2, 5, 3),
    "internlm_w4":      (TINY_INTERNLM, 4, 0, 2, 5, 3),
    "internlm_w4g128":  (TINY_INTERNLM, 4, 128, 2, 5, 3),
}

QUANT_SUFFIXES = ("mixer.Wqkv.weight", "mixer.out_proj.weight", "mlp.w1.weight", "mlp.w2.weight", "mlp.w3.weight")


def ffn_hidden(args):
    m = args.get("multiple_of", 256)
    return m * ((int(args["hidden_size"] * args.get("mlp_ratio", 8 / 3)) + m - 1) // m)


def state_dict(args: dict, seed: int = 0) -> dict:
    """InternLM master weights in the module's own names (oracle/weights.py's laws).  The biases are drawn U(-0.5, 0.5):
    the module's reset_parameters zeroes them, which would leave the bias epilogues untested."""
    D, L, V = args["hidden_size"], args["num_layers"], args["vocab_size"]
    Fh = ffn_hidden(args)
    u, nw = weights._uniform, weights._norm_weight
    sd = {"embedding.weight": u("embedding.weight", (V, D), D, seed)}
    for i in range(L):
        p = f"layers.{i}."
        sd[p + "mixer.Wqkv.weight"] = u(p + "Wqkv", (3 * D, D), D, seed)
        sd[p + "mixer.Wqkv.bias"] = u(p + "Wqkv.bias", (3 * D,), 4, seed)
        sd[p + "mixer.out_proj.weight"] = u(p + "out_proj", (D, D), D, seed)
        sd[p + "mixer.out_proj.bias"] = u(p + "out_proj.bias", (D,), 4, seed)
        sd[p + "mlp.w1.weight"] = u(p + "w1", (Fh, D), D, seed)
        sd[p + "mlp.w2.weight"] = u(p + "w2", (Fh, D), D, seed)
        sd[p + "mlp.w3.weight"] = u(p + "w3", (D, Fh), Fh, seed)
        sd[p + "norm1.weight"] = nw(p + "n1", D, seed, True)
        sd[p + "norm2.weight"] = nw(p + "n2", D, seed, True)
    sd["norm.weight"] = nw("norm", D, seed, True)
    sd["head.weight"] = u("head.weight", (V, D), D, seed)
    return sd


def fake_quantize(sd: dict, bits: int, group_size: int = 0) -> dict:
    """Every linear of every block through the pinned OmniQuant fake quantisation (embedding, norms, head and biases fp16)."""
    return {k: (omniquant.quantize_weight(v, bits, group_size)["w_hat"] if k.endswith(QUANT_SUFFIXES) else v)
            for k, v in sd.items()}


def quant_records(sd: dict, n_heads: int, bits: int, group_size: int = 0) -> dict:
    """Records of the engine's linears, keyed by checkpoint.InternLMView's LLaMA names.  Quantisation is per output row, so
    quantising the viewed (row-permuted, split) tensors gives the records of the module's Wqkv, reordered."""
    from llama2_accessory_b200.checkpoint import QUANTISED_KEY, InternLMView
    view = InternLMView(sd, n_heads)
    return {k: omniquant.quantize_weight(view[k], bits, group_size) for k in view if QUANTISED_KEY.search(k)}


def build_case(name):
    """-> (args, master fp16 sd, sd the reference runs (fake-quantised for W-bit cases), records keyed by the view's names,
    tokens)."""
    args, bits, gs, bsz, plen, ndec = CASES[name]
    sd = state_dict(args)
    sd_ref = fake_quantize(sd, bits, gs) if bits else sd
    recs = quant_records(sd, args["num_attention_heads"], bits, gs) if bits else {}
    toks = weights.synthetic_tokens(bsz, plen + ndec, args["vocab_size"])
    return args, sd, sd_ref, recs, toks


def rope(x, freqs_cis):
    """internlm.py:31-40: pairs (i, i + hd/2) as complex, fp32 multiply, rotated pairs interleaved, cast back."""
    xc = torch.view_as_complex(x.float().reshape(*x.shape[:-1], 2, -1).transpose(-1, -2).contiguous())
    fc = freqs_cis.view(1, x.shape[1], 1, xc.shape[-1])
    return torch.view_as_real(xc * fc).flatten(3).type_as(x)


class InternLMPortModel:
    """forward_inference of internlm.Transformer (SDPA path) with the module's rounding points and GEMM shapes."""

    def __init__(self, args: dict, sd: dict, dtype=torch.float16):
        self.a, self.dtype = dict(args), dtype
        a = self.a
        self.D, self.L, self.H = a["hidden_size"], a["num_layers"], a["num_attention_heads"]
        self.hd = self.D // self.H
        self.eps = a.get("layer_norm_epsilon", 1e-5)
        self.max_seq_len = a.get("max_seq_len", 2048)
        self.sd = {k: v.to(dtype) for k, v in sd.items()}
        self.device = next(iter(self.sd.values())).device
        self.freqs_cis = precompute_freqs_cis(self.hd, self.max_seq_len * 2, a.get("rope_theta", 10000),
                                              a.get("rope_scaling")).to(self.device)
        self.k_cache = self.v_cache = None

    def alloc_cache(self, bsz):
        shape = (bsz, self.max_seq_len, self.H, self.hd)
        if self.k_cache is None or self.k_cache[0].shape != shape:
            self.k_cache = [torch.zeros(shape, dtype=self.dtype, device=self.device) for _ in range(self.L)]
            self.v_cache = [torch.zeros(shape, dtype=self.dtype, device=self.device) for _ in range(self.L)]

    def attention(self, i, x, start_pos, fc, causal):
        p = f"layers.{i}.mixer."
        B, S, _ = x.shape
        qkv = F.linear(x, self.sd[p + "Wqkv.weight"], self.sd[p + "Wqkv.bias"]).view(B, S, 3, self.H, self.hd)
        q, k, v = qkv.unbind(dim=2)
        q, k = rope(q, fc), rope(k, fc)
        self.k_cache[i][:B, start_pos:start_pos + S] = k
        self.v_cache[i][:B, start_pos:start_pos + S] = v
        keys = self.k_cache[i][:B, :start_pos + S].transpose(1, 2)
        vals = self.v_cache[i][:B, :start_pos + S].transpose(1, 2)
        mask = causal_mask(S, keys.shape[2]).to(self.device) if causal else None
        o = F.scaled_dot_product_attention(q.transpose(1, 2), keys, vals, dropout_p=0.0, attn_mask=mask)
        o = o.transpose(1, 2).contiguous().view(B, S, -1)
        return F.linear(o, self.sd[p + "out_proj.weight"]) + self.sd[p + "out_proj.bias"]

    def ffn(self, i, x):
        p = f"layers.{i}.mlp."
        return F.linear(F.silu(F.linear(x, self.sd[p + "w1.weight"])) * F.linear(x, self.sd[p + "w2.weight"]),
                        self.sd[p + "w3.weight"])

    @torch.inference_mode()
    def forward_inference(self, tokens, start_pos):
        """tokens int64 [B, S] -> logits [B, vocab] of the LAST position, fp32."""
        B, S = tokens.shape
        if start_pos == 0:
            self.alloc_cache(B)
        h = F.embedding(tokens, self.sd["embedding.weight"])
        fc = self.freqs_cis[start_pos:start_pos + S]
        for i in range(self.L):
            p = f"layers.{i}."
            r = self.attention(i, rmsnorm(h, self.sd[p + "norm1.weight"], self.eps), start_pos, fc, S != 1) + h
            h = self.ffn(i, rmsnorm(r, self.sd[p + "norm2.weight"], self.eps)) + r
        hn = rmsnorm(h, self.sd["norm.weight"], self.eps)
        return F.linear(hn[:, -1, :], self.sd["head.weight"]).float()


def reference_available() -> bool:
    """True where the reference tree that oracle/ref_import.py reads holds internlm.py (the staged copy under oracle/_ref
    carries only the LLaMA / Mixtral modules)."""
    from . import ref_import
    return os.path.isfile(os.path.join(ref_import.REF_ROOT, "accessory", "model", "LLM", "internlm.py"))


def reference_model(args: dict, sd: dict, dtype):
    """The unmodified internlm.Transformer on CPU with `sd` loaded (needs the reference tree: reference_available())."""
    from . import ref_import
    if not reference_available():
        raise RuntimeError(f"internlm.py is not present under {ref_import.REF_ROOT}")
    mod = ref_import.load("internlm")
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            model = mod.Transformer(mod.ModelArgs(**args))
    finally:
        torch.set_default_dtype(old)
    missing, unexpected = model.load_state_dict({k: v.to(dtype) for k, v in sd.items()}, strict=True)
    assert not missing and not unexpected
    return model.eval()


def port_logits(name, dtype=torch.float16):
    args, sd, sd_ref, recs, toks = build_case(name)
    _, _, _, _, plen, ndec = CASES[name]
    return run_schedule(InternLMPortModel(args, sd_ref, dtype=dtype), toks, plen, ndec)
