"""ORACLE TEST INFRASTRUCTURE: mixtral_sparse (accessory/model/LLM/mixtral_sparse.py) -- the CPU port of its MoE, its
small parity cases and its state-dict layout.

The sparse model is the base Mixtral with two differences that matter to inference:
  * weights: per layer one tensor per projection, ``feed_forward.w1`` / ``w2`` / ``w3`` [E * F, D] (no ``.weight``),
    expert e owning rows [e F, (e+1) F); the down projection is applied as x @ w2 (mixtral_sparse.py:244-264, 458);
  * router: softmax in fp32 (not rounded to fp16), top-k on the fp32 scores, renormalised in fp32, cast to fp16 once
    (mixtral_sparse.py:417-428).
Tensor parallelism slices every expert: rank r holds rows [r F/TP, (r+1) F/TP) of each (mixtral_sparse.py:210-219); each
rank forms its slots' partial outputs fp16(y * w), sums them per token, and the ranks' sums are all-reduced.

The port is pinned to the unmodified module run through oracle/shims/{megablocks,stk} on the same host
(tests/test_mixtral_sparse_cpu.py): bit for bit in fp16; in fp32 to 4e-6, because the module's GEMMs run over the 128-row
padded slot rows and fp32 GEMM blocking follows the row count.  oracle/make_golden_sparse.py writes
tests/golden/mixtral_sparse_*.npz from the module itself.
"""
import torch
import torch.nn.functional as F

from . import omniquant, weights
from .cases import run_schedule
from .llama_port import PortModel

# hidden_dim 1024: TP = 2 / 4 / 8 keep 128-row expert slices (mixtral_sparse.py:333)
TINY_SPARSE = dict(dim=512, hidden_dim=1024, n_layers=2, n_heads=4, n_kv_heads=2, norm_eps=1e-5,
                   rope_theta=1000000.0, vocab_size=1024, max_seq_len=64, max_batch_size=4,
                   moe=dict(num_experts=4, num_experts_per_tok=2))

# name -> (args, bits (0 = fp16 weights), group_size, bsz, prefill_len, n_decode)
CASES = {
    "mixtral_sparse_fp16": (TINY_SPARSE, 0, 0, 2, 5, 3),
    "mixtral_sparse_w4":   (TINY_SPARSE, 4, 0, 4, 6, 3),
}


def to_sparse(sd: dict, num_experts: int) -> dict:
    """Base-form Mixtral master weights (experts.{e}.w1 / w3 [F, D], w2 [D, F]) -> the mixtral_sparse layout."""
    out = {}
    for k, v in sd.items():
        if ".feed_forward.experts." in k:
            continue
        out[k] = v
        if k.endswith("feed_forward.gate.weight"):
            p = k[:-len("gate.weight")]
            for w in ("w1", "w2", "w3"):
                blocks = [sd[f"{p}experts.{e}.{w}.weight"] for e in range(num_experts)]
                out[p + w] = torch.cat([b.t() if w == "w2" else b for b in blocks], dim=0).contiguous()
    return out


def build_case(name):
    """-> (args, sparse master fp16 sd, sparse sd the reference runs (fake-quantised for W-bit cases), quant records keyed
    by the per-expert names of checkpoint.SparseExpertView, tokens)."""
    args, bits, gs, bsz, plen, ndec = CASES[name]
    E = args["moe"]["num_experts"]
    base = weights.mixtral_state_dict(args)
    if bits:
        # the down projection is quantised as the [D, F] linear it is, groups along F
        base_ref, recs = omniquant.fake_quantize_state_dict(base, bits, gs)
    else:
        base_ref, recs = base, {}
    toks = weights.synthetic_tokens(bsz, plen + ndec, args["vocab_size"])
    return args, to_sparse(base, E), to_sparse(base_ref, E), recs, toks


class SparsePortModel(PortModel):
    """PortModel (oracle/llama_port.py) with mixtral_sparse's MoE; `sd` in the sparse layout."""

    def __init__(self, args: dict, sd: dict, dtype=torch.float16, tp: int = 1):
        super().__init__("mixtral", args, sd, dtype=dtype, tp=1)
        self.tp = tp  # attention / wo as PortModel; experts sliced by rows below
        self.Fh = args["hidden_dim"]
        assert self.Fh % tp == 0

    def moe(self, i, x):
        p = f"layers.{i}.feed_forward."
        shp = x.shape
        x = x.view(-1, shp[-1])
        D, E, k = shp[-1], self.E, self.topk
        probs = F.softmax(F.linear(x, self._w(p + "gate.weight")), dim=1, dtype=torch.float)
        ew, ei = torch.topk(probs, k, dim=-1)
        if self.record is not None:
            self.record[-1]["own"].append(ei.view(*shp[:-1], k).cpu().clone())
            self.record[-1]["scores"].append(probs.view(*shp[:-1], -1).cpu().clone())
        forced = (self.force_routes or {}).get((self._start_pos, i))
        if forced is not None:
            ei = forced.to(self.device).long().view(-1, k)
            ew = probs.gather(-1, ei)
        if self.record is not None:
            self.record[-1]["routes"].append(ei.view(*shp[:-1], k).cpu().clone())
        ew = (ew / ew.sum(dim=-1, keepdim=True)).flatten().to(x.dtype)
        flat = ei.flatten()
        xr = x.repeat_interleave(k, dim=0)
        w1, w2, w3 = (self._w(p + w).view(E, self.Fh, D) for w in ("w1", "w2", "w3"))
        fl = self.Fh // self.tp
        # the products are formed over all of a rank's expert rows at once and masked to each slot's expert (the dense
        # form of the block-sparse sdd / dsd): the same GEMM shapes as the reference, hence the same bits on one host
        mask = (torch.arange(E, device=x.device)[None, :, None] == flat[:, None, None]).expand(-1, -1, fl).reshape(-1, E * fl)
        parts = []
        for r in range(self.tp):
            rows = lambda w: w[:, r * fl:(r + 1) * fl].reshape(E * fl, D)  # noqa: E731
            act = F.silu(xr @ rows(w1).t()) * (xr @ rows(w3).t())
            y = torch.where(mask, act, torch.zeros_like(act)) @ rows(w2)
            slots = (y.float() * ew.float()[:, None]).to(x.dtype)
            parts.append(slots.view(-1, k, D).sum(dim=1))
        return self._rank_sum(parts).view(*shp)


def port_logits(name, dtype=torch.float16, tp=1):
    args, sd, sd_ref, recs, toks = build_case(name)
    _, _, _, _, plen, ndec = CASES[name]
    return run_schedule(SparsePortModel(args, sd_ref, dtype=dtype, tp=tp), toks, plen, ndec)
