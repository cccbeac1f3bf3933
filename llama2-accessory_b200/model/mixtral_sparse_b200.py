"""`llama_type = mixtral_sparse_b200`: drop-in replacement of accessory/model/LLM/mixtral_sparse.py for inference.
Every tensor-parallel rank holds 1/TP of every expert (mixtral_sparse.py:222-264), so every rank streams the same
weight bytes whatever the router picks; the router uses the fp32 score rule (mixtral_sparse.py:417-428).
See llama_b200.py."""
import functools
from dataclasses import dataclass, field
from typing import Dict, Optional

import torch
import torch.nn as nn

from .. import parallel_layers as pl
from ..checkpoint import sparse_expert_merge, sparse_expert_split
from ..parallel_layers import ColumnParallelLinear, ParallelEmbedding
from .llama_b200 import Attention, RMSNorm
from .llama_b200 import Transformer as _LlamaTransformer


@dataclass
class ModelArgs:
    # mixtral_sparse.py:47-68
    dim: int = 4096
    hidden_dim: int = 16384
    head_dim: int = 128
    n_layers: int = 32
    n_heads: int = 32
    n_kv_heads: Optional[int] = None
    vocab_size: int = -1
    norm_eps: float = 1e-5
    rope_theta: float = 1000000
    max_batch_size: int = 32
    max_seq_len: int = 2048
    moe: Dict[str, int] = field(default_factory=lambda: {"num_experts_per_tok": 2, "num_experts": 8})
    load_balancing_weight: float = 0.1
    rope_scaling: Optional[float] = None
    wbits: int = 4
    group_size: int = 0


class MoE(nn.Module):
    """mixtral_sparse.py:222-266: w1 / w2 / w3 [E * hidden_dim / TP, dim] (no `.weight` suffix), expert e owning rows
    [e F_loc, (e+1) F_loc); w2 is applied as x @ w2.  The gate is replicated."""

    def __init__(self, dim, hidden, num_experts):
        super().__init__()
        ws = pl.get_model_parallel_world_size()
        assert hidden % ws == 0
        self.num_experts, self.hidden_dim_per_partition = num_experts, hidden // ws
        for name in ("w1", "w2", "w3"):
            w = nn.Parameter(torch.empty(self.hidden_dim_per_partition * num_experts, dim))
            w.is_model_parallel = True
            w.model_parallel_merge = functools.partial(sparse_expert_merge, num_experts=num_experts)
            w.model_parallel_split = functools.partial(sparse_expert_split, num_experts=num_experts)
            setattr(self, name, w)
        self.gate = nn.Linear(dim, num_experts, bias=False)


class TransformerBlock(nn.Module):
    def __init__(self, layer_id, args):
        super().__init__()
        self.layer_id = layer_id
        self.attention = Attention(args)
        self.feed_forward = MoE(args.dim, args.hidden_dim, args.moe["num_experts"])
        self.attention_norm = RMSNorm(args.dim, eps=args.norm_eps)
        self.ffn_norm = RMSNorm(args.dim, eps=args.norm_eps)


class Transformer(_LlamaTransformer):
    KIND = "mixtral_sparse"

    def _build_modules(self, args):
        self.tok_embeddings = ParallelEmbedding(args.vocab_size, args.dim, init_method=None)
        self.layers = nn.ModuleList([TransformerBlock(i, args) for i in range(args.n_layers)])
        self.norm = RMSNorm(args.dim, eps=args.norm_eps)
        self.output = ColumnParallelLinear(args.dim, args.vocab_size, bias=False, init_method=None)

    def forward(self, examples, image=None):
        return super().forward(examples, image), {}  # mixtral_sparse.py:631 returns (logits, aux_loss_dict)
