"""`llama_type = internlm_b200`: drop-in replacement of accessory/model/LLM/internlm.py for inference.

The reference's `ModelArgs` and state-dict keys (embedding / layers.{i}.{norm1, norm2, mixer.Wqkv, mixer.out_proj,
mlp.w1, mlp.w2, mlp.w3} / norm / head, with the Wqkv and out_proj biases); the engine reads them through
checkpoint.InternLMView.  Like the reference module it runs at tensor-parallel size 1 only.  See llama_b200.py.
"""
from dataclasses import dataclass
from typing import Optional

import torch.nn as nn

from ..engine import DecodeEngine, EngineConfig
from ..parallel_layers import ColumnParallelLinear, ParallelEmbedding, RowParallelLinear
from .llama_b200 import RMSNorm
from .llama_b200 import Transformer as _LlamaTransformer


@dataclass
class ModelArgs:
    # internlm.py:45-64
    num_layers: int = 32
    hidden_size: int = 4096
    num_attention_heads: int = 32
    mlp_ratio: float = 8 / 3
    drop_rate: float = 0.0
    layer_norm_epsilon: float = 1e-5
    norm_type: str = "rmsnorm"
    norm_eps: float = 1e-5
    use_scaled_init: bool = True
    use_swiglu: bool = True
    vocab_size: int = -1
    multiple_of: int = 256
    rope_theta: float = 10000
    max_batch_size: int = 32
    max_seq_len: int = 2048
    rope_scaling: Optional[float] = None
    wbits: int = 4
    group_size: int = 0


def ffn_hidden(args: ModelArgs) -> int:
    m = args.multiple_of
    return m * ((int(args.hidden_size * args.mlp_ratio) + m - 1) // m)


class MHA(nn.Module):
    def __init__(self, args):
        super().__init__()
        D = args.hidden_size
        self.Wqkv = ColumnParallelLinear(D, 3 * D, bias=True, gather_output=False, init_method=None)
        self.out_proj = RowParallelLinear(D, D, bias=True, input_is_parallel=True, init_method=None)


class FeedForward(nn.Module):
    """internlm.py:181-196: w1 gate [F, D], w2 up [F, D] (a RowParallelLinear(dim, hidden)), w3 down [D, F]."""

    def __init__(self, dim, hidden):
        super().__init__()
        self.w1 = ColumnParallelLinear(dim, hidden, bias=False, gather_output=False, init_method=None)
        self.w2 = RowParallelLinear(dim, hidden, bias=False, input_is_parallel=True, init_method=None)
        self.w3 = ColumnParallelLinear(hidden, dim, bias=False, gather_output=False, init_method=None)


class PackedFlashBaseLayer1D(nn.Module):
    def __init__(self, layer_idx, args):
        super().__init__()
        self.layer_idx = layer_idx
        self.mixer = MHA(args)
        self.norm1 = RMSNorm(args.hidden_size, eps=args.layer_norm_epsilon)
        self.norm2 = RMSNorm(args.hidden_size, eps=args.layer_norm_epsilon)
        self.mlp = FeedForward(args.hidden_size, ffn_hidden(args))


class Transformer(_LlamaTransformer):
    KIND = "internlm"

    def __init__(self, args: ModelArgs, with_visual=False):
        # the shared surface of llama_b200.Transformer reads n_layers
        args.n_layers = args.num_layers
        super().__init__(args, with_visual)

    def _build_modules(self, args):
        # EngineConfig refuses what the engine does not serve (LayerNorm, no SwiGLU, TP > 1) before any weight is built
        EngineConfig.from_model_args("internlm", self._engine_args())
        self.embedding = ParallelEmbedding(args.vocab_size, args.hidden_size, init_method=None)
        self.layers = nn.ModuleList([PackedFlashBaseLayer1D(i, args) for i in range(args.num_layers)])
        self.norm = RMSNorm(args.hidden_size, eps=args.layer_norm_epsilon)
        self.head = ColumnParallelLinear(args.hidden_size, args.vocab_size, bias=False, init_method=None)

    def _engine_args(self):
        a = self.args
        return {k: getattr(a, k) for k in a.__dataclass_fields__ if k not in ("wbits", "group_size")}

    def _engine_config(self, device):
        from .. import parallel_layers as pl
        return EngineConfig.from_model_args("internlm", self._engine_args(), bits=self.args.wbits,
                                            group_size=self.args.group_size, tp_rank=pl.get_model_parallel_rank(),
                                            tp_world=pl.get_model_parallel_world_size())

    @classmethod
    def from_engine(cls, engine: DecodeEngine):
        raise NotImplementedError("internlm_b200 is built from a checkpoint (build_engine_from_pretrained or the module)")
