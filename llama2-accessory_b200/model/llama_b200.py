"""`llama_type = llama_b200`: drop-in replacement of accessory/model/LLM/llama.py for inference.

Same surface as the reference module (meta.py:29-54, SURVEY.md 8b): `ModelArgs`, and
`Transformer(args, with_visual=False)` with `forward_inference(tokens[bsz,seqlen], start_pos) -> fp32
[bsz, vocab]`, `forward(examples)`, `_allocate_kv_cache`, `_destroy_kv_cache`, `get_trainable_params`,
`args`, `image_words`, `cache_image_words`, `layers`, and the reference's state-dict keys
(tok_embeddings / layers.{i}.attention.{wq,wk,wv,wo} / feed_forward.{w1,w2,w3} / *_norm / norm / output).

The parameters only exist to receive a checkpoint; the first inference call quantises them
(OmniQuant-style W{2,3,4}A16, `ModelArgs.wbits / group_size`), packs them for the C-ABI engine and frees
the fp16 copies.  All arithmetic then runs in libb200decode.so; there is no PyTorch fallback.
"""
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from .. import parallel_layers as pl
from ..engine import DecodeEngine, EngineConfig, llama_ffn_hidden
from ..parallel_layers import ColumnParallelLinear, ParallelEmbedding, RowParallelLinear


@dataclass
class ModelArgs:
    # llama.py:28-43
    dim: int = 4096
    n_layers: int = 32
    n_heads: int = 32
    n_kv_heads: Optional[int] = None
    vocab_size: int = -1
    multiple_of: int = 256
    ffn_dim_multiplier: Optional[float] = None
    norm_eps: float = 1e-5
    rope_theta: float = 10000
    max_batch_size: int = 32
    max_seq_len: int = 2048
    rope_scaling: Optional[float] = None
    # engine knobs (JSON-configurable like every other field, meta.py:33-45)
    wbits: int = 4
    group_size: int = 0


class RMSNorm(nn.Module):
    """Parameter holder (components.py:24-26); the normalisation itself is fused into the next GEMV."""

    def __init__(self, dim, eps=1e-6):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(dim))


class Attention(nn.Module):
    def __init__(self, args):
        super().__init__()
        n_kv = args.n_heads if args.n_kv_heads is None else args.n_kv_heads
        hd = args.dim // args.n_heads
        self.wq = ColumnParallelLinear(args.dim, args.n_heads * hd, bias=False, gather_output=False, init_method=None)
        self.wk = ColumnParallelLinear(args.dim, n_kv * hd, bias=False, gather_output=False, init_method=None)
        self.wv = ColumnParallelLinear(args.dim, n_kv * hd, bias=False, gather_output=False, init_method=None)
        self.wo = RowParallelLinear(args.n_heads * hd, args.dim, bias=False, input_is_parallel=True, init_method=None)


class FeedForward(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.w1 = ColumnParallelLinear(dim, hidden, bias=False, gather_output=False, init_method=None)
        self.w2 = RowParallelLinear(hidden, dim, bias=False, input_is_parallel=True, init_method=None)
        self.w3 = ColumnParallelLinear(dim, hidden, bias=False, gather_output=False, init_method=None)


class TransformerBlock(nn.Module):
    def __init__(self, layer_id, args):
        super().__init__()
        self.layer_id = layer_id
        self.attention = Attention(args)
        self.feed_forward = FeedForward(args.dim, llama_ffn_hidden(args.dim, args.multiple_of, args.ffn_dim_multiplier))
        self.attention_norm = RMSNorm(args.dim, eps=args.norm_eps)
        self.ffn_norm = RMSNorm(args.dim, eps=args.norm_eps)


class Transformer(nn.Module):
    KIND = "llama"

    def __init__(self, args: ModelArgs, with_visual=False):
        super().__init__()
        if with_visual:
            raise NotImplementedError("llama_b200 covers the text decode hot path; visual prefixes are out of scope")
        self.args = args
        self.vocab_size = args.vocab_size
        self.n_layers = args.n_layers
        self.image_words = 0
        self.cache_image_words = 0
        self.engine: Optional[DecodeEngine] = None
        self._build_modules(args)

    def _build_modules(self, args):
        self.tok_embeddings = ParallelEmbedding(args.vocab_size, args.dim, init_method=None)
        self.layers = nn.ModuleList([TransformerBlock(i, args) for i in range(args.n_layers)])
        self.norm = RMSNorm(args.dim, eps=args.norm_eps)
        self.output = ColumnParallelLinear(args.dim, args.vocab_size, bias=False, init_method=None)

    # ---- engine construction ---------------------------------------------------------------
    @classmethod
    def from_engine(cls, engine: DecodeEngine):
        """Wrap an already-built engine (bench.py: weights generated directly in packed form)."""
        self = cls.__new__(cls)
        nn.Module.__init__(self)
        c = engine.cfg
        self.args = ModelArgs(dim=c.dim, n_layers=c.n_layers, n_heads=c.n_heads, n_kv_heads=c.n_kv_heads,
                              vocab_size=c.vocab_size, norm_eps=c.norm_eps, rope_theta=c.rope_theta,
                              max_batch_size=c.max_batch_size, max_seq_len=c.max_seq_len, wbits=c.bits,
                              group_size=c.group_size)
        self.vocab_size, self.n_layers = c.vocab_size, c.n_layers
        self.image_words = self.cache_image_words = 0
        self.layers = nn.ModuleList()
        self.engine = engine
        return self

    def _engine_config(self, device):
        a = self.args
        return EngineConfig.from_model_args(
            self.KIND, {k: getattr(a, k) for k in a.__dataclass_fields__ if k not in ("wbits", "group_size")},
            bits=a.wbits, group_size=a.group_size, tp_rank=pl.get_model_parallel_rank(),
            tp_world=pl.get_model_parallel_world_size())

    def _local_state_dict(self):
        return {k: v.detach() for k, v in self.state_dict().items()}

    def build_engine(self, free_params=True):
        """Quantise + pack this rank's shards (rank-local min/max quantisation) and hand them to the engine."""
        dev = self.norm.weight.device
        if dev.type != "cuda":
            raise RuntimeError("llama_b200 needs its parameters on a CUDA device (no CPU fallback)")
        cfg = self._engine_config(dev)
        eng = DecodeEngine(cfg, dev, group=pl.get_model_parallel_group())
        eng.load_local_state_dict(self._local_state_dict())
        self.engine = eng
        if free_params:
            for p in self.parameters():
                p.data = torch.empty(0, dtype=p.dtype, device=p.device)
        return eng

    # ---- reference surface -----------------------------------------------------------------
    def get_trainable_params(self):
        return {}

    @torch.inference_mode()
    def forward_inference(self, tokens: torch.Tensor, start_pos: int, image=None):
        """llama.py:394-427."""
        if image is not None:
            raise NotImplementedError("image prefixes are out of scope for llama_b200")
        if self.engine is None:
            self.build_engine()
        if start_pos == 0:
            self.cache_image_words = 0
        # a fresh tensor like the reference's output(h).float() (llama.py:426-427): the engine's decode step returns a view of
        # its static graph output buffer, which the next step overwrites
        return self.engine.forward_inference(tokens, start_pos).clone()

    @torch.inference_mode()
    def forward(self, examples, image=None):
        """llama.py:373-391 (inference use: MetaModel.compute_logits): full-sequence logits, kills the KV cache."""
        if image is not None:
            raise NotImplementedError("image prefixes are out of scope for llama_b200")
        if self.engine is None:
            self.build_engine()
        out = self.engine.forward_full(examples)
        self._destroy_kv_cache()
        return out

    def _allocate_kv_cache(self, max_batch_size: int) -> None:
        if self.engine is not None:
            self.engine.allocate_kv_cache(max_batch_size)

    def _destroy_kv_cache(self) -> None:
        if self.engine is not None:
            self.engine.destroy_kv_cache()
