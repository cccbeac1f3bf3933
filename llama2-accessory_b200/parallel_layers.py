"""fairscale-style tensor-parallel layers (the API LLaMA2-Accessory imports from
`fairscale.nn.model_parallel.layers`, llama.py:10-15; signatures as subclassed at
accessory/model/peft.py:79-89,189-199) re-provided on top of the sm_90a kernels.

Parameters keep the reference's names and shard shapes (Column: [out/TP, in], Row: [out, in/TP],
Embedding here: full table replicated -- see DESIGN.md), so checkpoints load unchanged.  Inference
forward of an (un)quantised layer is one C-ABI GEMV launch; `quantize_omni` mirrors the mechanics of
accessory/util/quant.py:95-163 (attach `quanted_layer`, rebind `forward`, delete `weight`).
"""
from types import MethodType

import torch
import torch.distributed as dist
import torch.nn as nn

from . import ops
from .quant import PackedLinear, pack_fp16, pack_quantized, quantize_weight

_MP_GROUP = None


def set_model_parallel_group(group):
    global _MP_GROUP
    _MP_GROUP = group


def get_model_parallel_group():
    return _MP_GROUP


def get_model_parallel_world_size():
    return dist.get_world_size(group=_MP_GROUP) if (dist.is_available() and dist.is_initialized()) else 1


def get_model_parallel_rank():
    return dist.get_rank(group=_MP_GROUP) if (dist.is_available() and dist.is_initialized()) else 0


def copy_to_model_parallel_region(x):
    return x


def reduce_from_model_parallel_region(x):
    if get_model_parallel_world_size() > 1:
        dist.all_reduce(x, group=_MP_GROUP)
    return x


def gather_from_model_parallel_region(x):
    ws = get_model_parallel_world_size()
    if ws == 1:
        return x
    parts = [torch.empty_like(x) for _ in range(ws)]
    dist.all_gather(parts, x.contiguous(), group=_MP_GROUP)
    return torch.cat(parts, dim=-1)


def scatter_to_model_parallel_region(x):
    ws = get_model_parallel_world_size()
    return x if ws == 1 else x.chunk(ws, dim=-1)[get_model_parallel_rank()].contiguous()


class B200Linear(nn.Module):
    """The `quanted_layer` plug-in (quant.py:117-130 puts a bnb.nn.Linear4bit here): y = x @ W^T with W in
    the packed W{2,3,4,16} format, computed by b200_gemv.  x[..., in_local] -> [..., out_local] fp16."""

    def __init__(self, packed: PackedLinear):
        super().__init__()
        self.packed = packed
        self.in_features, self.out_features = packed.K, packed.N

    @torch.inference_mode()
    def forward(self, x):
        shp = x.shape
        x2 = x.reshape(-1, shp[-1]).to(torch.float16).contiguous()
        out = torch.empty((x2.shape[0], self.out_features), dtype=torch.float16, device=x2.device)
        for t0 in range(0, x2.shape[0], 32):
            t1 = min(x2.shape[0], t0 + 32)
            ops.gemv(self.packed, t1 - t0, xin=x2[t0:t1], out=out[t0:t1], epilogue=ops.B200_EPI_F16)
        return out.reshape(*shp[:-1], self.out_features).to(x.dtype)


class _ParallelLinearBase(nn.Module):
    def _packed_fp16(self):
        if getattr(self, "_packed", None) is None or self._packed_version != self.weight._version:
            self._packed = B200Linear(pack_fp16(self.weight.detach(), self.weight.device))
            self._packed_version = self.weight._version
        return self._packed

    def _matmul(self, x):
        if getattr(self, "quanted_layer", None) is not None:
            return self.quanted_layer(x)
        return self._packed_fp16()(x)


class ColumnParallelLinear(_ParallelLinearBase):
    def __init__(self, in_features, out_features, bias=True, gather_output=True,
                 init_method=nn.init.xavier_normal_, stride=1, keep_master_weight_for_test=False):
        super().__init__()
        ws = get_model_parallel_world_size()
        assert out_features % ws == 0
        self.in_features, self.out_features, self.gather_output = in_features, out_features, gather_output
        self.output_size_per_partition = out_features // ws
        self.weight = nn.Parameter(torch.empty(self.output_size_per_partition, in_features))
        self.weight.is_model_parallel = True
        self.bias = nn.Parameter(torch.zeros(self.output_size_per_partition)) if bias else None
        if init_method is not None:
            init_method(self.weight)

    def forward(self, x):  # quant.py:18-30
        y = self._matmul(copy_to_model_parallel_region(x))
        if self.bias is not None:
            y = y + self.bias
        return gather_from_model_parallel_region(y) if self.gather_output else y


class RowParallelLinear(_ParallelLinearBase):
    def __init__(self, in_features, out_features, bias=True, input_is_parallel=False,
                 init_method=nn.init.xavier_normal_, stride=1, keep_master_weight_for_test=False):
        super().__init__()
        ws = get_model_parallel_world_size()
        assert in_features % ws == 0
        self.in_features, self.out_features, self.input_is_parallel = in_features, out_features, input_is_parallel
        self.input_size_per_partition = in_features // ws
        self.weight = nn.Parameter(torch.empty(out_features, self.input_size_per_partition))
        self.weight.is_model_parallel = True
        self.bias = nn.Parameter(torch.zeros(out_features)) if bias else None
        if init_method is not None:
            init_method(self.weight)

    def forward(self, x):  # quant.py:32-46
        if not self.input_is_parallel:
            x = scatter_to_model_parallel_region(x)
        y = reduce_from_model_parallel_region(self._matmul(x))
        return y if self.bias is None else y + self.bias


class ParallelEmbedding(nn.Module):
    """llama.py:376: sharded along the embedding dim like fairscale ([vocab, D/TP]) so checkpoints load;
    forward all-gathers the shards (the engine itself keeps a full replicated table instead)."""

    def __init__(self, num_embeddings, embedding_dim, padding_idx=None, max_norm=None, norm_type=2.0,
                 scale_grad_by_freq=False, sparse=False, init_method=nn.init.xavier_normal_,
                 keep_master_weight_for_test=False):
        super().__init__()
        ws = get_model_parallel_world_size()
        assert embedding_dim % ws == 0
        self.num_embeddings, self.embedding_dim, self.padding_idx = num_embeddings, embedding_dim, padding_idx
        self.embedding_dim_per_partition = embedding_dim // ws
        self.weight = nn.Parameter(torch.empty(num_embeddings, self.embedding_dim_per_partition))
        self.weight.is_model_parallel = True
        if init_method is not None:
            init_method(self.weight)

    def forward(self, tokens):
        y = nn.functional.embedding(tokens, self.weight, self.padding_idx)
        return gather_from_model_parallel_region(y)


def _forward_quant(self, x):
    return type(self).forward(self, x)


def quantize_omni(model: nn.Module, wbits: int = 4, group_size: int = 0, blocklist=()):
    """OmniQuant-style counterpart of accessory/util/quant.py:95-163 `quantize(model, BitsAndBytesConfig)`:
    for every Column/RowParallelLinear (and nn.Linear) not in the blocklist and not a LoRA branch, attach
    `module.quanted_layer` (a B200Linear over the packed W-bit weight) and delete `module.weight`."""
    for name, mod in list(model.named_modules()):
        if "lora" in name or name in blocklist:
            continue
        if isinstance(mod, (ColumnParallelLinear, RowParallelLinear)) or type(mod) is nn.Linear:
            w = mod.weight.detach()
            q, s, z, g = quantize_weight(w, wbits, group_size)
            mod.quanted_layer = B200Linear(pack_quantized(q, s, z, wbits, 0 if g >= w.shape[1] else g, w.device))
            if type(mod) is nn.Linear:
                mod.forward = MethodType(lambda self, x: (self.quanted_layer(x) if self.bias is None
                                                          else self.quanted_layer(x) + self.bias), mod)
            del mod.weight
            mod.register_parameter("weight", None)
    return model
