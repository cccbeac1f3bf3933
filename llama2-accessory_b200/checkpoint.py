"""On-disk formats either side of the decode path (SURVEY.md 8f, rank 1): the reference's tensor-parallel
checkpoint folders in, the engine's packed W-bit shards out.

Mirrors the behaviour of accessory/util/tensor_parallel.py without needing an nn.Module instance (the engine
has no parameters to match against, so the tensor-parallel dimension of a tensor is derived from its key):

  * formats (tensor_parallel.py:40-45): ``meta_ori``  consolidated.NN.pth (keys without the ``llma.`` prefix),
    ``consolidated``  consolidated.NN-of-MM.model.pth (optionally wrapped in {"model": ...}, :219-226),
    ``consolidated_diff``  consolidated.NN-of-MM.model-diff.pth (values ADDED to the keys already loaded, :387-422);
  * format / tensor-parallel size inference from the folder listing (:333-384) with the same failure mode
    (NotImplementedError) for unknown, mixed or incomplete folders;
  * change of tensor-parallel size on load: merge ranks when ckpt_mp % tp == 0 (:83-130), split a rank when
    tp % ckpt_mp == 0 (:133-161), otherwise NotImplementedError (:164-168);
  * sharding dims (:34-38): ColumnParallelLinear weight dim 0, RowParallelLinear weight dim 1,
    ParallelEmbedding weight dim 1, everything else replicated; Mixtral experts live whole on the rank that
    owns their id (mixtral.py:237-241);
  * ``meta.json`` / ``config.json`` / tokenizer probing of MetaModel.from_pretrained (meta.py:157-186,
    tokenizer.py:134-156).

Plus what the reference does not have: recovering (q, scale, zero) from an OmniQuant *fake-quantised* fp16
checkpoint (weights stored as dequant(quant(W))), and saving / loading the engine's packed shards so that a
model is quantised and packed once, offline.
"""
import json
import os
import re
from collections import OrderedDict
from collections.abc import Mapping
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from .quant import PackedLinear, dequantize

FORMAT_FILENAME_PATTERNS: Dict[str, "re.Pattern"] = {
    "meta_ori": re.compile(r"^consolidated\.(\d{2})\.pth$"),
    "consolidated": re.compile(r"^consolidated\.(\d{2})-of-(\d{2})\.model\.pth$"),
    "consolidated_diff": re.compile(r"^consolidated\.(\d{2})-of-(\d{2})\.model-diff\.pth$"),
}

_COLUMN = re.compile(r"(^|\.)(attention\.w[qkv]|feed_forward\.w[13]|output)\.weight$")
_ROW = re.compile(r"(^|\.)(attention\.wo|feed_forward\.w2)\.weight$")
_EMBED = re.compile(r"(^|\.)tok_embeddings\.weight$")
_EXPERT = re.compile(r"(^|\.)feed_forward\.experts\.(\d+)\.w[123]\.weight$")


def get_tensor_parallel_shards_file_name(format: str, mp_size: int) -> List[str]:
    """File name of every tensor-parallel shard of a checkpoint (tensor_parallel.py:171-197)."""
    if format == "meta_ori":
        return [f"consolidated.{i:02d}.pth" for i in range(mp_size)]
    if format == "consolidated":
        return [f"consolidated.{i:02d}-of-{mp_size:02d}.model.pth" for i in range(mp_size)]
    if format == "consolidated_diff":
        return [f"consolidated.{i:02d}-of-{mp_size:02d}.model-diff.pth" for i in range(mp_size)]
    raise NotImplementedError(f"Checkpoint format {format} is unknown.")


def infer_checkpoint_format_and_mp_size(path: str) -> Tuple[str, int]:
    """(format, tensor-parallel size) of a checkpoint folder (tensor_parallel.py:333-384)."""
    if not os.path.isdir(path):
        raise NotImplementedError("The given path does not point to a valid folder.")
    files = [fn for fn in os.listdir(path) if os.path.isfile(os.path.join(path, fn))]
    found = [(fmt, [fn for fn in files if pat.match(fn)]) for fmt, pat in FORMAT_FILENAME_PATTERNS.items()]
    found = [(fmt, fns) for fmt, fns in found if fns]
    if not found:
        raise NotImplementedError(f"Files in the given folder do not match any format. Contents: {sorted(os.listdir(path))}.")
    if len(found) > 1:
        raise NotImplementedError(f"Multiple matched format detected: {found[0][0]} and {found[1][0]}.")
    fmt, fns = found[0]
    for fn in get_tensor_parallel_shards_file_name(fmt, len(fns)):
        if fn not in files:
            raise NotImplementedError("An expected file is not found in the target folder: " + fn)
    return fmt, len(fns)


def load_tensor_parallel_shard_state_dict(path: str, format: str, shard_id: int, num_shards: int) -> Dict[str, torch.Tensor]:
    """One rank's state dict as stored, keys normalised to carry the ``llma.`` prefix (tensor_parallel.py:200-226)."""
    fn = os.path.join(path, get_tensor_parallel_shards_file_name(format, num_shards)[shard_id])
    try:  # memory-mapped: a 70B shard is never resident as a whole, pages come in as tensors are touched
        shard = torch.load(fn, map_location="cpu", weights_only=True, mmap=True)
    except (RuntimeError, ValueError, TypeError):  # legacy (non-zipfile) serialisation cannot be mapped
        shard = torch.load(fn, map_location="cpu", weights_only=True)
    if format.startswith("consolidated"):
        if "model" in shard and isinstance(shard["model"], dict):
            shard = shard["model"]
    elif format == "meta_ori":
        shard = {"llma." + k: v for k, v in shard.items()}
    return shard


def weight_parallel_dim(key: str) -> Optional[int]:
    """Dimension along which the reference shards this tensor, None when it is replicated."""
    if _EXPERT.search(key):
        return None  # whole experts: ownership by id, never sliced
    if _COLUMN.search(key):
        return 0
    if _ROW.search(key) or _EMBED.search(key):
        return 1
    return None


def _expert_id(key: str) -> Optional[int]:
    m = _EXPERT.search(key)
    return int(m.group(2)) if m else None


def _num_experts(keys) -> int:
    ids = [e for e in (_expert_id(k) for k in keys) if e is not None]
    return max(ids) + 1 if ids else 0


def load_tensor_parallel_state_dict(path: str, tp_rank: int = 0, tp_world: int = 1, format: Optional[str] = None,
                                    verbose: bool = False) -> "OrderedDict[str, torch.Tensor]":
    """The state dict local to tensor-parallel rank `tp_rank` of `tp_world`, re-sharded from whatever
    tensor-parallel size the checkpoint was saved with (tensor_parallel.py:229-296)."""
    if format is None:
        format, ckpt_mp = infer_checkpoint_format_and_mp_size(path)
    else:
        ckpt_mp = len([fn for fn in os.listdir(path) if FORMAT_FILENAME_PATTERNS[format].match(fn)])
        if ckpt_mp == 0:
            raise AssertionError(f'"{path}" is not a valid {format} format checkpoint path: no file with valid name is found.')
    out: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    if ckpt_mp % tp_world == 0:
        # ---- merge ckpt_mp / tp_world consecutive checkpoint ranks into this rank ----
        n_local = ckpt_mp // tp_world
        shards = [load_tensor_parallel_shard_state_dict(path, format, s, ckpt_mp)
                  for s in range(n_local * tp_rank, n_local * (tp_rank + 1))]
        keys = list(OrderedDict.fromkeys(k for sh in shards for k in sh))
        for key in keys:
            parts = [sh[key] for sh in shards if key in sh]
            dim = weight_parallel_dim(key)
            if dim is not None:
                out[key] = torch.cat(parts, dim=dim) if len(parts) > 1 else parts[0]
            else:
                if verbose and any(not torch.equal(parts[0], p) for p in parts[1:]):
                    print(f"WARNING! Found unequal replicas of non-tensor-parallel params: name={key}")
                out[key] = parts[0]
            for sh in shards:
                sh.pop(key, None)
    elif tp_world % ckpt_mp == 0:
        # ---- split one checkpoint rank between tp_world / ckpt_mp ranks ----
        split_to = tp_world // ckpt_mp
        shard = load_tensor_parallel_shard_state_dict(path, format, tp_rank // split_to, ckpt_mp)
        split_id = tp_rank % split_to
        n_exp = None
        for key, val in shard.items():
            e = _expert_id(key)
            if e is not None:
                # this checkpoint rank holds a contiguous id range of whole experts; hand each new rank its slice
                if n_exp is None:
                    ids = sorted({_expert_id(k) for k in shard if _expert_id(k) is not None})
                    n_exp = (ids[0], len(ids))
                first, count = n_exp
                if count % split_to:
                    raise NotImplementedError("experts of a checkpoint rank do not divide over the new ranks")
                per = count // split_to
                if first + per * split_id <= e < first + per * (split_id + 1):
                    out[key] = val
                continue
            dim = weight_parallel_dim(key)
            out[key] = torch.chunk(val, split_to, dim)[split_id].contiguous() if dim is not None else val
    else:
        raise NotImplementedError(f"cannot redistribute a tensor-parallel size {ckpt_mp} checkpoint over {tp_world} ranks")
    return out


class LazyMergedStateDict(Mapping):
    """The TP = 1 (or rank-local) view of ONE checkpoint folder that merges / slices a tensor only when it is asked for and
    keeps nothing: with memory-mapped shards the peak host memory of loading is one merged tensor, not the model
    (LLaMA2-70B: ~140 GB per rank with the eager loader, times 8 ranks on one node).  Same values, key order and
    ``llma.``-less names as ``load_tensor_parallel_state_dict_list([path], tp_rank, tp_world)``; supports the merge direction
    (checkpoint TP size a multiple of tp_world) -- the split direction and ``*_diff`` chains use the eager loader."""

    def __init__(self, path: str, tp_rank: int = 0, tp_world: int = 1):
        fmt, ckpt_mp = infer_checkpoint_format_and_mp_size(path)
        if fmt.endswith("_diff"):
            raise AssertionError("The first checkpoint in the list cannot be a *_diff checkpoint.")
        if ckpt_mp % tp_world:
            raise NotImplementedError("LazyMergedStateDict covers checkpoint TP sizes that are multiples of tp_world")
        n_local = ckpt_mp // tp_world
        self._shards = [load_tensor_parallel_shard_state_dict(path, fmt, s, ckpt_mp)
                        for s in range(n_local * tp_rank, n_local * (tp_rank + 1))]
        strip = lambda k: k[5:] if k.startswith("llma.") else k  # noqa: E731
        self._raw = OrderedDict((strip(k), k) for sh in self._shards for k in sh)

    def __len__(self):
        return len(self._raw)

    def __iter__(self):
        return iter(self._raw)

    def __contains__(self, key):
        return key in self._raw

    def __getitem__(self, key):
        raw = self._raw[key]
        parts = [sh[raw] for sh in self._shards if raw in sh]
        dim = weight_parallel_dim(raw)
        if dim is not None and len(parts) > 1:
            return torch.cat(parts, dim=dim)
        return parts[0]


class LazyQuantRecords(Mapping):
    """quant_records for DecodeEngine.load_master_state_dict computed per key on demand from a fake-quantised state dict
    (recover_quant_records without holding the integers of every linear at once)."""

    def __init__(self, sd: Mapping, bits: int, group_size: int = 0, check: bool = True):
        self._sd, self._bits, self._gs, self._check = sd, bits, group_size, check
        self._keys = [k for k in sd if QUANTISED_KEY.search(k[5:] if k.startswith("llma.") else k)]

    def __len__(self):
        return len(self._keys)

    def __iter__(self):
        return iter(self._keys)

    def __contains__(self, key):
        return key in self._sd and bool(QUANTISED_KEY.search(key))

    def __getitem__(self, key):
        w = self._sd[key]
        q, s, z, g = recover_quant_from_fake(w, self._bits, self._gs)
        if self._check and not torch.equal(dequantize(q, s, z, g), w.to(torch.float16)):
            raise ValueError(f"{key}: recovered (q, scale, zero) do not reproduce the checkpoint bit-exactly")
        return {"q": q, "scale": s, "zero": z, "group_size": g}


def load_tensor_parallel_state_dict_list(path_list: Union[str, Sequence[str]], tp_rank: int = 0, tp_world: int = 1,
                                         verbose: bool = False) -> "OrderedDict[str, torch.Tensor]":
    """Checkpoints applied in order: a base format overrides earlier values of a key, a ``*_diff`` format is
    added to them (tensor_parallel.py:425-483, :387-422).  Returns this rank's state dict (``llma.`` stripped)."""
    if isinstance(path_list, str):
        path_list = [path_list]
    acc: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for i, path in enumerate(path_list):
        fmt, _ = infer_checkpoint_format_and_mp_size(path)
        if i == 0 and fmt.endswith("_diff"):
            raise AssertionError("The first checkpoint in the list cannot be a *_diff checkpoint.")
        sd = load_tensor_parallel_state_dict(path, tp_rank, tp_world, fmt, verbose)
        for key, val in sd.items():
            if fmt.endswith("_diff") and key in acc:
                acc[key] = acc[key] + val.to(acc[key].dtype)
            else:
                if verbose and key in acc:
                    print(f"A key ({key}) is overrided by a full checkpoint (at {path}).")
                acc[key] = val
    return OrderedDict(((k[5:] if k.startswith("llma.") else k), v) for k, v in acc.items())


def save_tensor_parallel_shards(master_sd: Dict[str, torch.Tensor], path: str, mp_size: int, format: str = "consolidated",
                                wrap_model: bool = True) -> List[str]:
    """Write a TP = 1 state dict as an `mp_size`-way checkpoint folder in one of the reference's formats
    (the layout misc.py's save path produces: every rank holds its Column / Row / Embedding slice, replicated
    tensors in every file, Mixtral experts in the file of the owning rank)."""
    os.makedirs(path, exist_ok=True)
    n_exp = _num_experts(master_sd.keys())
    if n_exp and n_exp % mp_size:
        raise ValueError("num_experts must be divisible by the tensor-parallel size")
    fns = get_tensor_parallel_shards_file_name(format, mp_size)
    for r, fn in enumerate(fns):
        sd = OrderedDict()
        for key, val in master_sd.items():
            k = key[5:] if key.startswith("llma.") else key
            e = _expert_id(k)
            if e is not None:
                per = n_exp // mp_size
                if not (per * r <= e < per * (r + 1)):
                    continue
                piece = val
            else:
                dim = weight_parallel_dim(k)
                piece = torch.chunk(val, mp_size, dim)[r].contiguous() if dim is not None else val
            sd[k if format == "meta_ori" else "llma." + k] = piece.clone()
        torch.save({"model": sd} if (wrap_model and format != "meta_ori") else sd, os.path.join(path, fn))
    return fns


# ---------------------------------------------------------------------------------------------------
# meta.json / config.json / tokenizer probing
# ---------------------------------------------------------------------------------------------------
def probe_tokenizer_path_from_pretrained(pretrained_path: str) -> Optional[str]:
    """sentencepiece ``tokenizer.model`` first, then a HuggingFace pair (tokenizer.py:134-156)."""
    spm = os.path.join(pretrained_path, "tokenizer.model")
    if os.path.exists(spm):
        return spm
    if all(os.path.exists(os.path.join(pretrained_path, f)) for f in ("tokenizer.json", "tokenizer_config.json")):
        return pretrained_path
    return None


def read_model_meta(pretrained_path: Union[str, Sequence[str]], llama_type: Optional[str] = None,
                    llama_config: Optional[Sequence[str]] = None) -> dict:
    """What MetaModel.from_pretrained derives from the LAST checkpoint folder (meta.py:157-186): ``llama_type`` from
    meta.json (ValueError when it cannot be determined), model arguments from config.json (defaults of the model's
    ModelArgs when absent; several config files are merged in order, meta.py:58-63), the tokenizer path."""
    last = pretrained_path if isinstance(pretrained_path, str) else pretrained_path[-1]
    if llama_type is None:
        mj = os.path.join(last, "meta.json")
        if not os.path.exists(mj):
            raise ValueError("Cannot determine llama_type")
        with open(mj) as f:
            llama_type = json.load(f)["llama_type"]
    if llama_config is None:
        cj = os.path.join(last, "config.json")
        llama_config = [cj] if os.path.exists(cj) else []
    elif isinstance(llama_config, str):
        llama_config = [llama_config]
    params = {}
    for cfg in llama_config:
        with open(cfg) as f:
            params.update(json.load(f))
    return {"llama_type": llama_type, "config": params, "tokenizer_path": probe_tokenizer_path_from_pretrained(last)}


# ---------------------------------------------------------------------------------------------------
# OmniQuant fake-quantised fp16 checkpoint -> (q, scale, zero)
# ---------------------------------------------------------------------------------------------------
QUANTISED_KEY = re.compile(r"(^|\.)(attention\.w[qkvo]|feed_forward\.w[123]|feed_forward\.experts\.\d+\.w[123])\.weight$")


def recover_quant_from_fake(w16: torch.Tensor, bits: int, group_size: int = 0):
    """Invert OmniQuant's fake quantisation.  `w16` [N, K] fp16 holds  fp16(fp16(q - z) * s16)  per group of
    `group_size` input features (0 = one group per output channel).  Returns (q uint8 [N,K], scale fp16 [N,G],
    zero fp16 [N,G], g) that reproduce `w16` BIT-EXACTLY through quant.dequantize.

    Only q - z is observable, so the pair is normalised to q_min = 0 (z = -n_min): any level set that an
    asymmetric b-bit quantiser can emit maps to a valid (q, z).  Raises ValueError if some group is not a b-bit
    uniform grid (i.e. the checkpoint was not quantised with these settings)."""
    assert w16.dim() == 2 and bits in (2, 3, 4)
    N, K = w16.shape
    g = K if (not group_size or group_size <= 0 or group_size >= K) else int(group_size)
    if K % g:
        raise ValueError(f"K={K} is not a multiple of group_size={g}")
    G = K // g
    v = w16.detach().to(torch.float16).float().reshape(N * G, g)
    levels = 2 ** bits - 1
    srt, _ = torch.sort(v, dim=1)
    d = srt[:, 1:] - srt[:, :-1]
    big = torch.finfo(torch.float32).max
    dmin = torch.where(d > 0, d, torch.full_like(d, big)).amin(dim=1)          # smallest gap between two levels
    const = dmin == big                                                         # single-level group
    vabs = v.abs().amax(dim=1)
    s_gap = torch.where(const, torch.where(vabs > 0, vabs, torch.ones_like(vabs)), dmin)
    target = v.to(torch.float16)
    n = torch.zeros_like(v)
    scale = torch.zeros(N * G, dtype=torch.float16)
    done = torch.zeros(N * G, dtype=torch.bool)
    # the smallest gap is one step unless every pair of neighbouring levels is absent from the group; then it is a
    # small multiple of the step: retry the unresolved groups with gap/2, gap/3, gap/4
    for div in (1, 2, 3, 4):
        todo = ~done
        if not bool(todo.any()):
            break
        vt = v[todo]
        s0 = s_gap[todo] / div
        nt = torch.round(vt / s0[:, None])
        # least-squares refinement of the step (the gap of two fp16-rounded levels is only good to ~1e-3 relative)
        nn_ = (nt * nt).sum(1)
        s_ls = torch.where(nn_ > 0, (nt * vt).sum(1) / nn_.clamp_min(1.0), s0)
        nt = torch.round(vt / s_ls[:, None])
        ok_rng = nt.abs().amax(dim=1) <= 2048
        n16 = nt.clamp(-2048, 2048).to(torch.float16)
        # the stored scale is an fp16 number next to the estimate: test the neighbours for bit-exact reproduction
        bits16 = s_ls.to(torch.float16).view(torch.int16).to(torch.int32)
        sc_t = torch.zeros(vt.shape[0], dtype=torch.float16)
        done_t = torch.zeros(vt.shape[0], dtype=torch.bool)
        for off in (0, 1, -1, 2, -2, 3, -3, 4, -4):
            cand = (bits16 + off).clamp(1, 0x7BFF).to(torch.int16).view(torch.float16)
            ok = ((n16 * cand[:, None]).to(torch.float16) == target[todo]).all(dim=1) & ok_rng & ~done_t
            sc_t = torch.where(ok, cand, sc_t)
            done_t |= ok
            if bool(done_t.all()):
                break
        idx = torch.nonzero(todo).squeeze(1)[done_t]
        n[idx] = nt[done_t]
        scale[idx] = sc_t[done_t]
        done[idx] = True
    if not bool(done.all()):
        raise ValueError(f"{int((~done).sum())} of {N * G} groups are not a W{bits} uniform grid with group size {g}")
    nmin = n.amin(dim=1, keepdim=True)
    q = n - nmin
    if float(q.max()) > levels:
        raise ValueError(f"more than {levels + 1} levels in a group: not a W{bits} checkpoint")
    zero = (-nmin).squeeze(1)
    if float(zero.abs().max()) > 1024:
        raise ValueError("|zero point| > 1024 is not representable in the packed format")
    return (q.to(torch.uint8).reshape(N, K), scale.reshape(N, G), zero.to(torch.float16).reshape(N, G), g)


def recover_quant_records(sd: Dict[str, torch.Tensor], bits: int, group_size: int = 0, check: bool = True) -> Dict[str, dict]:
    """quant_records for DecodeEngine.load_master_state_dict from a fake-quantised MASTER state dict: every
    attention / feed-forward / expert linear (embeddings, norms, the lm_head and the MoE router stay fp16,
    SURVEY.md 8c)."""
    recs = {}
    for key, w in sd.items():
        k = key[5:] if key.startswith("llma.") else key
        if not QUANTISED_KEY.search(k):
            continue
        q, s, z, g = recover_quant_from_fake(w, bits, group_size)
        if check and not torch.equal(dequantize(q, s, z, g), w.to(torch.float16)):
            raise ValueError(f"{key}: recovered (q, scale, zero) do not reproduce the checkpoint bit-exactly")
        recs[k] = {"q": q, "scale": s, "zero": z, "group_size": g}
    return recs


# ---------------------------------------------------------------------------------------------------
# packed engine shards on disk
# ---------------------------------------------------------------------------------------------------
def _pl_to_dict(pl: Optional[PackedLinear]):
    if pl is None:
        return None
    return {"bits": pl.bits, "N": pl.N, "K": pl.K, "group_size": pl.group_size, "qweight": pl.qweight.cpu(),
            "scales": None if pl.scales is None else pl.scales.cpu()}


def _pl_from_dict(d, device) -> Optional[PackedLinear]:
    if d is None:
        return None
    return PackedLinear(d["bits"], d["N"], d["K"], d["group_size"], d["qweight"].to(device),
                        None if d["scales"] is None else d["scales"].to(device))


PACKED_FORMAT_VERSION = 1


def packed_shard_file_name(tp_rank: int, tp_world: int) -> str:
    return f"b200_packed.{tp_rank:02d}-of-{tp_world:02d}.pth"


def save_packed(engine, path: str) -> str:
    """Write this rank's packed weights (the exact device images the kernels stream) next to the engine config."""
    from dataclasses import asdict
    os.makedirs(path, exist_ok=True)
    c = engine.cfg
    layers = []
    for lw in engine.layers:
        layers.append({"attn_norm": lw.attn_norm.cpu(), "ffn_norm": lw.ffn_norm.cpu(), "wqkv": _pl_to_dict(lw.wqkv),
                       "wo": _pl_to_dict(lw.wo), "w13": _pl_to_dict(lw.w13), "w2": _pl_to_dict(lw.w2),
                       "gate": None if lw.gate is None else lw.gate.cpu(),
                       "e_w13": [_pl_to_dict(p) for p in lw.e_w13], "e_w2": [_pl_to_dict(p) for p in lw.e_w2]})
    blob = {"version": PACKED_FORMAT_VERSION, "config": asdict(c), "tok_emb": engine.tok_emb.cpu(),
            "final_norm": engine.final_norm.cpu(), "lm_head": _pl_to_dict(engine.lm_head), "layers": layers}
    fn = os.path.join(path, packed_shard_file_name(c.tp_rank, c.tp_world))
    torch.save(blob, fn)
    return fn


def load_packed(engine, path: str):
    """Load a shard written by save_packed into an engine built with the same configuration."""
    from dataclasses import asdict
    c = engine.cfg
    blob = torch.load(os.path.join(path, packed_shard_file_name(c.tp_rank, c.tp_world)), map_location="cpu",
                      weights_only=False)
    if blob.get("version") != PACKED_FORMAT_VERSION:
        raise ValueError(f"packed shard version {blob.get('version')} != {PACKED_FORMAT_VERSION}")
    mine, theirs = asdict(c), blob["config"]
    for k in ("kind", "dim", "n_layers", "n_heads", "n_kv_heads", "ffn_hidden", "vocab_size", "num_experts",
              "experts_per_tok", "bits", "group_size", "tp_rank", "tp_world"):
        if mine[k] != theirs[k]:
            raise ValueError(f"packed shard was written for {k}={theirs[k]}, engine has {k}={mine[k]}")
    dev = engine.device
    engine.tok_emb = blob["tok_emb"].to(dev)
    engine.final_norm = blob["final_norm"].to(dev)
    engine.lm_head = _pl_from_dict(blob["lm_head"], dev)
    for lw, d in zip(engine.layers, blob["layers"]):
        lw.attn_norm, lw.ffn_norm = d["attn_norm"].to(dev), d["ffn_norm"].to(dev)
        lw.wqkv, lw.wo = _pl_from_dict(d["wqkv"], dev), _pl_from_dict(d["wo"], dev)
        lw.w13, lw.w2 = _pl_from_dict(d["w13"], dev), _pl_from_dict(d["w2"], dev)
        lw.gate = None if d["gate"] is None else d["gate"].to(dev)
        lw.e_w13 = [_pl_from_dict(p, dev) for p in d["e_w13"]]
        lw.e_w2 = [_pl_from_dict(p, dev) for p in d["e_w2"]]
    return engine


# ---------------------------------------------------------------------------------------------------
# one call: checkpoint folder(s) -> engine
# ---------------------------------------------------------------------------------------------------
_KIND_OF_TYPE = {"llama": "llama", "llama_b200": "llama", "mixtral": "mixtral", "mixtral_b200": "mixtral"}


def build_engine_from_pretrained(pretrained_path: Union[str, Sequence[str]], *, llama_type: Optional[str] = None,
                                 llama_config: Optional[Sequence[str]] = None, bits: int = 4, group_size: int = 0,
                                 fake_quantised: bool = False, max_seq_len: int = 4096, max_batch_size: int = 32,
                                 device="cuda", tp_rank: int = 0, tp_world: int = 1, group=None):
    """MetaModel.from_pretrained's loading steps (meta.py:157-196) ending in a DecodeEngine: probe meta.json /
    config.json, load (and re-shard) the checkpoint list, quantise -- or, for an OmniQuant fake-quantised
    checkpoint, recover the stored integers -- and pack.

    Quantisation needs the MASTER weights (quantise, then shard: SURVEY.md 8e), so every rank reads the merged
    TP = 1 tensors and keeps its own slice."""
    from .engine import DecodeEngine, EngineConfig
    meta = read_model_meta(pretrained_path, llama_type, llama_config)
    kind = _KIND_OF_TYPE.get(meta["llama_type"])
    if kind is None:
        raise ValueError(f"llama_type {meta['llama_type']!r} is not served by this decode engine")
    args = dict(meta["config"])
    args.setdefault("vocab_size", 32000)
    args["max_seq_len"], args["max_batch_size"] = max_seq_len, max_batch_size
    if kind == "llama":  # defaults of llama.py:28-43
        for k, dflt in (("dim", 4096), ("n_layers", 32), ("n_heads", 32), ("multiple_of", 256), ("norm_eps", 1e-5)):
            args.setdefault(k, dflt)
    else:  # defaults of mixtral.py:33-54
        for k, dflt in (("dim", 4096), ("hidden_dim", 16384), ("n_layers", 32), ("n_heads", 32), ("norm_eps", 1e-5),
                        ("rope_theta", 1000000.0), ("moe", {"num_experts_per_tok": 2, "num_experts": 8})):
            args.setdefault(k, dflt)
    cfg = EngineConfig.from_model_args(kind, args, bits=bits, group_size=group_size, tp_rank=tp_rank, tp_world=tp_world)
    eng = DecodeEngine(cfg, device, group=group)
    paths = [pretrained_path] if isinstance(pretrained_path, str) else list(pretrained_path)
    if len(paths) == 1:
        # streaming: every linear is merged from the memory-mapped shards, quantised (or recovered), sharded, packed and
        # dropped before the next one is touched -- peak host memory is one merged tensor, not the master model
        sd = LazyMergedStateDict(paths[0], 0, 1)
        recs = LazyQuantRecords(sd, bits, group_size) if (fake_quantised and bits != 16) else None
    else:  # base + *_diff chains need the accumulated values: eager
        sd = load_tensor_parallel_state_dict_list(paths, 0, 1)
        recs = recover_quant_records(sd, bits, group_size) if (fake_quantised and bits != 16) else None
    eng.load_master_state_dict(sd, quant_records=recs)
    return eng, meta
