"""MetaModel.generate / stream_generate / sample_top_p for the decode engine (SURVEY.md 8f rank 2).

Same signatures, argument meaning and results as accessory/model/meta.py:372-565, with the tokenizer handed in
(`MetaModel` owns one; here it is any object with the reference Tokenizer's methods: ``encode(s, bos, eos)``,
``decode(ids)``, ``eos_id``, ``encode_segment``, ``encode_wo_prefix_space``).

Two drivers produce the same tokens:

* the **host loop** follows meta.py:434-461 statement by statement over any model exposing
  ``forward_inference(tokens, start_pos)`` -- one host round trip per token, as the reference has;
* the **device loop** (default for an engine-backed model) keeps the whole step on the GPU: the decode step, token
  selection (`b200_argmax` / `b200_sample_top_p`) and the prompt-forcing / stop bookkeeping (`b200_generate_update`)
  are captured in ONE CUDA graph that is replayed `sync_every` times between host checks of the finished-sequence
  counter; the reference's per-token ``.item()`` / ``stopped.all()`` synchronisations (meta.py:458) disappear.

Token selection runs on the device in both drivers; tests inject ``select=`` to drive the host loop with a CPU model.
Images / visual prefixes are outside the decode hot path (NotImplementedError).
"""
from typing import Callable, Iterable, List, Optional

import torch

from . import _cabi, ops


def _device_of(model):
    """Where the loop's token buffers live: next to the engine, else next to the model's parameters."""
    eng = getattr(model, "engine", None)
    if eng is not None:
        return eng.device
    try:
        return next(model.parameters()).device
    except (StopIteration, AttributeError, TypeError):
        return torch.device("cuda" if torch.cuda.is_available() else "cpu")


def device_select(logits: torch.Tensor, temperature: float, top_p: float) -> torch.Tensor:
    """meta.py:438-443: greedy arg-max for temperature 0, else top-p sampling -- on the device, through the C ABI."""
    if not logits.is_cuda:
        raise RuntimeError("token selection runs on the GPU (b200_argmax / b200_sample_top_p); there is no CPU path")
    logits = logits.float().contiguous()
    T, V = logits.shape
    out = torch.empty(T, dtype=torch.int64, device=logits.device)
    if temperature > 0:
        u = torch.rand(T, dtype=torch.float32, device=logits.device)
        ops.sample_top_p(logits, u, out, T, V, temperature, top_p)
    else:
        ops.argmax(logits, out, T, V)
    return out


def sample_top_p(probs: torch.Tensor, p: float, uniform: Optional[torch.Tensor] = None) -> torch.Tensor:
    """MetaModel.sample_top_p (meta.py:550-565) for callers that already hold probabilities: [bsz, V] -> [bsz, 1]."""
    if not probs.is_cuda:
        raise RuntimeError("sample_top_p runs on the GPU; there is no CPU path")
    T, V = probs.shape
    logits = torch.log(probs.float().clamp_min(1e-38)).contiguous()  # softmax(log p) == p
    u = uniform if uniform is not None else torch.rand(T, dtype=torch.float32, device=probs.device)
    out = torch.empty(T, dtype=torch.int64, device=probs.device)
    ops.sample_top_p(logits, u.float().contiguous(), out, T, V, 1.0, p)
    return out.reshape(T, 1)


class _Plan:
    """What meta.py:399-432 computes before the loop."""

    def __init__(self, model, tokenizer, prompts, max_gen_len, additional_stop_symbols, device):
        if isinstance(prompts, str):
            raise ValueError("generate expects a batched LIST of prompts, but str is given")
        args = model.args
        self.bsz = len(prompts)
        assert self.bsz <= args.max_batch_size, (self.bsz, args.max_batch_size)
        toks = [tokenizer.encode(x, bos=True, eos=False) for x in prompts]
        self.min_prompt = min(len(t) for t in toks)
        max_prompt = max(len(t) for t in toks)
        max_seq_len = args.max_seq_len
        self.total_len = min(max_seq_len, max_gen_len + max_prompt)
        # left-truncate long prompts so that max_gen_len tokens still fit (meta.py:415-416)
        self.prompt_tokens = [t[-(max_seq_len - max_gen_len):] for t in toks]
        self.tokens = torch.zeros((self.bsz, self.total_len), dtype=torch.int64, device=device)
        self.mask = torch.zeros((self.bsz, self.total_len), dtype=torch.bool, device=device)
        for k, t in enumerate(self.prompt_tokens):
            self.tokens[k, :len(t)] = torch.tensor(t, dtype=torch.int64)
            self.mask[k, :len(t)] = True
        self.stop_lists = [[tokenizer.eos_id]]
        self.stop_lists += [list(tokenizer.encode_segment(s)) for s in additional_stop_symbols]
        self.stop_lists += [list(tokenizer.encode_wo_prefix_space(s)) for s in additional_stop_symbols]

    def decode(self, tokenizer, tokens_list, stop_pos_list) -> List[str]:
        return [tokenizer.decode(t[len(self.prompt_tokens[i]):stop_pos_list[i]]) for i, t in enumerate(tokens_list)]


def _host_loop(model, plan: _Plan, temperature, top_p, select):
    """meta.py:434-461."""
    tokens, mask = plan.tokens, plan.mask
    dev = tokens.device
    start_pos, prev_pos = plan.min_prompt, 0
    stops = [torch.tensor(s, dtype=tokens.dtype, device=dev) for s in plan.stop_lists]
    stopped = torch.zeros(plan.bsz, dtype=torch.bool, device=dev)
    stop_pos = torch.full((plan.bsz,), start_pos + 1, dtype=torch.int64, device=dev)
    for cur_pos in range(start_pos, plan.total_len):
        logits = model.forward_inference(tokens[:, prev_pos:cur_pos], prev_pos).float()
        next_token = select(logits, temperature, top_p).reshape(-1).to(dev)
        next_token = torch.where(mask[:, cur_pos], tokens[:, cur_pos], next_token)  # prompt tokens are forced
        tokens[:, cur_pos] = next_token
        stop_pos = torch.where(stopped, stop_pos, torch.full_like(stop_pos, cur_pos + 1))
        for st in stops:
            n = st.numel()
            if cur_pos + 1 - n >= 0:
                hit = (tokens[:, cur_pos + 1 - n:cur_pos + 1] == st.unsqueeze(0)).all(dim=-1)
                new_stop = hit & ~mask[:, cur_pos] & ~stopped
                stop_pos = torch.where(new_stop, torch.full_like(stop_pos, cur_pos + 1 - n), stop_pos)
                stopped = stopped | new_stop
        if bool(stopped.all()):
            break
        prev_pos = cur_pos
    return tokens.tolist(), [int(v) for v in stop_pos.tolist()]


def _device_loop(model, plan: _Plan, temperature, top_p, sync_every):
    """The same loop with every step resident on the device (one CUDA graph per step, polled every `sync_every`)."""
    eng = model.engine
    dev, bsz, total_len, start_pos = eng.device, plan.bsz, plan.total_len, plan.min_prompt
    if bsz > eng.t_max:
        raise ValueError(f"device generate loop handles up to {eng.t_max} sequences per call")
    tokens, mask = plan.tokens, plan.mask
    n_stop = len(plan.stop_lists)
    max_l = max(len(s) for s in plan.stop_lists)
    stop_seqs = torch.zeros((n_stop, max_l), dtype=torch.int64, device=dev)
    for i, s in enumerate(plan.stop_lists):
        stop_seqs[i, :len(s)] = torch.tensor(s, dtype=torch.int64)
    stop_lens = torch.tensor([len(s) for s in plan.stop_lists], dtype=torch.int32, device=dev)
    stopped = torch.zeros(bsz, dtype=torch.uint8, device=dev)
    stop_pos = torch.full((bsz,), start_pos + 1, dtype=torch.int32, device=dev)
    cur_pos = torch.full((1,), start_pos, dtype=torch.int32, device=dev)
    n_stopped = torch.zeros(1, dtype=torch.int32, device=dev)
    sampled = torch.zeros(bsz, dtype=torch.int64, device=dev)
    uniform = torch.zeros(bsz, dtype=torch.float32, device=dev)
    V = eng.cfg.vocab_size

    st = _cabi.GenerateState()
    st.bsz, st.total_len = bsz, total_len
    st.tokens, st.text_mask = tokens.data_ptr(), mask.data_ptr()
    st.stop_seqs, st.stop_lens, st.n_stop, st.max_stop_len = stop_seqs.data_ptr(), stop_lens.data_ptr(), n_stop, max_l
    st.stopped, st.stop_pos = stopped.data_ptr(), stop_pos.data_ptr()
    st.step_tokens, st.step_pos = eng.tokens.data_ptr(), eng.pos.data_ptr()
    st.cur_pos, st.n_stopped = cur_pos.data_ptr(), n_stopped.data_ptr()

    def select_into(logits):
        logits = logits.contiguous()
        if temperature > 0:
            uniform.uniform_(0.0, 1.0)
            ops.sample_top_p(logits, uniform, sampled, bsz, V, temperature, top_p)
        else:
            ops.argmax(logits, sampled, bsz, V)
        ops.generate_update(st, sampled)

    # prefill of the common prefix, first token
    logits = model.forward_inference(tokens[:, :start_pos], 0)
    select_into(logits.float())
    if total_len - (start_pos + 1) <= 0:
        torch.cuda.synchronize()
        return tokens.tolist(), [int(v) for v in stop_pos.tolist()]

    def body():
        select_into(eng._step(bsz, 1, eng.cache_seq))

    # warm-up once outside capture (lazy kernel attributes, NCCL), then restore the loop state it advanced
    keep = [t.clone() for t in (tokens, stopped, stop_pos, cur_pos, n_stopped, eng.tokens, eng.pos)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        body()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for dst, src in zip((tokens, stopped, stop_pos, cur_pos, n_stopped, eng.tokens, eng.pos), keep):
        dst.copy_(src)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()
    for dst, src in zip((tokens, stopped, stop_pos, cur_pos, n_stopped, eng.tokens, eng.pos), keep):
        dst.copy_(src)  # capture does not execute, but keep the state explicit

    remaining = total_len - (start_pos + 1)
    while remaining > 0:
        n = min(remaining, max(1, int(sync_every)))
        for _ in range(n):
            graph.replay()
        remaining -= n
        if int(n_stopped.item()) >= bsz:  # the only host synchronisation of the loop (meta.py:458 does it per token)
            break
    torch.cuda.synchronize()
    return tokens.tolist(), [int(v) for v in stop_pos.tolist()]


@torch.inference_mode()
def generate(model, tokenizer, prompts: List[str], images=None, max_gen_len: int = 512, temperature: float = 0.0,
             top_p: float = 0.95, additional_stop_symbols: Iterable[str] = (), *, device_loop: Optional[bool] = None,
             sync_every: int = 16, select: Optional[Callable] = None) -> List[str]:
    """MetaModel.generate (meta.py:372-468): batched prompts -> generated continuations (prompt and stop symbol
    stripped).  `device_loop` defaults to True for an engine-backed model; `select` replaces the on-device token
    selection of the host loop (tests)."""
    if images is not None:
        raise NotImplementedError("image prefixes are outside the decode hot path served here")
    dev = _device_of(model)
    plan = _Plan(model, tokenizer, prompts, max_gen_len, tuple(additional_stop_symbols), dev)
    eng = getattr(model, "engine", None)
    if device_loop is None:
        device_loop = select is None and hasattr(model, "build_engine")
    if device_loop:
        if select is not None:
            raise ValueError("`select` applies to the host loop only")
        if eng is None:
            model.build_engine()
        toks, stop_pos = _device_loop(model, plan, temperature, top_p, sync_every)
    else:
        toks, stop_pos = _host_loop(model, plan, temperature, top_p, select or device_select)
    return plan.decode(tokenizer, toks, stop_pos)


@torch.inference_mode()
def stream_generate(model, tokenizer, prompt: str, image=None, max_gen_len: int = 512, temperature: float = 0.0,
                    top_p: float = 0.95, additional_stop_symbols: Iterable[str] = (), *,
                    select: Optional[Callable] = None):
    """MetaModel.stream_generate (meta.py:470-548): yields {"text", "end_of_content"} after every token.  Streaming
    needs the text on the host after each token, so this is the host loop by construction."""
    if image is not None:
        raise NotImplementedError("image prefixes are outside the decode hot path served here")
    select = select or device_select
    dev = _device_of(model)
    args = model.args
    prompt_tokens = tokenizer.encode(prompt, bos=True, eos=False)
    max_seq_len = args.max_seq_len
    prompt_tokens = prompt_tokens[-(max_seq_len - max_gen_len):]  # truncate from the left, leave room to generate
    prompt_size = len(prompt_tokens)
    total_len = min(max_seq_len, max_gen_len + prompt_size)
    tokens = torch.zeros(total_len, dtype=torch.int64, device=dev)
    tokens[:prompt_size] = torch.tensor(prompt_tokens, dtype=torch.int64)
    start_pos, prev_pos, generate_until = prompt_size, 0, prompt_size
    for cur_pos in range(start_pos, total_len):
        logits = model.forward_inference(tokens[None, prev_pos:cur_pos], prev_pos).float()
        next_token = int(select(logits, temperature, top_p).reshape(-1)[0])
        if next_token == tokenizer.eos_id:
            break
        tokens[cur_pos] = next_token
        prev_pos = cur_pos
        generate_until = cur_pos + 1
        generated = tokenizer.decode(tokens[start_pos:generate_until].tolist())
        for stop_symbol in additional_stop_symbols:
            at = generated.find(stop_symbol)
            if at != -1:
                yield {"text": generated[:at], "end_of_content": True}
                return
        yield {"text": generated, "end_of_content": False}
    yield {"text": tokenizer.decode(tokens[start_pos:generate_until].tolist()), "end_of_content": True}
