"""GPU: the UNMODIFIED reference `MetaModel` (accessory/model/meta.py, imported byte-for-byte from /root/reference or its
staged copy oracle/_ref) constructed with ``llama_type="llama_b200"`` and driven through its own ``generate()``.

This is the integration level 3 of INTEGRATION.md executed end to end: `MetaModel.__init__` (meta.py:20-78) resolves
``accessory.model.LLM.llama_b200`` with importlib (meta.py:29), reads the JSON config into our ``ModelArgs``, builds our
``Transformer``; a checkpoint-shaped state dict is loaded into ``model.llma``; ``MetaModel.generate`` (meta.py:372-468)
then calls ``self.llma.forward_inference`` once per token -- every one of those calls runs in libb200decode.so.

The modules meta.py imports but this path never touches (util.misc / util.tensor_parallel / model.tokenizer) are stubbed
as in oracle/make_golden_generate.py; the tokenizer is the toy whitespace tokenizer the generate-loop goldens use.
"""
import importlib
import json
import os
import sys
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import generation  # noqa: E402
from llama2_accessory_b200.model import llama_b200  # noqa: E402
from oracle import cases, ref_import  # noqa: E402
from oracle.toy_tokenizer import ToyTokenizer  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "generate.json")
PROMPTS = ["the quick brown fox", "hello world", "a b c d e f g"]


class _PathTokenizer(ToyTokenizer):
    """accessory/model/tokenizer.py::Tokenizer(model_path=...) stand-in: 'toy:<n_words>:<eos_id>'."""

    def __init__(self, model_path):
        _, n, eos = model_path.split(":")
        super().__init__(int(n), int(eos))


def _import_meta():
    if not ref_import.available():
        pytest.skip("reference tree not staged (oracle/_ref)")
    ref_import.load("llama")  # registers the accessory namespace packages + the fairscale shim
    stubs = (("accessory.util.misc", {"mark_mp_params": lambda model: None}),
             ("accessory.util.tensor_parallel", {}),
             ("accessory.model.tokenizer", {"Tokenizer": _PathTokenizer, "probe_tokenizer_path_from_pretrained": None}))
    for name, attrs in stubs:
        m = sys.modules.get(name)
        if m is None:
            m = types.ModuleType(name)
            sys.modules[name] = m
            parent, leaf = name.rsplit(".", 1)
            setattr(sys.modules[parent], leaf, m)
        for k, v in attrs.items():
            setattr(m, k, v)
    # the two-line plug-in file of INTEGRATION.md section 3 (accessory/model/LLM/llama_b200.py), registered in memory
    plug = types.ModuleType("accessory.model.LLM.llama_b200")
    plug.ModelArgs, plug.Transformer = llama_b200.ModelArgs, llama_b200.Transformer
    sys.modules["accessory.model.LLM.llama_b200"] = plug
    meta = importlib.import_module("accessory.model.meta")
    meta.Tokenizer = _PathTokenizer  # in case meta.py was imported earlier in this process with another stub
    return meta


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _metamodel(meta, tmp_path, wbits, eos_id=2):
    args = dict(cases.TINY_LLAMA)
    cfg = {k: v for k, v in args.items() if k not in ("vocab_size", "max_seq_len", "max_batch_size")}
    cfg["wbits"] = wbits
    p = tmp_path / f"config_w{wbits}.json"
    p.write_text(json.dumps(cfg))
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float16)
    try:
        with torch.device("cuda"):
            model = meta.MetaModel("llama_b200", str(p), f"toy:{args['vocab_size']}:{eos_id}", with_visual=False,
                                   max_seq_len=args["max_seq_len"])
    finally:
        torch.set_default_dtype(old)
    assert type(model.llma) is llama_b200.Transformer and model.llma.args.max_batch_size == 32
    sd = cases.master_state_dict("llama", args)
    missing, unexpected = model.load_state_dict({"llma." + k: v.cuda() for k, v in sd.items()}, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    return model.eval()


def test_unmodified_metamodel_generate_runs_on_the_b200_engine(tmp_path):
    meta = _import_meta()
    model = _metamodel(meta, tmp_path, wbits=4)
    texts = model.generate(list(PROMPTS), max_gen_len=6)
    assert model.llma.engine is not None and model.llma.engine.cfg.bits == 4  # forward_inference built the packed engine
    # the loop runs to max(prompt length) + max_gen_len for every row (meta.py:415-433): shorter prompts generate more tokens
    plens = [len(model.tokenizer.encode(x, bos=True, eos=False)) for x in PROMPTS]
    assert [len(t.split()) for t in texts] == [max(plens) + 6 - n for n in plens], texts
    tok = model.tokenizer
    # same tokens as this repo's statement of the loop (host and device drivers) over the same engine
    assert generation.generate(model.llma, tok, list(PROMPTS), max_gen_len=6, device_loop=False) == texts
    assert generation.generate(model.llma, tok, list(PROMPTS), max_gen_len=6, device_loop=True) == texts
    # eos / stop-symbol handling of the reference loop over our logits
    row0 = [int(w[1:]) for w in texts[0].split()]
    model.tokenizer.eos_id = row0[2]
    cut = model.generate(list(PROMPTS), max_gen_len=6)
    first = row0.index(row0[2])  # the reference stops a row at the FIRST occurrence of eos among its generated tokens
    assert cut[0] == " ".join(texts[0].split()[:first]), (cut, texts)
    assert cut == generation.generate(model.llma, model.tokenizer, list(PROMPTS), max_gen_len=6, device_loop=False)
    model.tokenizer.eos_id = 2
    stops = (f"w{row0[1]} w{row0[2]}",)
    stop = model.generate(list(PROMPTS), max_gen_len=6, additional_stop_symbols=stops)
    assert stop == generation.generate(model.llma, model.tokenizer, list(PROMPTS), max_gen_len=6, additional_stop_symbols=stops,
                                       device_loop=False)
    assert len(stop[0].split()) < len(texts[0].split()), (stop, texts)
    ys = list(model.stream_generate(PROMPTS[0], max_gen_len=5))
    assert ys[-1]["end_of_content"] and ys[-1]["text"] == model.generate([PROMPTS[0]], max_gen_len=5)[0]


def test_metamodel_fp16_engine_against_the_reference_goldens():
    """wbits = 16: the same weights the fp32 goldens of the unmodified reference model were generated from
    (tests/golden/generate.json); fp16 logits can flip a near-tie, so agreement is counted, not demanded token for token.
    Self-contained: the drop-in Transformer is built as MetaModel builds it (max_batch_size 32, vocab from the tokenizer)
    and driven by this repo's statement of MetaModel.generate, which tests/test_generation_cpu.py pins to the same goldens."""
    args = dict(cases.TINY_LLAMA)
    cfg = {k: v for k, v in args.items() if k not in ("max_batch_size",)}
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float16)
    try:
        with torch.device("cuda"):
            model = llama_b200.Transformer(llama_b200.ModelArgs(**cfg, max_batch_size=32, wbits=16))
    finally:
        torch.set_default_dtype(old)
    missing, unexpected = model.load_state_dict({k: v.cuda() for k, v in cases.master_state_dict("llama", args).items()},
                                                strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    model.eval()
    texts = generation.generate(model, ToyTokenizer(args["vocab_size"], 2), list(PROMPTS), max_gen_len=6, device_loop=False)
    gold = next(c for c in json.load(open(GOLD))["cases"] if c["name"] == "greedy")["texts"]
    first = sum(a.split()[0] == b.split()[0] for a, b in zip(texts, gold))
    n_tok = sum(len(b.split()) for b in gold)
    n_same = sum(x == y for a, b in zip(texts, gold) for x, y in zip(a.split(), b.split()))
    print(f"\n[MetaModel(llama_b200, fp16) vs reference fp32 goldens] first tokens {first}/3, all tokens {n_same}/{n_tok}")
    assert first >= 2 and n_same >= n_tok // 2, (texts, gold)
