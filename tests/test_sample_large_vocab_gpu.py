"""GPU: b200_sample_top_p over vocabularies whose probabilities do not fit in shared memory (csrc/sample.cu's
sample_top_p_radix_kernel, selected for V > 57856 with the H100's 227 KB opt-in), against the same float64 statement of
MetaModel.sample_top_p's rule (meta.py:550-565) and tolerances as tests/test_zz_generation_gpu.py: V = 57856 / 57857
(either side of the kernel switch), 103168 (InternLM-7B / -20B) and 256000; the nucleus distribution, a run-to-run
identical cut, and the device generate loop sampling at temperature > 0 from a 103168-token head."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import llama2_accessory_b200 as pkg  # noqa: E402
from llama2_accessory_b200 import generation, ops  # noqa: E402
from llama2_accessory_b200.engine import DecodeEngine, EngineConfig  # noqa: E402
from llama2_accessory_b200.model.llama_b200 import Transformer as B200Transformer  # noqa: E402
from oracle import cases, weights  # noqa: E402
from oracle.toy_tokenizer import ToyTokenizer  # noqa: E402

DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _built():
    pkg.build()


def _rule(logits, u, temperature, top_p):
    """float64 statement: (mass strictly above each token, cumulative kept intervals in index order, target)."""
    x = logits.astype(np.float64) / temperature
    p = np.exp(x - x.max())
    p /= p.sum()
    asc = np.sort(p)
    csum = np.cumsum(asc)
    mass_gt = csum[-1] - csum[np.searchsorted(asc, p, side="right") - 1]
    pk = np.where(mass_gt <= top_p, p, 0.0)
    hi = np.cumsum(pk)
    return mass_gt, hi - pk, hi, u * hi[-1]


def _sample(logits, u, temperature, top_p):
    T, V = logits.shape
    out = torch.full((T,), -1, dtype=torch.int64, device=DEV)
    ops.sample_top_p(logits, u, out, T, V, temperature, top_p)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("V,T,temperature,top_p", [(57856, 8, 1.0, 0.9), (57857, 8, 1.0, 0.9), (103168, 8, 0.7, 0.9),
                                                    (103168, 32, 1.0, 0.95), (103168, 4, 0.3, 0.5),
                                                    (103168, 4, 1.3, 1.0), (256000, 8, 1.0, 0.95)])
def test_large_vocab_follows_the_reference_rule(V, T, temperature, top_p):
    g = torch.Generator().manual_seed(V + T + int(top_p * 100))
    logits = (torch.randn(T, V, generator=g) * 2.5).float()
    u = torch.rand(T, generator=g).float()
    out = _sample(logits.to(DEV), u.to(DEV), temperature, top_p).cpu().numpy()
    for t in range(T):
        mass_gt, lo, hi, target = _rule(logits[t].numpy(), float(u[t]), temperature, top_p)
        i = int(out[t])
        assert 0 <= i < V
        assert mass_gt[i] <= top_p + 1e-5, (t, i, mass_gt[i])
        assert lo[i] - 2e-5 <= target <= hi[i] + 2e-5, (t, i, lo[i], target, hi[i])


@pytest.mark.parametrize("V", [57857, 103168])
def test_large_vocab_distribution_and_limits(V):
    n = 3000
    head = torch.tensor([2.0, 1.5, 1.0, 0.5, 0.0, -0.5, -1.0, -1.5] + [-3.0] * 8)
    spots = torch.linspace(0, V - 1, 16).long()             # spread over the row, in increasing index order
    row = torch.full((V,), -40.0)                            # ~1e-18 each: never inside a nucleus below 1
    row[spots] = head
    p = torch.softmax(head.double(), 0).numpy()
    rows = row.repeat(n, 1).to(DEV)
    u = torch.rand(n, device=DEV)
    top_p = 0.8
    out = _sample(rows, u, 1.0, top_p)
    order = np.argsort(-p)
    before = np.cumsum(p[order]) - p[order]
    kept = np.zeros(16, bool)
    kept[order[before <= top_p]] = True
    idx = out.cpu().numpy()
    assert np.isin(idx, spots.numpy()).all()
    freq = np.array([(idx == int(s)).sum() for s in spots]) / n
    expect = np.where(kept, p, 0) / p[kept].sum()
    assert np.abs(freq - expect).max() < 0.03, (freq, expect)
    assert freq[~kept].sum() == 0
    # the cut is computed in fixed point: the same row and uniform give the same token on every call
    assert torch.equal(_sample(rows, u, 1.0, top_p), out)
    # a tiny nucleus is the arg-max; a full nucleus with u -> 1 stays inside the vocabulary
    assert int((_sample(rows, u, 1.0, 1e-4) != int(spots[0])).sum()) == 0
    last = _sample(rows, torch.full((n,), 0.99999994, device=DEV), 1.0, 1.0)
    assert int(last.min()) >= 0 and int(last.max()) < V


def test_device_loop_samples_from_a_large_head():
    V = 103168
    args = dict(cases.TINY_LLAMA, vocab_size=V)
    eng = DecodeEngine(EngineConfig.from_model_args("llama", args, bits=4, group_size=0), DEV)
    eng.load_master_state_dict(weights.llama_state_dict(args))
    model = B200Transformer.from_engine(eng)
    tok = ToyTokenizer(V, 2)
    prompts = ["the quick brown fox", "hello world", "a b c d e f g"]
    torch.manual_seed(0)
    for device_loop in (True, False):
        texts = generation.generate(model, tok, prompts, max_gen_len=8, temperature=0.8, top_p=0.9,
                                    device_loop=device_loop)
        assert len(texts) == 3
        for t in texts:
            ids = [int(w[1:]) for w in t.split()]
            assert all(0 <= i < V for i in ids), t
    # a nucleus that holds only the arg-max makes sampling greedy, in both loops
    greedy = generation.generate(model, tok, prompts, max_gen_len=8)
    for device_loop in (True, False):
        assert generation.generate(model, tok, prompts, max_gen_len=8, temperature=1.0, top_p=1e-6,
                                   device_loop=device_loop) == greedy
