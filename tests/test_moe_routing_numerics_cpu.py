"""CPU restatement of moe_route_kernel's routing arithmetic (csrc/moe.cu) against the reference's statements
(mixtral.py:275-280: fp16 gate logits -> softmax -> fp16 -> top-k -> renormalise in fp16).

    kernel      logits fp16 (fp32-accumulated F.linear, rounded); softmax in fp32 with expf, scores rounded to fp16;
                top-k on the fp16 scores (ties: lowest index); sum of the k fp16 scores rounded to fp16; weight = fp16(v / sum)
    reference   scores = gate(x).softmax(-1)   (half tensor: computed in fp32 inside ATen, rounded to fp16)
                w, idx = topk(scores, k);  w = w / w.sum(-1, keepdim=True)      (fp16 sum, fp16 division)

Routing is a DISCRETE decision: a score that rounds differently moves a token to another expert.  The two statements must
pick the same experts wherever the k-th and (k+1)-th fp16 scores differ, with weights equal to the last fp16 bit.
"""
import numpy as np
import pytest
import torch

from oracle.numerics import kernel_route, kernel_scores


@pytest.mark.parametrize("E,k", [(8, 2), (8, 1), (16, 4), (64, 8)])
def test_routing_model_equals_the_reference_statements(E, k):
    g = torch.Generator().manual_seed(E * 10 + k)
    T = 20000
    logits16 = (torch.randn(T, E, generator=g) * 1.5).half()
    idx_k, w_k = kernel_route(logits16, k)
    scores = logits16.softmax(dim=-1)                                   # mixtral.py:275 on a half tensor
    w_r, idx_r = torch.topk(scores, k, dim=-1)                          # :276
    w_r = w_r / w_r.sum(dim=-1, keepdim=True)                           # :280
    # the fp16 scores themselves: identical up to the rare last-bit difference of the two exp implementations
    sc_k = torch.from_numpy(np.sort(kernel_scores(logits16), -1))
    sc_r = scores.float().sort(-1).values
    assert float((sc_k != sc_r).float().mean()) < 2e-3
    # tokens whose selection is unambiguous in BOTH statements (no tie at the k-th place, same fp16 scores)
    srt = scores.float().sort(-1, descending=True).values
    clear = torch.ones(T, dtype=torch.bool) if k == E else (srt[:, k - 1] > srt[:, k])
    distinct = (srt[:, :k].diff(dim=-1) < 0).all(-1) if k > 1 else torch.ones(T, dtype=torch.bool)
    same_scores = (sc_k == sc_r).all(-1)
    ok = clear & distinct & same_scores
    assert float(ok.float().mean()) > 0.95
    assert torch.equal(idx_k[ok], idx_r[ok])
    assert torch.equal(w_k[ok], w_r[ok])                                # weights to the last fp16 bit
    # everywhere: the same SET of experts unless two fp16 scores tie at the boundary or the scores differ in the last bit
    same_set = (idx_k.sort(-1).values == idx_r.sort(-1).values).all(-1)
    assert float(same_set[clear & same_scores].float().mean()) == 1.0


def test_weights_of_a_token_sum_to_one_within_fp16():
    g = torch.Generator().manual_seed(3)
    idx, w = kernel_route((torch.randn(5000, 8, generator=g) * 2).half(), 2)
    assert float((w.float().sum(-1) - 1).abs().max()) <= 2.0 ** -10
    assert (idx[:, 0] != idx[:, 1]).all()
