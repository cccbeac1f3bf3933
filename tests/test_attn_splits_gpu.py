"""Decode attention (csrc/attn.cu) with every split count merged through the workspace by the last CTA of a (token, kv head).
Checked against an fp32 reference at split counts from 1 to one split per tile (the one-round-trip merge of <= 16 splits and
the staged merge of more), kv lengths that are not multiples of 32, GQA groups of 4 and 8, several tokens with mixed
positions, and two launches in a row (the merging CTA resets its head's counter)."""
import math

import pytest
import torch

from llama2_accessory_b200 import kvlayout, ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ref(q, k, v, pos, tps, Hq, Hkv):
    """k, v canonical [B, Hkv, S, 128] -> fp32 [T, Hq * 128]."""
    T, n_rep = q.shape[0], Hq // Hkv
    out = torch.zeros(T, Hq, 128, device=q.device)
    for t in range(T):
        b, n = t // tps, int(pos[t]) + 1
        kk = k[b, :, :n].float().repeat_interleave(n_rep, 0)                  # [Hq, n, 128]
        vv = v[b, :, :n].float().repeat_interleave(n_rep, 0)
        s = torch.einsum("hnd,hd->hn", kk, q[t].float()) / math.sqrt(128)
        out[t] = torch.einsum("hn,hnd->hd", torch.softmax(s, -1), vv)
    return out.reshape(T, Hq * 128)


def _tiles(poss, Hkv):
    return sum(Hkv * ((p + 32) // 32) for p in poss)


#                       T  tps  Hq  Hkv    S   positions
CASES = [
    ("7B_bs1",          1, 1,   32, 32, 2400, [2100]),          # the flagship's shape: 66 tiles per head
    ("gqa4_bs1",        1, 1,   32,  8, 1024, [1000]),
    ("gqa8_bs1",        1, 1,   64,  8,  512, [450]),
    ("gqa4_bs4_mixed",  4, 1,   16,  4, 1024, [5, 600, 1023, 31]),
    ("gqa8_chunk5",     5, 5,   16,  2,  512, [300, 301, 302, 303, 304]),   # one sequence, positions cross a tile
    ("mha_bs3_short",   3, 1,    6,  6,  256, [0, 32, 63]),
    ("mha_bs2_chunk2",  4, 2,    4,  4,  256, [30, 31, 200, 201]),
]


@pytest.mark.parametrize("name,T,tps,Hq,Hkv,S,poss", CASES, ids=[c[0] for c in CASES])
def test_attention_at_every_split_count_matches_fp32(name, T, tps, Hq, Hkv, S, poss):
    B = T // tps
    g = torch.Generator(device=DEV).manual_seed(S + 7 * T + Hq)
    q = torch.randn(T, Hq, 128, device=DEV, generator=g).half()
    k = (torch.randn(B, Hkv, S, 128, device=DEV, generator=g) * 0.7).half()
    v = torch.randn(B, Hkv, S, 128, device=DEV, generator=g).half()
    kc, vt = kvlayout.k_to_engine(k), kvlayout.v_to_engine(v)
    pos = torch.tensor(poss, dtype=torch.int32, device=DEV)
    ref = _ref(q, k, v, pos, tps, Hq, Hkv)
    tiles = _tiles(poss, Hkv)
    chosen = ops.attn_split(T, Hkv, S)
    assert 1 <= chosen <= T * Hkv * (S // 32)
    # 1 split; a few; the product's choice; one split per tile, and more requested than there are tiles
    splits = sorted({1, 2, 3, 7, max(1, tiles // 5), tiles - 1 if tiles > 1 else 1, tiles, chosen, tiles + 5})
    for ns in splits:
        ws = torch.zeros(ops.attn_workspace_bytes(T, Hq, ns), dtype=torch.uint8, device=DEV)
        cnt = torch.zeros(T * Hkv, dtype=torch.int32, device=DEV)
        out = torch.full((T, Hq * 128), float("nan"), device=DEV, dtype=torch.float16)
        for rep in range(2):  # the second launch needs the counters the first one reset
            out.fill_(float("nan"))
            ops.attn_decode(q, kc, vt, pos, out, T=T, Hq=Hq, Hkv=Hkv, cache_seq=S, tokens_per_seq=tps,
                            max_kv_len=max(poss) + 1, ws=ws, counters=cnt, n_split=ns)
            torch.cuda.synchronize()
            err = (out.float() - ref).abs().max().item()
            assert err <= 4e-3, (ns, rep, err)
            assert int(cnt.abs().sum()) == 0, (ns, rep)


def test_a_graph_sized_for_the_longest_context_serves_shorter_ones():
    """The engine captures its decode graph with the split count chosen for cache_seq; the split boundaries follow pos[]."""
    T, Hq, Hkv, S = 1, 32, 32, 2400
    g = torch.Generator(device=DEV).manual_seed(3)
    q = torch.randn(T, Hq, 128, device=DEV, generator=g).half()
    k = (torch.randn(1, Hkv, S, 128, device=DEV, generator=g) * 0.7).half()
    v = torch.randn(1, Hkv, S, 128, device=DEV, generator=g).half()
    kc, vt = kvlayout.k_to_engine(k), kvlayout.v_to_engine(v)
    ns = ops.attn_split(T, Hkv, S)
    ws = torch.zeros(ops.attn_workspace_bytes(T, Hq, ns), dtype=torch.uint8, device=DEV)
    cnt = torch.zeros(T * Hkv, dtype=torch.int32, device=DEV)
    out = torch.empty((T, Hq * 128), device=DEV, dtype=torch.float16)
    for p in (0, 31, 32, 257, 2048, 2191, S - 1):
        pos = torch.tensor([p], dtype=torch.int32, device=DEV)
        ops.attn_decode(q, kc, vt, pos, out, T=T, Hq=Hq, Hkv=Hkv, cache_seq=S, tokens_per_seq=1, max_kv_len=S,
                        ws=ws, counters=cnt, n_split=ns)
        torch.cuda.synchronize()
        err = (out.float() - _ref(q, k, v, pos, 1, Hq, Hkv)).abs().max().item()
        assert err <= 4e-3, (p, err)
        assert int(cnt.abs().sum()) == 0, p
