"""ORACLE TEST INFRASTRUCTURE: megablocks.ops restated in plain torch, only the calls mixtral_sparse.py makes
(sort, histogram, round_up, inclusive_cumsum, padded_gather, padded_scatter, topology).

NOT VERIFIED against megablocks itself: megablocks is not installed here, and these semantics, in particular the
rounding points of padded_scatter (each slot fp16(y * w) with the product formed in fp32, then the top_k slots of a token
summed by torch's fp16 .sum, i.e. fp32 accumulation rounded once), are restated from memory of megablocks' public source.
"""
import torch


def sort(x, end_bit=None):
    """Radix sort of non-negative ints -> (sorted values, int32 permutation); stable, as a radix sort is."""
    v, i = torch.sort(x, stable=True)
    return v, i.int()


def histogram(x, num_bins):
    return torch.bincount(x.long().flatten(), minlength=num_bins).int()


def round_up(x, value):
    return ((x + value - 1) // value * value).int()


def inclusive_cumsum(x, dim):
    return torch.cumsum(x, dim).int()


def _bounds(bins, padded_bins, e):
    start = 0 if e == 0 else int(bins[e - 1])
    pstart = 0 if e == 0 else int(padded_bins[e - 1])
    return start, int(bins[e]), pstart


def padded_gather(x, indices, bin_ids, bins, padded_bins, top_k):
    """[T, D] -> [padded_bins[-1], D]: the k-th slot of token t (flat index t * top_k + k, sorted by expert) goes to the
    row of its expert's 128-row-padded bin; padding rows are 0."""
    out = torch.zeros((int(padded_bins[-1]), x.shape[1]), dtype=x.dtype, device=x.device)
    for e in range(bins.numel()):
        start, end, pstart = _bounds(bins, padded_bins, e)
        for j in range(start, end):
            out[pstart + j - start] = x[int(indices[j]) // top_k]
    return out


def padded_scatter(x, indices, bin_ids, weights, bins, padded_bins, top_k, num_bits=-1):
    """[padded rows, D] -> [T, D]: slot s = fp16(fp32(row) * fp32(weights[s])), then the top_k slots of each token summed."""
    T = indices.numel() // top_k
    slots = torch.zeros((T * top_k, x.shape[1]), dtype=x.dtype, device=x.device)
    for e in range(bins.numel()):
        start, end, pstart = _bounds(bins, padded_bins, e)
        for j in range(start, end):
            s = int(indices[j])
            slots[s] = (x[pstart + j - start].float() * weights[s].float()).to(x.dtype)
    return slots.view(T, top_k, -1).sum(dim=1)


def topology(padded_bins, blocking, block_rows, blocks_per_row):
    """Column block indices of the block-sparse [padded rows, E * F_loc] matrix: block row b lies in the bin of expert e
    and holds that expert's blocks_per_row column blocks."""
    cols = []
    for b in range(block_rows):
        e = int(torch.searchsorted(padded_bins, torch.tensor(b * blocking, dtype=padded_bins.dtype), right=True))
        cols.extend(range(e * blocks_per_row, (e + 1) * blocks_per_row))
    return torch.tensor(cols, dtype=torch.int32, device=padded_bins.device)
