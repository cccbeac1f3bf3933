"""ORACLE TEST INFRASTRUCTURE: stk.ops restated in plain torch (see stk/__init__.py).  sdd and dsd form the dense
product and keep / read only the topology's blocks: the values of the non-zero blocks are those of the dense product."""
import torch


def row_indices(shape, data, offsets, column_indices):
    """Block row of every non-zero block (offsets: CSR row pointers over blocks)."""
    counts = (offsets[1:] - offsets[:-1]).long()
    return torch.repeat_interleave(torch.arange(counts.numel(), dtype=torch.int32, device=offsets.device), counts)


def sdd(a, b, topo):
    """dense [M, K] x dense [K, N] -> the topology's blocks of the product, [nnz, bs, bs] (stk.Matrix)."""
    from . import Matrix
    bs = topo.blocking
    full = a @ b
    blocks = torch.stack([full[int(r) * bs:(int(r) + 1) * bs, int(c) * bs:(int(c) + 1) * bs]
                          for r, c in zip(topo.row_indices, topo.column_indices)])
    return Matrix(topo.size(), blocks, topo.row_indices, topo.column_indices, topo.offsets, topo.column_indices_t,
                  topo.offsets_t, topo.block_offsets_t)


def dsd(a, b):
    """block-sparse [M, K] (stk.Matrix) x dense [K, N] -> dense [M, N]; blocks outside the topology are 0."""
    bs = a.blocking
    dense = torch.zeros(a.size(), dtype=a.data.dtype, device=a.data.device)
    for blk, r, c in zip(a.data, a.row_indices, a.column_indices):
        dense[int(r) * bs:(int(r) + 1) * bs, int(c) * bs:(int(c) + 1) * bs] = blk
    return dense @ b
