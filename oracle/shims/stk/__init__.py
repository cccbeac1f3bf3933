"""ORACLE TEST INFRASTRUCTURE: a plain-torch stand-in for the parts of stk (stanford-futuredata/stk) that
accessory/model/LLM/mixtral_sparse.py calls: the block-sparse Matrix and ops.row_indices / sdd / dsd, blocking 128.
NOT VERIFIED against stk itself (not installed here): restated from memory of its public source."""
from . import ops  # noqa: F401


class Matrix:
    """Block-sparse matrix: `data` [nnz, blocking, blocking] holds the non-zero blocks in row-major block order."""

    def __init__(self, size, data, row_indices, column_indices, offsets, column_indices_t=None, offsets_t=None,
                 block_offsets_t=None):
        self._size = tuple(size)
        self.data, self.row_indices, self.column_indices, self.offsets = data, row_indices, column_indices, offsets
        self.column_indices_t, self.offsets_t, self.block_offsets_t = column_indices_t, offsets_t, block_offsets_t

    def size(self):
        return self._size

    @property
    def blocking(self):
        return self.data.shape[1]
