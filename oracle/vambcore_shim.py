"""TEST INFRASTRUCTURE -- stand-in for the ``vambcore`` Rust wheel (vambcore==0.1.2,
pyproject.toml:6), which is not installed here.

Only ``overwrite_matrix`` is on the hot path (vamb/vambtools.py:302,319
<- vamb/cluster.py:322-328).  Its semantics are pinned by
test/test_vambtools.py:271-298: rows where ``mask`` is true are
moved to the front of ``matrix`` in their original order and the number of kept
rows is returned.  ``kmercounts`` is off-path and only stubbed.
"""
import numpy as np


def overwrite_matrix(matrix: np.ndarray, mask: np.ndarray) -> int:
    if matrix.ndim != 2:
        raise ValueError("matrix must be 2-dimensional")
    if len(mask) != len(matrix):
        raise ValueError("Lengths of array and mask must match")
    mask = np.asarray(mask, dtype=bool)
    idx = np.flatnonzero(mask)
    n = len(idx)
    # rows only ever move towards the front, so a forward pass is safe in place
    if n and idx[-1] != n - 1:
        matrix[:n] = matrix[idx]
    return int(n)


def kmercounts(counts, seq):  # pragma: no cover - off the hot path
    raise NotImplementedError("vambcore.kmercounts is outside the hot path")
