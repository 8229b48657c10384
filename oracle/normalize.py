"""TEST INFRASTRUCTURE -- NumPy restatement of the input normalisation of the reference.

Follows vamb/encode.py:93-126 (``make_dataloader`` up to the four tensors; the
DataLoader wrapping of :129-144 is not needed by the oracle, which indexes the tensors directly) and
vamb/vambtools.py:250-288 (``zscore``).  Used by ``bench.py --impl reference`` and the
``cpu_baseline`` leg so that the reference arm never imports the product package.
tests/test_oracle_normalize.py pins it against the live reference and against the product's own
``vamb_b200.encode.make_dataloader`` (bit-identical tensors).
"""
from __future__ import annotations

import numpy as np


def _zscore_inplace(a: np.ndarray, axis=None) -> None:
    """vambtools.py:272-285 with ``inplace=True``: (a - mean) / std, constant slices -> std 1."""
    mean = a.mean(axis=axis)
    std = a.std(axis=axis)
    if axis is None:
        if std == 0:
            std = 1
    else:
        std[std == 0.0] = 1
        shape = tuple(1 if ax == axis else dim for ax, dim in enumerate(a.shape))
        mean = mean.reshape(shape)
        std = std.reshape(shape)
    a -= mean
    a /= std


def normalize(abundance: np.ndarray, tnf: np.ndarray, lengths: np.ndarray):
    """(depths [N, S], tnf [N, 103], total_abundance [N, 1], weights [N, 1]) float32, on copies."""
    if abundance.dtype != np.float32 or tnf.dtype != np.float32:
        raise ValueError("TNF and abundance must be Numpy arrays of dtype float32")
    abundance = abundance.copy()
    tnf = tnf.copy()
    colsum = abundance.sum(axis=0)  # encode.py:99
    if np.any(colsum == 0):
        raise ValueError("One or more samples have zero depth in all sequences, so cannot be depth normalized")
    abundance *= 1_000_000 / colsum  # :104
    total = abundance.sum(axis=1)  # :105
    nsamples = abundance.shape[1]
    zero = total == 0  # :108-113
    abundance[zero] = 1 / nsamples
    div = total.copy()
    div[zero] = 1.0
    abundance /= div.reshape((-1, 1))
    total = np.log(total.clip(min=0.001))  # :116
    _zscore_inplace(total)  # :117
    _zscore_inplace(tnf, axis=0)  # :118
    total.shape = (len(total), 1)
    lens = lengths.astype(np.float32)  # :122-126
    weights = np.log(lens).astype(np.float32) - 5.0
    weights[weights < 2.0] = 2.0
    weights *= len(weights) / weights.sum()
    weights.shape = (len(weights), 1)
    return abundance, tnf, total, weights
