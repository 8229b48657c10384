"""TEST INFRASTRUCTURE -- CPU oracle for the medoid clusterer.

A restatement of vamb/cluster.py (CPU path, ``cuda=False``) in
NumPy + C (oracle/csrc/oracle_kernels.c).  It follows the reference's *sequential*
algorithm literally -- one full distance scan per ``sample_medoid`` call, physical
row packing after every emitted cluster -- so that it is an independent check of
the batched / pruned / mask-based CUDA design in vamb_b200.

The only deliberate difference from the reference is that the three tensor
reductions whose floating-point order the reference leaves to MKL/ATen are
evaluated in a DEFINED order ("vk arithmetic v1", DESIGN.md section 3):
  * distances:  8-lane fmaf chains + xor butterfly (ok_dists)
  * local density: exact integer sum in units of 2^-29 (ok_sample)
  * weighted histogram: exact integer sums, rounded once to fp32 (ok_hist)
  * row norm: sum of squares in fp64, ascending k (ok_normalize_rows)
Everything else (seed order, RNG call sequence, success window, peak/valley
scan in Python floats) is the reference's logic, cited line by line.

PARITY PINNING: tests/test_oracle_vs_reference.py compares this oracle with the
live reference (oracle/ref_loader.py, build container only) and with the golden
fixtures in tests/golden/ generated from the reference by oracle/make_golden.py.
"""
from __future__ import annotations

import ctypes
import os
import random
from collections import deque
from typing import NamedTuple, Optional

import numpy as np

MEDOID_RADIUS = 0.05  # cluster.py:14
DEFAULT_RADIUS = 0.06  # cluster.py:12
DELTA_X = 0.005  # cluster.py:16
XMAX = 0.3  # cluster.py:17
NBINS = 60  # ceil(XMAX / DELTA_X), cluster.py:231
DENSITY_SCALE = 2.0 ** -29

# cluster.py:39-73 -- N(0, 0.01) pdf sampled at 31 points, times DELTA_X, in fp32
_PDF_VALUES = [
    2.43432053e-11, 9.13472041e-10, 2.66955661e-08, 6.07588285e-07, 1.07697600e-05,
    1.48671951e-04, 1.59837411e-03, 1.33830226e-02, 8.72682695e-02, 4.43184841e-01,
    1.75283005e00, 5.39909665e00, 1.29517596e01, 2.41970725e01, 3.52065327e01,
    3.98942280e01, 3.52065327e01, 2.41970725e01, 1.29517596e01, 5.39909665e00,
    1.75283005e00, 4.43184841e-01, 8.72682695e-02, 1.33830226e-02, 1.59837411e-03,
    1.48671951e-04, 1.07697600e-05, 6.07588285e-07, 2.66955661e-08, 9.13472041e-10,
    2.43432053e-11,
]
NORMALPDF = np.float32(DELTA_X) * np.array(_PDF_VALUES, dtype=np.float32)


def linspace_edges(nbins: int = NBINS, xmax: float = XMAX) -> np.ndarray:
    """The fp32 edge table of ``torch.linspace(0.0, xmax, nbins + 1)`` (cluster.py:288),
    restated: step = (end-start)/(steps-1) in fp32; first half fma(step, i, start), second
    half fma(-step, steps-1-i, end) (ATen's vectorised kernel fuses the multiply-add; the
    product step*i is exact in fp64 so rounding the fp64 expression once emulates the fma)."""
    steps = nbins + 1
    start, end = np.float32(0.0), np.float32(xmax)
    step = np.float32((end - start) / np.float32(steps - 1))
    out = np.empty(steps, dtype=np.float32)
    half = steps // 2
    for i in range(steps):
        if i < half:
            out[i] = np.float32(float(start) + float(step) * i)
        else:
            out[i] = np.float32(float(end) - float(step) * (steps - 1 - i))
    return out


_lib = None


def _load_lib():
    global _lib
    if _lib is not None:
        return _lib
    here = os.path.dirname(os.path.abspath(__file__))
    path = os.path.join(here, "_build", "liboracle.so")
    if not os.path.isfile(path):
        from . import build as _build

        _build.build()
    lib = ctypes.CDLL(path)
    f32p = ctypes.POINTER(ctypes.c_float)
    i64p = ctypes.POINTER(ctypes.c_int64)
    u64p = ctypes.POINTER(ctypes.c_uint64)
    u8p = ctypes.POINTER(ctypes.c_uint8)
    lib.ok_normalize_rows.argtypes = [f32p, ctypes.c_int64, ctypes.c_int]
    lib.ok_normalize_rows.restype = None
    lib.ok_dists.argtypes = [f32p, ctypes.c_int64, ctypes.c_int, ctypes.c_int64, f32p]
    lib.ok_dists.restype = None
    lib.ok_sample.argtypes = [f32p, f32p, ctypes.c_int64, ctypes.c_float, i64p, u64p]
    lib.ok_sample.restype = ctypes.c_int64
    lib.ok_hist.argtypes = [f32p, f32p, ctypes.c_int64, f32p, ctypes.c_int, ctypes.c_float, u64p]
    lib.ok_hist.restype = ctypes.c_int64
    lib.ok_smaller.argtypes = [f32p, ctypes.c_int64, ctypes.c_float, i64p]
    lib.ok_smaller.restype = ctypes.c_int64
    lib.ok_pack_rows.argtypes = [f32p, f32p, i64p, u8p, ctypes.c_int64, ctypes.c_int]
    lib.ok_pack_rows.restype = ctypes.c_int64
    _lib = lib
    return lib


def _p(a: np.ndarray, ct):
    return a.ctypes.data_as(ctypes.POINTER(ct))


def normalize(matrix: np.ndarray) -> np.ndarray:
    """In-place row normalisation (cluster.py:653-669) with the defined arithmetic."""
    assert matrix.dtype == np.float32 and matrix.flags.c_contiguous and matrix.ndim == 2
    _load_lib().ok_normalize_rows(_p(matrix, ctypes.c_float), matrix.shape[0], matrix.shape[1])
    return matrix


def calc_distances(matrix: np.ndarray, index: int) -> np.ndarray:
    """cluster.py:672-676 with the defined arithmetic."""
    out = np.empty(matrix.shape[0], dtype=np.float32)
    _load_lib().ok_dists(
        _p(matrix, ctypes.c_float), matrix.shape[0], matrix.shape[1], int(index), _p(out, ctypes.c_float)
    )
    return out


def smooth_histogram(hist32: np.ndarray) -> np.ndarray:
    """cluster.py:497-500: 31-tap smoothing by 60 shifted fp32 AXPYs, cropped."""
    pdf_len = len(NORMALPDF)
    dens = np.zeros(len(hist32) + pdf_len - 1, dtype=np.float32)
    for i in range(len(hist32)):
        dens[i : i + pdf_len] += NORMALPDF * hist32[i]
    return dens[15:-15]


def scan_densities(densities: np.ndarray, pvr: float):
    """cluster.py:483-543, the peak/valley scan in Python floats.
    Returns None (NoThreshold) or (threshold, observed_pvr)."""
    peak_density = 0.0
    peak_over = False
    minimum_x = 0.0
    threshold = None
    delta_x = XMAX / len(densities)
    x = 0
    density_at_minimum = 0.0
    for density in densities.tolist():
        if not peak_over and density > peak_density:
            if x > 0.1:
                return None
            peak_density = density
        if not peak_over and density < 0.6 * peak_density:
            peak_over = True
            density_at_minimum = density
        if peak_over and density > 1.5 * density_at_minimum:
            break
        if peak_over and density < density_at_minimum:
            minimum_x, density_at_minimum = x, density
            if density < pvr * peak_density:
                threshold = minimum_x
        x += delta_x
    if threshold is None:
        return None
    if threshold > 0.2 + pvr:
        return None
    return (threshold, density_at_minimum / peak_density)


class OracleCluster(NamedTuple):
    medoid: int
    seed: int
    members: np.ndarray
    maximal_pvr: float
    observed_pvr: Optional[float]
    radius: Optional[float]
    successes: int
    attempts: int

    @property
    def kind_str(self) -> str:  # cluster.py:111-119
        if self.observed_pvr is not None:
            return "normal"
        return "loner" if self.radius is None else "fallback"


class OracleClusterGenerator:
    """Sequential restatement of ``vamb.cluster.ClusterGenerator`` (cuda=False)."""

    def __init__(
        self,
        matrix: np.ndarray,
        lengths: np.ndarray,
        maxsteps: int = 25,
        windowsize: int = 300,
        minsuccesses: int = 15,
        destroy: bool = False,
        normalized: bool = False,
        rng_seed: int = 0,
        order: Optional[np.ndarray] = None,
    ):
        # cluster.py:204-222
        if matrix.dtype != np.float32:
            raise ValueError("Matrix must be of dtype float32")
        if maxsteps < 1:
            raise ValueError(f"maxsteps must be a positive integer, not {maxsteps}")
        if windowsize < 1:
            raise ValueError(f"windowsize must be at least 1, not {windowsize}")
        if minsuccesses < 1 or minsuccesses > windowsize:
            raise ValueError(f"minsuccesses must be between 1 and windowsize, not {minsuccesses}")
        if len(matrix) < 1:
            raise ValueError("Matrix must have at least 1 observation.")
        if len(lengths) != len(matrix):
            raise ValueError("N sequences in lengths and matrix do not match")
        if not destroy:
            matrix = matrix.copy()
        matrix = np.ascontiguousarray(matrix)
        if not normalized:
            normalize(matrix)
        self.lib = _load_lib()
        self.matrix = matrix
        self.nrows = len(matrix)  # rows of self.matrix still in use (packed prefix)
        self.lens = np.asarray(lengths).astype(np.float32)  # torch.Tensor(lengths), cluster.py:277
        self.indices = np.arange(len(matrix), dtype=np.int64)
        # cluster.py:275 (ties: NumPy-build defined; callers may pass the order explicitly)
        self.order = np.argsort(lengths)[::-1].copy() if order is None else np.array(order)
        self.order_index = 0
        self.maxsteps = maxsteps
        self.minsuccesses = minsuccesses
        self.rng = random.Random(rng_seed)
        self.n_emitted_clusters = 0
        self.n_remaining_points = len(matrix)
        self.peak_valley_ratio = 0.1
        self.attempts: deque = deque(maxlen=windowsize)
        self.successes = 0
        self.edges = linspace_edges()
        self.n_sample_calls = 0  # statistics only
        self.trace: list = []  # optional decision trace (filled when self.record is True)
        self.record = False

    def __iter__(self):
        return self

    # ---- cluster.py:606-637 (without the memo: it has no semantic effect) ----
    def sample_medoid(self, medoid: int):
        n = self.nrows
        self.n_sample_calls += 1
        d = np.empty(n, dtype=np.float32)
        self.lib.ok_dists(
            _p(self.matrix, ctypes.c_float), n, self.matrix.shape[1], int(medoid), _p(d, ctypes.c_float)
        )
        idx = np.empty(n, dtype=np.int64)
        dens = (ctypes.c_uint64 * 2)()
        cnt = self.lib.ok_sample(
            _p(d, ctypes.c_float), _p(self.lens, ctypes.c_float), n,
            ctypes.c_float(MEDOID_RADIUS), _p(idx, ctypes.c_int64), dens,
        )
        return idx[:cnt], d, (int(dens[1]) << 12) + int(dens[0])

    # ---- cluster.py:415-450 ----
    def wander_medoid(self, seed: int):
        medoid = seed
        tried = {medoid}
        cluster, distances, local_density = self.sample_medoid(seed)
        candidates = [i for i in cluster.tolist() if i not in tried]
        candidates = self.rng.sample(candidates, k=min(len(candidates), self.maxsteps))
        i = 0
        while i < len(candidates):
            sampled = candidates[i]
            tried.add(sampled)
            s_cluster, s_distances, s_density = self.sample_medoid(sampled)
            if s_density > local_density:
                medoid, distances, local_density = sampled, s_distances, s_density
                candidates = [j for j in s_cluster.tolist() if j not in tried]
                candidates = self.rng.sample(candidates, k=min(len(candidates), self.maxsteps))
                i = 0
            else:
                i += 1
        return medoid, distances, local_density

    # ---- cluster.py:452-543 ----
    def find_threshold(self, distances: np.ndarray):
        n = self.nrows
        hist = np.zeros(NBINS, dtype=np.uint64)
        n_lt = self.lib.ok_hist(
            _p(distances, ctypes.c_float), _p(self.lens, ctypes.c_float), n,
            _p(self.edges, ctypes.c_float), NBINS, ctypes.c_float(MEDOID_RADIUS), _p(hist, ctypes.c_uint64),
        )
        if n_lt == 1:
            return "loner"
        hist32 = hist.astype(np.float32)  # exact sums rounded once to fp32
        return scan_densities(smooth_histogram(hist32), self.peak_valley_ratio)

    def _smaller(self, distances: np.ndarray, thr: float) -> np.ndarray:
        out = np.empty(self.nrows, dtype=np.int64)
        cnt = self.lib.ok_smaller(_p(distances, ctypes.c_float), self.nrows, ctypes.c_float(thr), _p(out, ctypes.c_int64))
        return out[:cnt]

    # ---- cluster.py:342-384 ----
    def get_next_seed(self) -> int:
        n_orig = len(self.order)
        i = self.order_index - 1
        live = self.indices[: self.nrows]
        while True:
            i = (i + 1) % n_orig
            if i == 0 and self.n_emitted_clusters > 0:
                self.order = self.order[self.order > -1]  # pack_order, cluster.py:337-340
                assert len(self.order) > 0
                n_orig = len(self.order)
            o = self.order[i]
            if o == -1:
                continue
            pos = int(np.searchsorted(live, o))
            if pos >= len(live) or live[pos] != o:
                self.order[i] = -1
                continue
            self.order_index = i + 1
            return pos

    # ---- cluster.py:386-413 ----
    def update_successes(self, success: bool):
        if len(self.attempts) == self.attempts.maxlen:
            self.successes -= self.attempts.popleft()
        self.successes += success
        self.attempts.append(success)
        if len(self.attempts) == self.attempts.maxlen and self.successes < self.minsuccesses:
            self.peak_valley_ratio += 0.1
            self.attempts.clear()
            self.successes = 0
            self.order_index = 0

    # ---- cluster.py:545-604 ----
    def find_cluster(self):
        while True:
            seed = self.get_next_seed()
            medoid, distances, density = self.wander_medoid(seed)
            thr = self.find_threshold(distances)
            if self.record:
                self.trace.append((int(self.indices[seed]), int(self.indices[medoid]), density, thr))
            orig_medoid = int(self.indices[medoid])
            if thr == "loner":
                c = OracleCluster(orig_medoid, seed, np.array([orig_medoid]), self.peak_valley_ratio,
                                  None, None, self.successes, len(self.attempts))
                return c, np.array([medoid], dtype=np.int64)
            if thr is None:
                if self.peak_valley_ratio > 0.55:
                    pts = self._smaller(distances, DEFAULT_RADIUS)
                    c = OracleCluster(orig_medoid, seed, self.indices[pts].copy(), self.peak_valley_ratio,
                                      None, DEFAULT_RADIUS, self.successes, len(self.attempts))
                    return c, pts
                self.update_successes(False)
                continue
            threshold, observed_pvr = thr
            pts = self._smaller(distances, threshold)
            c = OracleCluster(orig_medoid, seed, self.indices[pts].copy(), self.peak_valley_ratio,
                              observed_pvr, threshold, self.successes, len(self.attempts))
            if self.peak_valley_ratio < 0.55:
                self.update_successes(True)
            return c, pts

    # ---- cluster.py:298-335 ----
    def __next__(self) -> OracleCluster:
        if self.n_remaining_points == 0:
            raise StopIteration
        cluster, points = self.find_cluster()
        self.n_emitted_clusters += 1
        self.n_remaining_points -= len(points)
        keep = np.ones(self.nrows, dtype=np.uint8)
        keep[points] = 0
        self.nrows = int(
            self.lib.ok_pack_rows(
                _p(self.matrix, ctypes.c_float), _p(self.lens, ctypes.c_float),
                _p(self.indices, ctypes.c_int64), _p(keep, ctypes.c_uint8), self.nrows, self.matrix.shape[1],
            )
        )
        return cluster
