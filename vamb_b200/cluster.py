__doc__ = """Iterative medoid clustering on H100 -- drop-in for ``vamb.cluster``.

Same public surface as the reference module (RasmussenLab/vamb, vamb/cluster.py):
``ClusterGenerator(matrix, lengths, maxsteps, windowsize, minsuccesses, destroy,
normalized, cuda, rng_seed)`` is an iterator of ``Cluster`` objects.  The host code
below keeps the reference's *decision logic* (seed order, Python ``random`` call
sequence, success window, peak/valley scan in Python floats); every O(N) tensor
expression is a hand-written sm_90a kernel reached through the C ABI of
include/vamb_b200.h:

    reference (vamb/cluster.py)                this module
    _normalize                :653-669    ->   vk_normalize_rows
    _calc_distances           :672-676  \\
    sample_medoid             :606-637   >->   vk_probe_sync   (one pass: distances, within
    find_threshold (head)     :457-481  /        set, exact density, histogram, neighbour list)
    wander_medoid candidates  :427-448    ->   vk_eval_candidates_sync (<= maxsteps medoids / pass)
    _smaller_indices + mask   :640-650,308 ->  vk_select_members_sync
    pack / overwrite_matrix   :318-335    ->   vk_compact_rows_sync (when < 90 % of the rows are live)

Results follow the reference's CPU semantics (``cuda=False`` path, where emitted rows
no longer exist) under "vk arithmetic v1" (DESIGN.md section 3) and are bit-identical to
oracle/cluster_oracle.py.  There is no CPU fallback: without the CUDA extension and an
sm_90 device construction raises.
"""

import os as _os
import random as _random
from collections import deque as _deque
from math import ceil as _ceil
from typing import Optional, Union

import numpy as _np
import torch as _torch

from . import _lib

_DEFAULT_RADIUS = 0.06  # vamb/cluster.py:12
_MEDOID_RADIUS = 0.05  # vamb/cluster.py:14
_DELTA_X = 0.005  # vamb/cluster.py:16
_XMAX = 0.3  # vamb/cluster.py:17
_NBINS = _ceil(_XMAX / _DELTA_X)
# A row within 0.05 of a candidate that is itself within 0.05 of the medoid lies within
# 0.19 of the medoid (angles add: 2 * acos(0.9) -> 0.5 * (1 - cos) = 0.19); 0.2 leaves a
# margin four orders of magnitude above fp32 rounding.
_PRUNE_RADIUS = 0.2
_DENSITY_UNIT = 2.0 ** -29

# N(0, 0.01^2) pdf at -0.075..0.075 in steps of _DELTA_X, times _DELTA_X, in fp32
# (vamb/cluster.py:39-73).
_NORMALPDF = _np.float32(_DELTA_X) * _np.array(
    [
        2.43432053e-11, 9.13472041e-10, 2.66955661e-08, 6.07588285e-07, 1.07697600e-05,
        1.48671951e-04, 1.59837411e-03, 1.33830226e-02, 8.72682695e-02, 4.43184841e-01,
        1.75283005e00, 5.39909665e00, 1.29517596e01, 2.41970725e01, 3.52065327e01,
        3.98942280e01, 3.52065327e01, 2.41970725e01, 1.29517596e01, 5.39909665e00,
        1.75283005e00, 4.43184841e-01, 8.72682695e-02, 1.33830226e-02, 1.59837411e-03,
        1.48671951e-04, 1.07697600e-05, 6.07588285e-07, 2.66955661e-08, 9.13472041e-10,
        2.43432053e-11,
    ],
    dtype=_np.float32,
)


def _histogram_edges() -> _np.ndarray:
    """fp32 edge table of ``torch.linspace(0, 0.3, 61)`` (vamb/cluster.py:288), spelled out so
    that it does not depend on the torch build: step in fp32, fused multiply-add per edge."""
    steps = _NBINS + 1
    start, end = _np.float32(0.0), _np.float32(_XMAX)
    step = _np.float32((end - start) / _np.float32(steps - 1))
    out = _np.empty(steps, dtype=_np.float32)
    for i in range(steps):
        if i < steps // 2:
            out[i] = _np.float32(float(start) + float(step) * i)
        else:
            out[i] = _np.float32(float(end) - float(step) * (steps - 1 - i))
    return out


class Loner:
    __slots__ = []


class NoThreshold:
    __slots__ = []


class Cluster:
    """One emitted cluster (same fields as vamb/cluster.py:76-119)."""

    __slots__ = [
        "medoid", "seed", "members", "maximal_pvr", "observed_pvr", "radius",
        "isdefault", "successes", "attempts",
    ]

    def __init__(self, medoid: int, seed: int, members: _np.ndarray, maximal_pvr: float,
                 observed_pvr: Optional[float], radius: Optional[float], successes: int, attempts: int):
        self.medoid = medoid
        self.seed = seed
        self.members = members
        self.maximal_pvr = maximal_pvr
        self.observed_pvr = observed_pvr
        self.radius = radius
        self.successes = successes
        self.attempts = attempts

    @property
    def kind_str(self) -> str:
        if self.observed_pvr is not None:
            return "normal"
        return "loner" if self.radius is None else "fallback"


class ClusterBlock:
    """A run of consecutive clusters as arrays (``ClusterGenerator.next_block``): what
    ``cluster_and_write_files`` (vamb/__main__.py:1325-1377) needs per cluster, without a Python object per
    cluster.  ``members`` holds the ascending original ids of cluster 0, then cluster 1, ...; cluster i owns
    ``members[offsets[i]:offsets[i + 1]]``.  ``radius`` / ``observed_pvr`` are NaN where the reference has None."""

    __slots__ = ["medoid", "seed", "offsets", "members", "maximal_pvr", "observed_pvr", "radius", "kind",
                 "successes", "attempts"]

    _KIND_STR = ("loner", "fallback", "normal")

    def __len__(self) -> int:
        return len(self.medoid)

    def kind_strs(self) -> list:
        return [self._KIND_STR[k] for k in self.kind.tolist()]

    def clusters(self):
        "The same clusters as ``Cluster`` objects (compatibility path)."
        for i in range(len(self)):
            k = int(self.kind[i])
            yield Cluster(
                int(self.medoid[i]), int(self.seed[i]), self.members[self.offsets[i]:self.offsets[i + 1]].copy(),
                float(self.maximal_pvr[i]), float(self.observed_pvr[i]) if k == 2 else None,
                None if k == 0 else float(self.radius[i]), int(self.successes[i]), int(self.attempts[i]),
            )


class _Probe:
    """Host view of one vk_probe_header."""

    __slots__ = ["medoid", "density", "hist", "n_within", "n_lt", "n_nl", "rank", "within"]


class ClusterGenerator:
    """Iterative medoid cluster generator. Iterate this object to get clusters.

    Inputs:
        matrix: A (obs x features) Numpy matrix of data type numpy.float32
        lengths: Numpy array of sequence lengths (integral values)
        maxsteps: Stop searching for optimal medoid after N futile attempts [25]
        windowsize: Length of window to count successes [300]
        minsuccesses: Minimum acceptable number of successes [15]
        destroy: Save memory by destroying matrix while clustering [False]
        normalized: Matrix is already preprocessed [False]
        cuda: accepted for API compatibility; this implementation always runs on the GPU
        rng_seed: seed of the Python RNG that samples medoid candidates [0]
    """

    __slots__ = [
        "maxsteps", "minsuccesses", "cuda", "rng", "lengths", "indices", "order", "order_index",
        "n_emitted_clusters", "n_remaining_points", "peak_valley_ratio", "attempts", "successes",
        "histogram", "histogram_edges", "kept_mask",
        # device state
        "_stream", "_d", "_n_act", "_n_total", "_m", "_len", "_kept", "_orig", "_m2", "_len2", "_kept2",
        "_orig2", "_nl_rows", "_nl_d", "_hdr", "_hdr_host", "_hdr_np", "_within_over", "_edges",
        "_cand_out", "_cand_out_host", "_members", "_members_host", "_tile_scratch", "_row_of_orig",
        "_user_matrix", "_prune_radius", "_nl_radius", "_n_probes", "_n_evals", "_pack_fraction",
        "_native", "_native_cfg", "_native_keep", "_result", "_native_cur",
    ]

    def __repr__(self) -> str:
        return f"ClusterGenerator({self.n_remaining_points} points, {self.n_emitted_clusters} clusters)"

    def __str__(self) -> str:
        return f"""ClusterGenerator({self.n_remaining_points} points, {self.n_emitted_clusters} clusters)
  CUDA:         True
  maxsteps:     {self.maxsteps}
  minsuccesses: {self.minsuccesses}
  pvr:          {self.peak_valley_ratio}
  successes:    {self.successes}/{len(self.attempts)}
"""

    # same argument checks, in the same order, as vamb/cluster.py:194-222
    def _check_params(self, matrix, lengths, maxsteps, windowsize, minsuccesses) -> None:
        if isinstance(matrix, _torch.Tensor):
            if matrix.dtype != _torch.float32 or not matrix.is_cuda:
                raise ValueError("A tensor matrix must be a float32 CUDA tensor")
        elif matrix.dtype != _np.float32:
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

    def __init__(
        self,
        matrix: _np.ndarray,
        lengths: _np.ndarray,
        maxsteps: int = 25,
        windowsize: int = 300,
        minsuccesses: int = 15,
        destroy: bool = False,
        normalized: bool = False,
        cuda: bool = False,
        rng_seed: int = 0,
        _driver: Optional[str] = None,
        _pack_fraction: float = 0.9,
    ):
        self._check_params(matrix, lengths, maxsteps, windowsize, minsuccesses)
        if matrix.ndim != 2:
            raise ValueError("Matrix must be 2-dimensional")
        n, d = matrix.shape
        lengths = _np.asarray(lengths)
        len32 = lengths.astype(_np.float32)  # torch.Tensor(lengths), vamb/cluster.py:277
        if n and not (_np.all(len32 >= 0) and _np.all(len32 == _np.floor(len32))):
            raise ValueError("lengths must be non-negative integral values (contig lengths)")
        if float(len32.astype(_np.float64).sum()) >= 2.0 ** 50:
            raise ValueError("total sequence length >= 2^50 is outside the exact-density range")
        if n >= 2 ** 31:
            raise ValueError("more than 2^31 - 1 observations are not supported")

        _lib.require_device()
        dev = _torch.device("cuda", _torch.cuda.current_device())
        self._stream = _torch.cuda.current_stream().cuda_stream

        self.maxsteps = maxsteps
        self.minsuccesses = minsuccesses
        self.cuda = True
        self.rng = _random.Random(rng_seed)
        self._d = d
        self._n_act = n
        self._n_total = n

        # ---- device-resident state (HBM layout: DESIGN.md section 4) ----
        if isinstance(matrix, _torch.Tensor):
            # a latent that is already resident in HBM (VAE.encode output kept on the device)
            self._m = matrix.contiguous() if destroy else matrix.clone().contiguous()
        else:
            self._m = _torch.from_numpy(_np.ascontiguousarray(matrix)).to(dev)
        self._len = _torch.from_numpy(len32).to(dev)
        self._kept = _torch.ones(n, dtype=_torch.uint8, device=dev)
        self._orig = _torch.arange(n, dtype=_torch.int32, device=dev)
        self._m2 = self._len2 = self._kept2 = self._orig2 = None  # compaction targets, allocated lazily
        self._nl_rows = _torch.empty(n, dtype=_torch.int32, device=dev)
        self._nl_d = _torch.empty(n, dtype=_torch.float32, device=dev)
        self._within_over = _torch.empty(n, dtype=_torch.int32, device=dev)
        self._hdr = _torch.zeros(_lib.HDR_SIZE, dtype=_torch.uint8, device=dev)
        self._hdr_host = _torch.zeros(_lib.HDR_SIZE, dtype=_torch.uint8).pin_memory()
        self._hdr_np = self._hdr_host.numpy()
        self._cand_out = _torch.zeros(3 * _lib.VK_MAX_CAND, dtype=_torch.int64, device=dev)
        self._cand_out_host = _torch.zeros(3 * _lib.VK_MAX_CAND, dtype=_torch.int64).pin_memory()
        self._members = _torch.empty(n + 1, dtype=_torch.int32, device=dev)
        self._members_host = _torch.zeros(4096, dtype=_torch.int32).pin_memory()
        self._tile_scratch = _torch.zeros(2 + (n + 1023) // 1024, dtype=_torch.int32, device=dev)
        self.histogram_edges = _histogram_edges()
        self._edges = _torch.from_numpy(self.histogram_edges).to(dev)
        self._n_probes = 0
        self._n_evals = 0
        self._pack_fraction = _pack_fraction
        self._native = None

        if not normalized:
            _lib.check(_lib.lib.vk_normalize_rows(self._m.data_ptr(), n, d, self._stream))
            self._prune_radius = _PRUNE_RADIUS
            self._nl_radius = _XMAX
        else:
            # the pruning bound needs |row|^2 = 1/2; verify instead of trusting the flag
            nbad = _torch.zeros(1, dtype=_torch.int32, device=dev)
            _lib.check(_lib.lib.vk_check_normalized(self._m.data_ptr(), n, d, 1e-4, nbad.data_ptr(), self._stream))
            if int(nbad.item()) == 0:
                self._prune_radius = _PRUNE_RADIUS
                self._nl_radius = _XMAX
            else:
                self._prune_radius = float("inf")
                self._nl_radius = float("inf")
        is_numpy = isinstance(matrix, _np.ndarray)
        if destroy and not normalized and is_numpy:
            # the reference normalises the caller's array in place (vamb/cluster.py:253-258)
            if matrix.flags.c_contiguous and matrix.flags.writeable:
                _torch.from_numpy(matrix).copy_(self._m)
        self._user_matrix = matrix if (destroy and is_numpy) else None

        # ---- host-side decision state (vamb/cluster.py:266-292) ----
        self.indices = _np.arange(n, dtype=_np.int64)  # original id of every live device row
        self.kept_mask = _np.ones(n, dtype=bool)  # host mirror of the device mask
        self.order = _np.argsort(lengths)[::-1].copy()
        self.order_index = 0
        self.lengths = len32
        self.n_emitted_clusters = 0
        self.n_remaining_points = n
        self.peak_valley_ratio = 0.1
        self.attempts = _deque(maxlen=windowsize)
        self.successes = 0
        self.histogram = _np.empty(_NBINS, dtype=_np.float32)

        driver = _driver or _os.environ.get("VAMB_B200_CLUSTER_DRIVER", "native")
        if driver not in ("native", "python"):
            raise ValueError(f"unknown cluster driver {driver!r}")
        if driver == "native":
            self._create_native(windowsize, rng_seed)

    def _create_native(self, windowsize: int, rng_seed: int) -> None:
        """Hand the decision loop to the C++ driver (vk_cluster_next): same logic, same clusters."""
        from . import _cluster_native as _cn

        n = self._n_total
        self._m2 = _torch.empty_like(self._m)
        self._len2 = _torch.empty_like(self._len)
        self._kept2 = _torch.empty_like(self._kept)
        self._orig2 = _torch.empty_like(self._orig)
        cfg = _cn.VkClusterConfig()
        cfg.n, cfg.d = n, self._d
        cfg.maxsteps, cfg.windowsize, cfg.minsuccesses = self.maxsteps, windowsize, self.minsuccesses
        cfg.nl_radius, cfg.prune_radius = self._nl_radius, self._prune_radius
        cfg.pack_fraction = self._pack_fraction
        for name, t in (("matrix", self._m), ("matrix2", self._m2), ("lengths", self._len), ("lengths2", self._len2),
                        ("kept", self._kept), ("kept2", self._kept2), ("orig", self._orig), ("orig2", self._orig2),
                        ("nl_rows", self._nl_rows), ("nl_dists", self._nl_d), ("hdr", self._hdr),
                        ("within_overflow", self._within_over), ("edges", self._edges), ("cand_out", self._cand_out),
                        ("members", self._members), ("tile_scratch", self._tile_scratch),
                        ("hdr_host", self._hdr_host), ("cand_out_host", self._cand_out_host),
                        ("members_host", self._members_host)):
            setattr(cfg, name, t.data_ptr())
        cfg.members_host_cap = self._members_host.numel()
        key = _cn.seed_key(rng_seed)
        order = _np.ascontiguousarray(self.order, dtype=_np.int64)
        pdf = _np.ascontiguousarray(_NORMALPDF, dtype=_np.float32)
        cfg.seed_key_len = len(key)
        cfg.seed_key = _lib.ctypes.cast(key, _lib.ctypes.c_void_p)
        cfg.order_host = order.ctypes.data
        cfg.normalpdf_host = pdf.ctypes.data
        cfg.stream = self._stream
        handle = _lib.ctypes.c_void_p()
        _lib.check(_cn._L.vk_cluster_create(_lib.ctypes.byref(handle), _lib.ctypes.byref(cfg)))
        self._native = handle
        self._native_cur = 0
        self._native_cfg = cfg
        self._native_keep = (key, order, pdf)
        self._result = _cn.VkClusterResult()

    def __del__(self):
        try:
            if self._native is not None:
                from . import _cluster_native as _cn

                _cn._L.vk_cluster_destroy(self._native)
                self._native = None
        except Exception:
            pass

    def _next_native(self) -> Cluster:
        from . import _cluster_native as _cn

        res = self._result
        rc = _cn._L.vk_cluster_next(self._native, _lib.ctypes.byref(res))
        if rc == 2:
            raise StopIteration
        _lib.check(rc)
        members = _np.ctypeslib.as_array(res.members_host, shape=(res.n_members,)).copy()
        kind = res.kind
        cluster = Cluster(
            int(res.medoid), int(res.seed), members, res.maximal_pvr,
            res.observed_pvr if kind == 2 else None,
            None if kind == 0 else res.radius,
            int(res.successes), int(res.attempts),
        )
        self.n_emitted_clusters += 1
        self.n_remaining_points = int(res.n_remaining)
        self.peak_valley_ratio = res.peak_valley_ratio
        self._sync_native_stats()
        return cluster

    def _sync_native_stats(self) -> None:
        from . import _cluster_native as _cn

        stats = (_lib.ctypes.c_int64 * 8)()
        _cn._L.vk_cluster_stats(self._native, stats)
        self._n_probes, self._n_evals, self._n_act = int(stats[0]), int(stats[1]), int(stats[3])
        if int(stats[4]) != self._native_cur:
            # the driver packed into the other buffer set: keep the Python-side views on the live one
            self._native_cur = int(stats[4])
            self._m, self._m2 = self._m2, self._m
            self._len, self._len2 = self._len2, self._len
            self._kept, self._kept2 = self._kept2, self._kept
            self._orig, self._orig2 = self._orig2, self._orig
        # mirror the window counters (``__str__``, callers that inspect them); ``indices`` / ``kept_mask`` / ``order``
        # are O(N) host arrays owned by the C++ driver in this mode and are not mirrored per cluster
        self.successes, self.order_index = int(stats[5]), int(stats[7])
        if len(self.attempts) != int(stats[6]):
            self.attempts = _deque([False] * int(stats[6]), maxlen=self.attempts.maxlen)

    def next_block(self, max_clusters: int = 1024) -> ClusterBlock:
        """Up to ``max_clusters`` further clusters in ONE foreign call, as arrays (empty block = exhausted).
        Interleaves freely with ``next()``; the Python driver falls back to a per-cluster loop."""
        blk = ClusterBlock()
        m = max(1, int(max_clusters))
        if self._native is None:
            got = []
            for _ in range(m):
                try:
                    got.append(next(self))
                except StopIteration:
                    break
            blk.medoid = _np.array([c.medoid for c in got], dtype=_np.int64)
            blk.seed = _np.array([c.seed for c in got], dtype=_np.int64)
            sizes = _np.array([len(c.members) for c in got], dtype=_np.int64)
            blk.offsets = _np.concatenate([[0], _np.cumsum(sizes)]).astype(_np.int64)
            blk.members = _np.concatenate([_np.asarray(c.members, dtype=_np.int64) for c in got]) if got else _np.empty(0, _np.int64)
            blk.maximal_pvr = _np.array([c.maximal_pvr for c in got], dtype=_np.float64)
            blk.observed_pvr = _np.array([_np.nan if c.observed_pvr is None else c.observed_pvr for c in got], dtype=_np.float64)
            blk.radius = _np.array([_np.nan if c.radius is None else c.radius for c in got], dtype=_np.float64)
            blk.kind = _np.array([{"loner": 0, "fallback": 1, "normal": 2}[c.kind_str] for c in got], dtype=_np.int32)
            blk.successes = _np.array([c.successes for c in got], dtype=_np.int32)
            blk.attempts = _np.array([c.attempts for c in got], dtype=_np.int32)
            return blk
        from . import _cluster_native as _cn

        arrs = {name: _np.empty(m, dtype=dt) for name, dt in (
            ("medoid", _np.int64), ("seed", _np.int64), ("n_members", _np.int64), ("maximal_pvr", _np.float64),
            ("observed_pvr", _np.float64), ("radius", _np.float64), ("kind", _np.int32), ("successes", _np.int32),
            ("attempts", _np.int32))}
        members = _np.empty(max(1, self.n_remaining_points), dtype=_np.int64)
        c = _cn.VkClusterBlock()
        c.max_clusters = m
        for name, a in arrs.items():
            setattr(c, name, a.ctypes.data)
        c.members = members.ctypes.data
        _lib.check(_cn._L.vk_cluster_next_block(self._native, _lib.ctypes.byref(c)))
        k = int(c.n_clusters)
        for name in ("medoid", "seed", "maximal_pvr", "observed_pvr", "radius", "kind", "successes", "attempts"):
            setattr(blk, name, arrs[name][:k])
        blk.offsets = _np.concatenate([[0], _np.cumsum(arrs["n_members"][:k])]).astype(_np.int64)
        blk.members = members[: int(c.n_members_total)]
        self.n_emitted_clusters += k
        self.n_remaining_points = int(c.n_remaining)
        self.peak_valley_ratio = float(c.peak_valley_ratio)
        self._sync_native_stats()
        return blk

    def iter_blocks(self, max_clusters: int = 1024):
        "Iterate the remaining clusters block by block."
        while True:
            blk = self.next_block(max_clusters)
            if len(blk) == 0:
                return
            yield blk

    def _probe_mapped_once(self, row: int, state: dict) -> None:
        """One probe exactly as the native driver issues it -- a single launch with the mapped completion
        (vk_probe_mapped) -- for timing tools (bench.py, tools/probe_speed.py).  ``state`` carries the pinned
        buffers between calls."""
        if not state:
            self._hdr.zero_()
            state["hdr"] = _torch.zeros(_lib.HDR_SIZE, dtype=_torch.uint8).pin_memory()
            state["ticket"] = _torch.zeros(2, dtype=_torch.int32, device=self._m.device)  # [ticket, work counter]
            state["flag"] = _torch.zeros(1, dtype=_torch.int32).pin_memory()
            state["seq"] = 0
            _torch.cuda.synchronize()
        state["seq"] += 1
        _lib.check(_lib.lib.vk_probe_mapped(
            self._m.data_ptr(), self._len.data_ptr(), self._kept.data_ptr(), self._n_act, self._d, int(row),
            self._nl_radius, self._edges.data_ptr(), self._hdr.data_ptr(), self._within_over.data_ptr(),
            self._nl_rows.data_ptr(), self._nl_d.data_ptr(), state["hdr"].data_ptr(), state["ticket"].data_ptr(),
            state["flag"].data_ptr(), state["seq"], state["ticket"].data_ptr() + 4, self._stream))

    def _timing(self) -> dict:
        "Host seconds the native driver spent per call kind so far (diagnostics / bench)."
        from . import _cluster_native as _cn

        out = (_lib.ctypes.c_double * 8)()
        if self._native is None:
            return {}
        _cn._L.vk_cluster_timing(self._native, out)
        return dict(zip(("probe", "eval", "select", "pack", "total", "lazy_moves", "rebases", "sum_nl_per_eval"),
                        (float(x) for x in out)))

    # ------------------------------------------------------------------ API extras
    @property
    def matrix(self) -> _torch.Tensor:
        """The (normalised) rows that are still unclustered, as a CPU tensor."""
        if self._user_matrix is not None and self.n_emitted_clusters == 0:
            return _torch.from_numpy(self._user_matrix)
        m = self._m[: self._n_act]
        if self.n_emitted_clusters:
            m = m[self._kept[: self._n_act].bool()]
        return m.cpu()

    def __iter__(self):
        return self

    # ------------------------------------------------------------------ device calls
    def _probe(self, row: int) -> _Probe:
        self._n_probes += 1
        _lib.check(
            _lib.lib.vk_probe_sync(
                self._m.data_ptr(), self._len.data_ptr(), self._kept.data_ptr(), self._n_act, self._d,
                int(row), self._nl_radius, self._edges.data_ptr(), self._hdr.data_ptr(),
                self._within_over.data_ptr(), self._nl_rows.data_ptr(), self._nl_d.data_ptr(),
                self._hdr_host.data_ptr(), self._stream,
            )
        )
        h = self._hdr_np
        p = _Probe()
        p.medoid = int(row)
        dens = h[_lib.HDR_DENSITY_LO:_lib.HDR_DENSITY_LO + 16].view(_np.uint64)
        p.density = (int(dens[1]) << 12) + int(dens[0])  # exact, in units of 2^-29
        p.hist = h[_lib.HDR_HIST:_lib.HDR_HIST + 8 * _NBINS].view(_np.uint64).copy()
        counts = h[_lib.HDR_NWITHIN:_lib.HDR_NWITHIN + 16].view(_np.int32)
        p.n_within, p.n_lt, p.n_nl, p.rank = (int(x) for x in counts)
        k = min(p.n_within, _lib.VK_PROBE_INLINE)
        within = h[_lib.HDR_WITHIN:_lib.HDR_WITHIN + 4 * k].view(_np.int32).copy()
        if p.n_within > _lib.VK_PROBE_INLINE:
            rest = self._within_over[_lib.VK_PROBE_INLINE:p.n_within].cpu().numpy()
            within = _np.concatenate([within, rest])
        within.sort()  # ascending row order = torch.nonzero order (vamb/cluster.py:626)
        p.within = within
        return p

    def _eval_candidates(self, probe: _Probe, rows: list) -> list:
        out: list = []
        for i in range(0, len(rows), _lib.VK_MAX_CAND):
            chunk = rows[i:i + _lib.VK_MAX_CAND]
            arr = (_lib.c_int32 * len(chunk))(*chunk)
            self._n_evals += 1
            _lib.check(
                _lib.lib.vk_eval_candidates_sync(
                    self._m.data_ptr(), self._len.data_ptr(), self._d, self._nl_rows.data_ptr(),
                    self._nl_d.data_ptr(), probe.n_nl, self._prune_radius, arr, len(chunk),
                    self._cand_out.data_ptr(), self._cand_out_host.data_ptr(), self._stream,
                )
            )
            res = self._cand_out_host.numpy().view(_np.uint64)
            lo, hi = res[: len(chunk)], res[_lib.VK_MAX_CAND:_lib.VK_MAX_CAND + len(chunk)]
            out.extend((int(h) << 12) + int(l) for l, h in zip(lo, hi))
        return out

    def _select_members(self, probe: _Probe, threshold: float) -> _np.ndarray:
        cap = self._members_host.numel()
        _lib.check(
            _lib.lib.vk_select_members_sync(
                self._nl_rows.data_ptr(), self._nl_d.data_ptr(), probe.n_nl, threshold,
                self._orig.data_ptr(), self._kept.data_ptr(), self._members.data_ptr(),
                self._members_host.data_ptr(), cap, self._stream,
            )
        )
        mh = self._members_host.numpy()
        cnt = int(mh[0])
        if cnt + 1 <= cap:
            ids = mh[1:1 + cnt].astype(_np.int64)
        else:
            ids = self._members[1:1 + cnt].cpu().numpy().astype(_np.int64)
        ids.sort()
        return ids

    def pack(self):
        "Physically remove emitted rows from the device arrays (vamb/cluster.py:318-335)."
        n, d = self._n_act, self._d
        if self._m2 is None:
            self._m2 = _torch.empty_like(self._m)
            self._len2 = _torch.empty_like(self._len)
            self._kept2 = _torch.empty_like(self._kept)
            self._orig2 = _torch.empty_like(self._orig)
        n_out = _lib.c_int64(0)
        _lib.check(
            _lib.lib.vk_compact_rows_sync(
                self._m.data_ptr(), self._len.data_ptr(), self._orig.data_ptr(), self._kept.data_ptr(), n, d,
                self._m2.data_ptr(), self._len2.data_ptr(), self._orig2.data_ptr(), self._kept2.data_ptr(),
                self._tile_scratch.data_ptr(), _lib.ctypes.byref(n_out), self._stream,
            )
        )
        self._m, self._m2 = self._m2, self._m
        self._len, self._len2 = self._len2, self._len
        self._kept, self._kept2 = self._kept2, self._kept
        self._orig, self._orig2 = self._orig2, self._orig
        self._n_act = int(n_out.value)
        self.indices = self.indices[self.kept_mask]
        self.kept_mask = _np.ones(self._n_act, dtype=bool)
        assert len(self.indices) == self._n_act

    def pack_order(self):
        "Remove all used points from self.order (vamb/cluster.py:337-340)."
        self.order = self.order[self.order > -1]
        assert len(self.order) > 0

    # ------------------------------------------------------------------ host decision logic
    def get_next_seed(self) -> int:
        "Next seed as a device row index (vamb/cluster.py:342-384)."
        n_original_contigs = len(self.order)
        i = self.order_index - 1
        while True:
            i = (i + 1) % n_original_contigs
            if i == 0 and self.n_emitted_clusters > 0:
                self.pack_order()
                n_original_contigs = len(self.order)
            order = self.order[i]
            if order == -1:
                continue
            row = int(_np.searchsorted(self.indices, order))
            if row >= len(self.indices) or self.indices[row] != order or not self.kept_mask[row]:
                self.order[i] = -1
                continue
            self.order_index = i + 1
            return row

    def update_successes(self, success: bool):
        "Success window / peak_valley_ratio relaxation (vamb/cluster.py:386-413)."
        if len(self.attempts) == self.attempts.maxlen:
            self.successes -= self.attempts.popleft()
        self.successes += success
        self.attempts.append(success)
        if len(self.attempts) == self.attempts.maxlen and self.successes < self.minsuccesses:
            self.peak_valley_ratio += 0.1
            self.attempts.clear()
            self.successes = 0
            self.order_index = 0

    def wander_medoid(self, seed: int):
        """vamb/cluster.py:415-450 with the candidates of a round evaluated in ONE device pass.
        The densities of a round do not depend on each other, so evaluating them together and
        then replaying the reference's sequential accept/restart rule is semantics-preserving."""
        tried = {seed}
        probe = self._probe(seed)
        seed_rank = probe.rank
        local_density = probe.density
        while True:
            candidates = [r for r in probe.within.tolist() if r not in tried]
            candidates = self.rng.sample(candidates, k=min(len(candidates), self.maxsteps))
            if not candidates:
                break
            densities = self._eval_candidates(probe, candidates)
            winner = -1
            for i, cand in enumerate(candidates):
                tried.add(cand)
                if densities[i] > local_density:
                    winner = i
                    break
            if winner < 0:
                break
            probe = self._probe(candidates[winner])
            if probe.density != densities[winner]:  # the two kernels share one arithmetic
                raise _lib.VkError("internal error: probe and candidate densities disagree")
            local_density = probe.density
        return probe, seed_rank

    def find_threshold(self, probe: _Probe) -> Union[Loner, NoThreshold, tuple]:
        "vamb/cluster.py:452-543 on the device-made histogram."
        if probe.n_lt == 1:
            return Loner()
        self.histogram[:] = probe.hist.astype(_np.float32)  # exact integer sums, rounded once
        pdf_len = len(_NORMALPDF)
        densities = _np.zeros(_NBINS + pdf_len - 1, dtype=_np.float32)
        for i in range(_NBINS):
            densities[i:i + pdf_len] += _NORMALPDF * self.histogram[i]
        densities = densities[15:-15]

        peak_density = 0.0
        peak_over = False
        minimum_x = 0.0
        threshold = None
        delta_x = _XMAX / _NBINS
        x = 0
        density_at_minimum = 0.0
        for density in densities.tolist():
            if not peak_over and density > peak_density:
                if x > 0.1:
                    return NoThreshold()
                peak_density = density
            if not peak_over and density < 0.6 * peak_density:
                peak_over = True
                density_at_minimum = density
            if peak_over and density > 1.5 * density_at_minimum:
                break
            if peak_over and density < density_at_minimum:
                minimum_x, density_at_minimum = x, density
                if density < self.peak_valley_ratio * peak_density:
                    threshold = minimum_x
            x += delta_x
        if threshold is None:
            return NoThreshold()
        if threshold > 0.2 + self.peak_valley_ratio:
            return NoThreshold()
        return (threshold, density_at_minimum / peak_density)

    def find_cluster(self):
        "vamb/cluster.py:545-604."
        while True:
            seed = self.get_next_seed()
            probe, seed_rank = self.wander_medoid(seed)
            medoid = probe.medoid
            threshold = self.find_threshold(probe)
            orig_medoid = int(self.indices[medoid])
            if isinstance(threshold, Loner):
                # only the medoid itself has d < 0.05 -> the entries with d <= 0 are {medoid}
                members = self._select_members(probe, 0.0)
                if len(members) != 1 or members[0] != orig_medoid:
                    raise _lib.VkError("internal error: loner selection")
                return Cluster(orig_medoid, seed_rank, _np.array([orig_medoid]), self.peak_valley_ratio,
                               None, None, self.successes, len(self.attempts))
            if isinstance(threshold, NoThreshold):
                if self.peak_valley_ratio > 0.55:
                    members = self._select_members(probe, _DEFAULT_RADIUS)
                    return Cluster(orig_medoid, seed_rank, members, self.peak_valley_ratio, None,
                                   _DEFAULT_RADIUS, self.successes, len(self.attempts))
                self.update_successes(False)
                continue
            thr, observed_pvr = threshold
            members = self._select_members(probe, thr)
            cluster = Cluster(orig_medoid, seed_rank, members, self.peak_valley_ratio, observed_pvr, thr,
                              self.successes, len(self.attempts))
            if self.peak_valley_ratio < 0.55:
                self.update_successes(True)
            return cluster

    def __next__(self) -> Cluster:
        if self._native is not None:
            return self._next_native()
        if self.n_remaining_points == 0:
            raise StopIteration
        assert self.n_remaining_points > 0
        cluster = self.find_cluster()
        self.n_emitted_clusters += 1
        self.n_remaining_points -= len(cluster.members)
        rows = _np.searchsorted(self.indices, cluster.members)
        self.kept_mask[rows] = False
        # physical compaction only when it pays: the scans are O(live rows)
        if self.n_remaining_points and self.n_remaining_points < self._pack_fraction * self._n_act:
            self.pack()
        return cluster


def write_clusters_tsv(generator: ClusterGenerator, sequence_names, sequence_lens, base_clusters_name: str,
                       bin_prefix: Optional[str] = None, max_clusters: Optional[int] = None,
                       block: int = 2048) -> tuple:
    """Stream the clusters of ``generator`` into ``<base>_unsplit.tsv`` and ``<base>_metadata.tsv`` with the exact
    text the reference's per-cluster loop prints (vamb/__main__.py:1310-1377, binsplitter disabled): cluster names
    ``bin_prefix + str(index + 1)``, one ``name\tcontig`` line per member, and the metadata columns name / radius
    (3 decimals) / peak valley ratio (2 decimals) / kind / bp / ncontigs / medoid.  Works block-wise on arrays:
    name lookups, base-pair sums and line assembly are NumPy operations per block of clusters, not Python per member.
    Returns (n_clusters, n_contigs)."""
    names = _np.asarray(sequence_names, dtype=object)
    lens = _np.asarray(sequence_lens)
    prefix = "" if bin_prefix is None else bin_prefix
    n_clusters = n_contigs = 0
    with open(base_clusters_name + "_metadata.tsv", "w") as meta, open(base_clusters_name + "_unsplit.tsv", "w") as unsplit:
        print("name\tradius\tpeak valley ratio\tkind\tbp\tncontigs\tmedoid", file=meta)
        print("clustername\tcontigname", file=unsplit)  # vamb.vambtools.CLUSTERS_HEADER
        while max_clusters is None or n_clusters < max_clusters:
            want = block if max_clusters is None else min(block, max_clusters - n_clusters)
            blk = generator.next_block(want)
            k = len(blk)
            if k == 0:
                break
            sizes = _np.diff(blk.offsets)
            cl_names = _np.array([prefix + str(i) for i in range(n_clusters + 1, n_clusters + k + 1)], dtype=object)
            member_names = names[blk.members]
            unsplit.write("\n".join((_np.repeat(cl_names, sizes) + "\t" + member_names).tolist()))
            unsplit.write("\n")
            bp = _np.add.reduceat(lens[blk.members], blk.offsets[:-1]) if len(blk.members) else _np.zeros(k, dtype=lens.dtype)
            kinds = blk.kind_strs()
            rows = []
            for i in range(k):  # per cluster (not per member): seven short fields
                radius = None if blk.kind[i] == 0 else round(float(blk.radius[i]), 3)
                pvr = round(float(blk.observed_pvr[i]), 2) if blk.kind[i] == 2 else None
                rows.append(f"{cl_names[i]}\t{radius}\t{pvr}\t{kinds[i]}\t{bp[i]}\t{sizes[i]}\t{names[blk.medoid[i]]}")
            meta.write("\n".join(rows))
            meta.write("\n")
            n_clusters += k
            n_contigs += int(sizes.sum())
    return n_clusters, n_contigs
