"""Host cost per cluster of writing the two TSV files (SURVEY 8f-1), CPU only: the reference's per-cluster / per-member
Python (vamb/__main__.py:1310-1377, restated in tests/test_cluster_writer_cpu.py) against the block-wise writer
`vamb_b200.cluster.write_clusters_tsv`, on clusters shaped like the C2 job's (1M contigs in ~27k clusters).
    python tools/writer_speed.py"""
import os, sys, tempfile, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import vamb_b200.cluster as vc
from tests.test_cluster_writer_cpu import FakeGenerator, reference_style

n, n_clusters = int(os.environ.get("N", 1_000_000)), int(os.environ.get("CLUSTERS", 27_000))
rng = np.random.default_rng(0)
names = [f"S{1 + i % 50}C{i}" for i in range(n)]
lens = rng.integers(2000, 90000, n)
cuts = np.sort(rng.choice(np.arange(1, n), n_clusters - 1, replace=False))
perm = rng.permutation(n)
clusters = []
for a, b in zip(np.r_[0, cuts], np.r_[cuts, n]):
    mem = np.sort(perm[a:b]).astype(np.int64)
    clusters.append(vc.Cluster(int(mem[0]), 0, mem, 0.1, 0.3 if len(mem) > 1 else None, 0.07 if len(mem) > 1 else None, 0, 0))
t0 = time.perf_counter()
u, m = reference_style(clusters, names, lens, "b")
t_ref = time.perf_counter() - t0
with tempfile.TemporaryDirectory() as d:
    base = os.path.join(d, "vae")
    t0 = time.perf_counter()
    got = vc.write_clusters_tsv(FakeGenerator(clusters), names, lens, base, bin_prefix="b", block=4096)
    t_blk = time.perf_counter() - t0
    same = open(base + "_unsplit.tsv").read() == u and open(base + "_metadata.tsv").read() == m
print(f"{n} contigs in {n_clusters} clusters; identical files: {same}")
print(f"reference-style per-cluster loop : {t_ref:.2f} s = {1e6 * t_ref / n_clusters:.1f} us per cluster ({1e9 * t_ref / n:.0f} ns per contig)")
print(f"block-wise writer (4096 / block) : {t_blk:.2f} s = {1e6 * t_blk / n_clusters:.1f} us per cluster ({1e9 * t_blk / n:.0f} ns per contig)"
      "   [includes packing Cluster objects into blocks: the native driver hands over arrays]")
