"""TEST INFRASTRUCTURE -- C1 trajectory fixture from the UNMODIFIED reference (BASELINE.json configs[0]).

    VAMB_REFERENCE_ROOT=<checkout of the reference> python -m oracle.make_golden_c1 SEED
    python -m oracle.make_golden_c1 merge     (combine the per-seed files into tests/golden/c1_trajectory.npz)

Runs the live reference -- ``vamb.encode.make_dataloader`` -> ``VAE(nsamples=4, seed=SEED).trainmodel(nepochs=300,
batchsteps=[25, 75, 150, 225])`` (the `bin default` schedule, vamb/__main__.py:2363-2512) -> ``encode`` ->
``vamb.cluster.ClusterGenerator(latent, lengths, windowsize=300, minsuccesses=15)`` to exhaustion -- on the planted
10,000 x 4 dataset ``oracle.synth.make_contigs(10000, 4, seed=0)`` and records, per model seed:
  * the per-epoch training loss and its CE / AB / SSE / KLD parts (parsed from the reference's own log lines,
    vamb/encode.py:427-437),
  * the number of clusters, their size histogram, and the adjusted Rand index of the clustering against the planted
    genomes (contigs weighted equally).
The GPU path draws its noise from Philox streams, not from torch's CPU generator, so trajectory parity is
STATISTICAL: tests/test_trajectory_gpu.py checks the CUDA run against the band spanned by the reference seeds.
"""
from __future__ import annotations

import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
N, S, NEPOCHS, BATCHSTEPS = 10_000, 4, 300, [25, 75, 150, 225]
LINE = re.compile(r"Epoch:\s*(\d+)\s+Loss:\s*(\S+)\s+CE:\s*(\S+)\s+AB:\s*(\S+)\s+SSE:\s*(\S+)\s+KLD:\s*(\S+)\s+Batchsize:\s*(\d+)")


def adjusted_rand(labels_a: np.ndarray, labels_b: np.ndarray) -> float:
    """Hubert & Arabie ARI from the contingency table (no sklearn needed on the GPU machine)."""
    _, ia = np.unique(labels_a, return_inverse=True)
    _, ib = np.unique(labels_b, return_inverse=True)
    table = np.zeros((ia.max() + 1, ib.max() + 1), dtype=np.int64)
    np.add.at(table, (ia, ib), 1)
    comb = lambda x: x * (x - 1) // 2
    sum_ij = comb(table).sum()
    sum_a, sum_b = comb(table.sum(1)).sum(), comb(table.sum(0)).sum()
    total = comb(np.int64(len(labels_a)))
    expected = sum_a * sum_b / total
    max_index = 0.5 * (sum_a + sum_b)
    return float((sum_ij - expected) / (max_index - expected))


def labels_of(clusters, n):
    lab = np.full(n, -1, dtype=np.int64)
    for k, c in enumerate(clusters):
        lab[np.asarray(list(c.members), dtype=np.int64)] = k
    assert (lab >= 0).all()
    return lab


def run(seed: int):
    import torch
    from loguru import logger

    from oracle import ref_loader, synth

    torch.set_num_threads(int(os.environ.get("C1_THREADS", "2")))
    ref = ref_loader.load()
    logger.enable("vamb")
    rows = []
    sink = logger.add(lambda m: rows.append(LINE.search(str(m))), level="INFO")
    ab, tnf, lens, genome = synth.make_contigs(N, S, seed=0, return_genome=True)
    dl = ref.encode.make_dataloader(ab.copy(), tnf.copy(), lens, batchsize=256)
    vae = ref.encode.VAE(S, seed=seed)
    vae.trainmodel(dl, nepochs=NEPOCHS, batchsteps=BATCHSTEPS)
    logger.remove(sink)
    traj = np.array([[float(m.group(i)) for i in range(2, 7)] for m in rows if m], dtype=np.float64)
    assert traj.shape == (NEPOCHS, 5), traj.shape
    latent = vae.encode(dl)
    clusters = list(ref.cluster.ClusterGenerator(latent.copy(), lens, windowsize=300, minsuccesses=15, rng_seed=seed))
    sizes = np.array(sorted((len(c.members) for c in clusters), reverse=True), dtype=np.int64)
    ari = adjusted_rand(labels_of(clusters, N), genome)
    out = os.path.join(GOLDEN, f"_c1_seed{seed}.npz")
    np.savez_compressed(out, traj=traj, n_clusters=len(clusters), sizes=sizes, ari=ari, seed=seed,
                        latent_norm=float(np.linalg.norm(latent) / np.sqrt(N)))
    print(f"seed {seed}: final loss {traj[-1, 0]:.5f}, {len(clusters)} clusters, ARI {ari:.4f} -> {out}")


def merge():
    files = sorted(f for f in os.listdir(GOLDEN) if f.startswith("_c1_seed"))
    parts = [np.load(os.path.join(GOLDEN, f)) for f in files]
    np.savez_compressed(
        os.path.join(GOLDEN, "c1_trajectory.npz"),
        traj=np.stack([p["traj"] for p in parts]),  # [seeds, 300 epochs, (loss, CE, AB, SSE, KLD)]
        n_clusters=np.array([int(p["n_clusters"]) for p in parts]),
        ari=np.array([float(p["ari"]) for p in parts]),
        seeds=np.array([int(p["seed"]) for p in parts]),
        latent_norm=np.array([float(p["latent_norm"]) for p in parts]),
        top_sizes=np.stack([np.pad(p["sizes"][:50], (0, max(0, 50 - len(p["sizes"])))) for p in parts]),
        params=np.array([N, S, NEPOCHS] + BATCHSTEPS),
    )
    for f in files:
        os.remove(os.path.join(GOLDEN, f))
    print("merged", files)


if __name__ == "__main__":
    merge() if sys.argv[1] == "merge" else run(int(sys.argv[1]))
