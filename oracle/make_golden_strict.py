"""TEST INFRASTRUCTURE -- strict-RNG trajectory fixture from the UNMODIFIED reference.

    VAMB_REFERENCE_ROOT=<checkout of the reference> python -m oracle.make_golden_strict

The live reference trains ``VAE(nsamples=4, seed=0)`` (default 512-512-32 network, dropout 0.2) on the planted
10,000 x 4 dataset ``oracle.synth.make_contigs(10000, 4, seed=0)`` for 6 epochs with batch 256 doubling at epochs 2
and 4, then encodes.  Stored in tests/golden/strict_rng_c1.npz: the per-epoch losses as logged (vamb/encode.py:427-437)
and the first 512 latent rows.  tests/test_trajectory_gpu.py runs the CUDA path in its strict-RNG parity mode
(``VAE.strict_rng = True``: the reference's batch order, dropout masks and noise, drawn from torch's global CPU generator)
and must follow this trajectory to fp32 rounding.
"""
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
N, S, NEPOCHS, BATCHSTEPS, SEED = 10_000, 4, 6, [2, 4], 0
LINE = re.compile(r"Epoch:\s*(\d+)\s+Loss:\s*(\S+)\s+CE:\s*(\S+)\s+AB:\s*(\S+)\s+SSE:\s*(\S+)\s+KLD:\s*(\S+)")


def main():
    import torch
    from loguru import logger

    from oracle import ref_loader, synth

    torch.set_num_threads(4)
    ref = ref_loader.load()
    logger.enable("vamb")
    rows = []
    sink = logger.add(lambda m: rows.append(LINE.search(str(m))), level="INFO")
    ab, tnf, lens = synth.make_contigs(N, S, seed=0)
    dl = ref.encode.make_dataloader(ab.copy(), tnf.copy(), lens, batchsize=256)
    vae = ref.encode.VAE(S, seed=SEED)
    vae.trainmodel(dl, nepochs=NEPOCHS, batchsteps=BATCHSTEPS)
    logger.remove(sink)
    traj = np.array([[float(m.group(i)) for i in range(2, 7)] for m in rows if m])
    assert traj.shape == (NEPOCHS, 5)
    latent = vae.encode(dl)
    out = os.path.join(ROOT, "tests", "golden", "strict_rng_c1.npz")
    np.savez_compressed(out, traj=traj, latent_head=latent[:512], params=np.array([N, S, NEPOCHS, SEED] + BATCHSTEPS),
                        mu_weight_norm=float(vae.state_dict()["mu.weight"].norm()))
    print("losses", traj[:, 0], "->", out)


if __name__ == "__main__":
    main()
