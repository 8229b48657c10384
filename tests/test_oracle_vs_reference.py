"""CPU suite: the torch-fp32 VAE oracle is PINNED -- it reproduces the reference-made golden fixtures bit for bit
(tests/golden/vae_*.npz, written by oracle/make_golden_vae.py from the unmodified reference, and
tests/golden/reference_live.npz, written by oracle/make_golden_live.py).  Also pins oracle/normalize.py."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_live as live
from oracle import vae_oracle as vo
from oracle.make_golden_vae import VAE_CASES, vae_inputs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def live_golden():
    return np.load(os.path.join(GOLDEN, "reference_live.npz"))


def unpack_keep(packed, batch, n):
    return torch.from_numpy(np.unpackbits(packed)[: batch * n].reshape(batch, n).astype(np.float32))


@pytest.mark.parametrize("case", VAE_CASES, ids=[c[0] for c in VAE_CASES])
def test_vae_oracle_reproduces_reference_goldens_bitwise(case):
    """Same batches, same recorded noise -> the reference's losses, d, parameters and latent, exactly."""
    from oracle import normalize as onorm

    name, S, nh, nl, dp, n, batch, nsteps, seed = case
    g = np.load(os.path.join(GOLDEN, f"vae_{name}.npz"))
    rpkm, tnfs, lens = vae_inputs(S, n, seed)
    d, t, a, w = (torch.from_numpy(x) for x in onorm.normalize(rpkm, tnfs, lens))
    o = vo.OracleVAE(S, nhiddens=nh, nlatent=nl, dropout=dp, seed=seed)
    hidden = o.nhiddens + o.nhiddens[::-1]
    for step in range(nsteps):
        idx = torch.from_numpy(g["batch_idx"][step])
        keeps = None
        if o.dropout > 0:
            keeps = [unpack_keep(g[f"keep{li}"][step], batch, hidden[li]) for li in range(len(hidden))]
        lo, _, _ = o.train_step(d[idx], t[idx], a[idx], w[idx], eps=torch.from_numpy(g["eps"][step]), keeps=keeps)
        assert lo == list(g["losses"][step]), (step, lo, g["losses"][step])
        assert o.d == float(g["d"][step])
    L = len(o.nhiddens)
    assert np.array_equal(o.state["mu.weight"].numpy(), g["mu_weight"])
    assert np.array_equal(o.state["outputlayer.bias"].numpy(), g["out_bias"])
    assert np.array_equal(o.state["encoderlayers.0.weight"].numpy()[:8], g["enc0_weight_head"])
    assert np.array_equal(o.state["encodernorms.0.running_mean"].numpy(), g["bn0_running_mean"])
    assert np.array_equal(o.state["encodernorms.0.running_var"].numpy(), g["bn0_running_var"])
    assert np.array_equal(o.state[f"decodernorms.{L - 1}.weight"].numpy(), g["bn_last_weight"])
    latent, _ = o.encode(d, t, a, batch=batch)
    assert np.array_equal(latent, g["latent"])


def test_normalize_restatement_matches_the_product_dataloader():
    """oracle/normalize.py (used by the reference arm of bench.py) == vamb_b200.encode.make_dataloader tensors."""
    pytest.importorskip("vamb_b200._lib")  # needs the built extension to import the package (no device needed)
    import vamb_b200.encode as ve
    from oracle import normalize as onorm
    from oracle import synth

    ab, tnf, lens = synth.make_contigs(3000, 5, seed=4)
    ab[7] = 0.0  # an all-zero abundance row takes the 1/S branch (vamb/encode.py:108-113)
    want = ve.make_dataloader(ab.copy(), tnf.copy(), lens).dataset.tensors
    got = onorm.normalize(ab, tnf, lens)
    for x, y in zip(got, want):
        assert np.array_equal(x, y.numpy())


def test_normalize_restatement_matches_the_live_reference():
    """The reference's ``make_dataloader`` tensors, recorded as a SHA-256 per tensor and a sample of rows."""
    from oracle import normalize as onorm
    from oracle import synth

    g = live_golden()
    ab, tnf, lens = synth.make_contigs(2000, 3, seed=5)
    rows = live.norm_sample_rows(len(lens))
    for name, x in zip("dtaw", onorm.normalize(ab, tnf, lens)):
        assert np.array_equal(x[rows], g[f"norm_{name}_rows"]), name
        assert hashlib.sha256(np.ascontiguousarray(x).tobytes()).hexdigest() == str(g[f"norm_{name}_sha256"]), name


def test_vae_oracle_equals_live_reference_over_training_steps():
    """Under the same ``torch.manual_seed`` stream the oracle and the unmodified reference stay bit-identical
    (losses, every parameter and buffer, encode) over 6 optimiser steps (the reference's run recorded by
    oracle/make_golden_live.py)."""
    from oracle import normalize as onorm

    g = live_golden()
    p = live.TRAIN
    S, n, batch, seed = p["S"], p["n"], p["batch"], p["seed"]
    rpkm, tnfs, lens = vae_inputs(S, n, seed)
    d, t, a, w = (torch.from_numpy(x) for x in onorm.normalize(rpkm, tnfs, lens))
    threads = torch.get_num_threads()
    torch.set_num_threads(live.THREADS)  # torch's CPU reductions split the work by thread count
    try:
        o = vo.OracleVAE(S, nhiddens=p["nhiddens"], nlatent=p["nlatent"], seed=seed)
        rng = np.random.default_rng(seed)
        for step in range(p["steps"]):
            idx = torch.from_numpy(rng.choice(n, size=batch, replace=False).astype(np.int64))
            torch.manual_seed(2000 + step)
            lo, _, _ = o.train_step(d[idx], t[idx], a[idx], w[idx])
            assert lo == list(g["train_losses"][step]), step
        latent = o.encode(d, t, a, batch=batch)[0]
    finally:
        torch.set_num_threads(threads)
    keys = [str(k) for k in g["train_state_keys"]]
    assert keys == list(o.state)
    for i, k in enumerate(keys):
        assert live.digest(o.state[k].numpy()) == str(g[f"train_state_{i}_sha256"]), k
    assert np.array_equal(latent[:16], g["train_latent_head"])
    assert live.digest(latent) == str(g["train_latent_sha256"])


def test_strict_rng_emulation_follows_the_live_reference_trainmodel():
    """``vamb_b200.encode.reference_epoch_noise`` (the strict-RNG parity mode of the CUDA path) consumes torch's global
    generator exactly like the reference's DataLoader + forward pass: driving the (bit-exact) oracle with it reproduces
    the per-epoch losses that the unmodified ``VAE.trainmodel`` logs, including a batch-size doubling."""
    pytest.importorskip("vamb_b200._lib")
    import vamb_b200.encode as ve
    from oracle import normalize as onorm
    from oracle import synth

    p = live.STRICT
    S, n, seed, nepochs, bsteps = p["S"], p["n"], p["seed"], p["nepochs"], p["bsteps"]
    ab, tnf, lens = synth.make_contigs(n, S, seed=p["data_seed"])
    want = [float(x) for x in live_golden()["strict_epoch_losses"]]
    assert len(want) == nepochs

    d, t, a, w = (torch.from_numpy(x) for x in onorm.normalize(ab, tnf, lens))
    o = vo.OracleVAE(S, nhiddens=p["nhiddens"], nlatent=p["nlatent"], seed=seed)  # torch.manual_seed(seed) + the reference's init draws
    batch, got = 128, []
    for epoch in range(nepochs):
        if epoch in bsteps:
            batch *= 2
        tot, k = 0.0, 0
        for idx, eps, keeps in ve.reference_epoch_noise(n, batch, n > batch, o.nhiddens, o.nlatent, o.dropout):
            lo, _, _ = o.train_step(d[idx], t[idx], a[idx], w[idx], eps=eps, keeps=keeps)
            tot += lo[0]
            k += 1
        got.append(tot / k)
    assert [f"{x:.5e}" for x in got] == [f"{x:.5e}" for x in want], (got, want)
