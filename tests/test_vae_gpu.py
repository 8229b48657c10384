"""GPU suite: the CUDA VAE path (through the C ABI) against the reference-made golden fixtures
and the torch-fp32 oracle.  Floating point: per-step losses within 2e-5 relative, gradients /
parameters within 2e-5 of the tensor norm (fp32 accumulation-order noise), eval-mode mu within
1e-4 absolute before bit masking (BASELINE.json north_star tolerance)."""
import io
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
from oracle.make_golden_vae import VAE_CASES, vae_inputs  # noqa: E402  (fixture definitions only)


def rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def unpack_keep(packed, batch, n):
    return np.unpackbits(packed)[: batch * n].reshape(batch, n)


def set_path(vae, tc):
    """Force the wgmma (3xTF32) GEMM path for every batch size (True: operands staged by the producing
    kernels, "prep": by separate prep launches), or the fp32 CUDA-core path (False).  The test ids keep the
    name "tcgen05" for the tensor-core path, so that results stay comparable across versions of the project."""
    vae._net.tc_min_batch = 1 if tc else 0
    vae._net.staging = 1 if tc == "prep" else 0
    vae._net.use_tma = 1 if tc == "tma" else 0  # weight operand through TMA (cp.async.bulk.tensor) vs the cp.async ring
    vae._net.wgrad_flush = 1 if tc == "flush" else 0  # wgrad accumulation chain cut every 128 batch rows
    return vae


@pytest.mark.parametrize("tc", [False, True, "prep", "tma"], ids=["ffma", "tcgen05", "tcgen05-prep", "tcgen05-tma"])
@pytest.mark.parametrize("case", VAE_CASES, ids=[c[0] for c in VAE_CASES])
def test_train_steps_and_encode_match_reference_golden(case, tc):
    import vamb_b200.encode as ve
    from oracle import vae_oracle as vo

    name, S, nh, nl, dp, n, batch, nsteps, seed = case
    g = np.load(os.path.join(GOLDEN, f"vae_{name}.npz"))
    rpkm, tnfs, lens = vae_inputs(S, n, seed)
    dl = ve.make_dataloader(rpkm.copy(), tnfs.copy(), lens, batchsize=batch)
    vae = set_path(ve.VAE(S, nhiddens=nh, nlatent=nl, dropout=dp, seed=seed), tc)
    # same seed -> the reference's initial weights, bit for bit
    init = vo.init_state(S, vae.nhiddens, nl, seed)
    sd = vae.state_dict()
    assert list(sd.keys()) == list(init.keys())
    for k in init:
        assert torch.equal(sd[k].cpu(), init[k]), k
    vae._reset_optimizer()
    hidden = vae.nhiddens + vae.nhiddens[::-1]
    for step in range(nsteps):
        keeps = None
        if vae.dropout > 0:
            keeps = [unpack_keep(g[f"keep{li}"][step], batch, hidden[li]) for li in range(len(hidden))]
        losses = vae._step_injected(dl.dataset.tensors, g["batch_idx"][step], g["eps"][step], keeps)
        assert np.allclose(losses, g["losses"][step], rtol=2e-5, atol=1e-7), (step, losses, g["losses"][step])
        assert abs(vae.dadapt_d - g["d"][step]) <= 2e-4 * g["d"][step], (step, vae.dadapt_d, g["d"][step])
    sd = vae.state_dict()
    L = len(vae.nhiddens)
    assert rel(sd["mu.weight"].cpu().numpy(), g["mu_weight"]) < 2e-5
    assert rel(sd["outputlayer.bias"].cpu().numpy(), g["out_bias"]) < 2e-5
    assert rel(sd["encoderlayers.0.weight"].cpu().numpy()[:8], g["enc0_weight_head"]) < 2e-5
    assert rel(sd["encodernorms.0.running_mean"].cpu().numpy(), g["bn0_running_mean"]) < 2e-5
    assert rel(sd["encodernorms.0.running_var"].cpu().numpy(), g["bn0_running_var"]) < 2e-5
    assert rel(sd[f"decodernorms.{L - 1}.weight"].cpu().numpy(), g["bn_last_weight"]) < 2e-5
    assert int(sd["encodernorms.0.num_batches_tracked"]) == nsteps
    # encode: eval mode, low 12 mantissa bits cleared
    lat = vae.encode(dl)
    assert lat.shape == (n, nl) and lat.dtype == np.float32 and lat.flags.owndata
    assert np.all(lat.view(np.uint32) & 0xFFF == 0)
    gl = g["latent"]
    assert np.all(np.abs(lat - gl) <= 1e-4 + np.abs(gl) * 2.0 ** -11)


@pytest.mark.parametrize("tc,B,S", [(False, 256, 50), (True, 256, 50), (True, 1024, 50), (True, 4096, 50),
                                    ("prep", 256, 50), ("prep", 4096, 50), (True, 1000, 50), (True, 256, 80),
                                    (True, 8192, 50), ("tma", 256, 50), ("tma", 1000, 50), ("tma", 4096, 50),
                                    ("flush", 256, 50), ("flush", 1000, 50), ("flush", 4096, 50), ("flush", 8192, 50),
                                    (True, 512, 100), ("tma", 2048, 100)],
                         ids=["ffma-256", "tcgen05-256", "tcgen05-1024-split2", "tcgen05-4096-split8", "tcgen05-prep-256",
                              "tcgen05-prep-4096", "tcgen05-1000-ragged", "tcgen05-256-wide-input",
                              "tcgen05-8192-grid-fallback", "tcgen05-tma-256", "tcgen05-tma-1000-ragged", "tcgen05-tma-4096",
                              "tcgen05-flush-256", "tcgen05-flush-1000-ragged", "tcgen05-flush-4096", "tcgen05-flush-8192",
                              "tcgen05-512-C3-shape-S100", "tcgen05-tma-2048-C3-shape-S100"])
def test_gradients_match_oracle_default_network(tc, B, S):
    """One fwd+bwd on the bin-default network (512-512-32): every gradient tensor.  S = 100 is BASELINE's C3 shape
    (D_in = 204); S = 80 / 100 make the
    reconstruction wider than the loss kernel stages itself (a prep launch takes over for that layer);
    B = 8192 exceeds the SM count with its forward grid, so operand staging falls back to prep launches."""
    import vamb_b200.encode as ve
    from oracle import vae_oracle as vo

    n = max(5000, B + 1000)
    rpkm, tnfs, lens = vae_inputs(S, n, 7)
    dl = ve.make_dataloader(rpkm.copy(), tnfs.copy(), lens, batchsize=B)
    d, t, a, w = dl.dataset.tensors
    vae = set_path(ve.VAE(S, seed=2), tc)
    o = vo.OracleVAE(S, seed=2)
    idx = torch.from_numpy(np.random.default_rng(0).choice(n, B, replace=False))
    torch.manual_seed(5)
    lo, grads, eps, keeps = o.grads(d[idx], t[idx], a[idx], w[idx])
    losses = vae._step_injected(dl.dataset.tensors, idx.numpy(), eps.numpy(), [k.numpy() for k in keeps], optimize=False)
    assert np.allclose(losses, lo, rtol=2e-5, atol=1e-7)
    got = vae._grad_dict()
    # Against an fp64 evaluation of the same step (tools/grad_error_fp64.py) every path -- the fp32 CPU oracle, the CUDA
    # 3xTF32 path with or without the wgrad flush, the CUDA fp32 path -- is fp32-grade at every batch size.  Two of the
    # cases are ill-conditioned for ANY fp32 pipeline: at B = 8192 the fp32 CPU oracle itself is far from fp64, and at
    # S = 100 / B = 2048 the BatchNorm backward of the first decoder block cancels heavily (torch's CPU kernel carries
    # the statistics in double) -- they keep a loose bound, everything else is held to fp32 grade.
    tol = 3e-5
    if B > 4096:
        tol = 2e-2
    elif S == 100 and B >= 2048:
        tol = 5e-3
    for k, gref in grads.items():
        assert rel(got[k].cpu().numpy(), gref.numpy()) < tol, k


@pytest.mark.parametrize("tc", [False, True, "prep", "tma"], ids=["ffma", "tcgen05", "tcgen05-prep", "tcgen05-tma"])
def test_odd_batch_and_many_steps_match_oracle(tc):
    """B not a multiple of the tile size, 12 steps: parameters track the oracle."""
    import vamb_b200.encode as ve
    from oracle import vae_oracle as vo

    S, n, B = 4, 500, 77
    rpkm, tnfs, lens = vae_inputs(S, n, 9)
    dl = ve.make_dataloader(rpkm.copy(), tnfs.copy(), lens, batchsize=B)
    d, t, a, w = dl.dataset.tensors
    vae = set_path(ve.VAE(S, nhiddens=[96, 33], nlatent=7, seed=1), tc)
    vae._reset_optimizer()
    o = vo.OracleVAE(S, nhiddens=[96, 33], nlatent=7, seed=1)
    rng = np.random.default_rng(1)
    for step in range(12):
        idx = torch.from_numpy(rng.choice(n, B, replace=False))
        torch.manual_seed(50 + step)
        lo, eps, keeps = o.train_step(d[idx], t[idx], a[idx], w[idx])
        losses = vae._step_injected(dl.dataset.tensors, idx.numpy(), eps.numpy(), [k.numpy() for k in keeps])
        assert np.allclose(losses, lo, rtol=1e-4, atol=1e-6), (step, losses, lo)
    sd = vae.state_dict()
    for k, v in o.state.items():
        if k.endswith("num_batches_tracked"):
            assert int(sd[k]) == int(v)
        else:
            assert rel(sd[k].cpu().numpy(), v.numpy()) < 2e-4, k
    assert abs(vae.dadapt_d - o.d) <= 1e-3 * o.d
    lat_raw = vae._encode_device(dl.dataset.tensors, mask_bits=0)
    _, oraw = o.encode(d, t, a)
    assert np.abs(lat_raw - oraw).max() < 1e-4


def test_forward_api_eval_and_train():
    import vamb_b200.encode as ve
    from oracle import vae_oracle as vo

    S, n = 6, 130
    rpkm, tnfs, lens = vae_inputs(S, n, 11)
    dl = ve.make_dataloader(rpkm.copy(), tnfs.copy(), lens, batchsize=64)
    d, t, a, w = dl.dataset.tensors
    vae = ve.VAE(S, nhiddens=[64, 64], nlatent=8, seed=3)
    o = vo.OracleVAE(S, nhiddens=[64, 64], nlatent=8, seed=3)
    vae.eval()
    do, to, ao, mu = vae(d, t, a)
    rd, rt, ra, rmu, _, _ = vo.forward(o.state, d, t, a, S, o.dropout, False, eps=torch.zeros(n, 8))
    assert mu.shape == (n, 8) and do.shape == (n, S) and to.shape == (n, 103) and ao.shape == (n, 1)
    assert np.abs(mu.numpy() - rmu.numpy()).max() < 1e-5
    assert np.allclose(do.sum(1).numpy(), 1.0, atol=1e-5)
    loss = vae.calc_loss(d, do, t, to, a, ao, mu, w)
    assert all(np.isfinite(float(x)) for x in loss)


# ---- the reference's TestVAE (test/test_encode.py:122-185) on the CUDA path ----
class TestReferenceVAESuite:
    tnfs = np.random.RandomState(1).random((128, 103)).astype(np.float32)
    rpkm = np.random.RandomState(2).random((128, 14)).astype(np.float32)
    lens = np.random.RandomState(3).randint(2000, 5000, size=128)

    def test_loss_falls(self):
        import vamb_b200.encode as ve

        vae = ve.VAE(self.rpkm.shape[1])
        rpkm_copy, tnfs_copy = self.rpkm.copy(), self.tnfs.copy()
        dl = ve.make_dataloader(rpkm_copy, tnfs_copy, self.lens, batchsize=16, destroy=True)
        di, ti, ai, we = next(iter(dl))
        vae.train()
        do, to, ao, mu = vae(di, ti, ai)
        before = vae.calc_loss(di, do, ti, to, ai, ao, mu, we)[0]
        vae.trainmodel(dl, nepochs=3, batchsteps=[1, 2])
        vae.train()
        do, to, ao, mu = vae(di, ti, ai)
        after = vae.calc_loss(di, do, ti, to, ai, ao, mu, we)[0]
        assert float(after) < float(before)

    def test_save_load_and_encoding(self):
        import vamb_b200.encode as ve

        vae = ve.VAE(self.rpkm.shape[1])
        dl = ve.make_dataloader(self.rpkm.copy(), self.tnfs.copy(), self.lens, batchsize=16)
        vae.trainmodel(dl, nepochs=2, batchsteps=None)
        enc1 = vae.encode(dl)
        assert enc1.dtype == np.float32 and enc1.shape == (len(self.rpkm), vae.nlatent)
        buf = io.BytesIO()
        vae.save(buf)
        buf.seek(0)
        vae2 = ve.VAE.load(buf)
        enc2 = vae2.encode(dl)
        assert np.all(np.abs(enc1 - enc2) < 1e-6)
        # the file is loadable as plain tensors with the reference's key set
        buf.seek(0)
        dct = torch.load(buf, weights_only=True)
        assert set(dct) == {"nsamples", "alpha", "beta", "dropout", "nhiddens", "nlatent", "state"}
        assert "encodernorms.1.num_batches_tracked" in dct["state"]

    def test_trainmodel_arg_errors(self):
        import vamb_b200.encode as ve

        vae = ve.VAE(self.rpkm.shape[1])
        dl = ve.make_dataloader(self.rpkm.copy(), self.tnfs.copy(), self.lens, batchsize=16)
        with pytest.raises(ValueError):
            vae.trainmodel(dl, nepochs=0)
        with pytest.raises(ValueError):
            vae.trainmodel(dl, nepochs=3, batchsteps=[1.5])
        with pytest.raises(ValueError):
            vae.trainmodel(dl, nepochs=3, batchsteps=[3])


def test_graph_replay_training_is_deterministic_and_learns():
    """Enough steps per epoch to go through the CUDA-graph path; same seed -> same bits."""
    import vamb_b200.encode as ve
    from oracle import synth

    ab, tnf, lens = synth.make_contigs(80000, 8, seed=0)
    lats = []
    for _ in range(2):
        dl = ve.make_dataloader(ab.copy(), tnf.copy(), lens, batchsize=256)
        vae = ve.VAE(8, seed=4)
        vae.trainmodel(dl, nepochs=3, batchsteps=[2])
        first = vae._last_epoch_losses
        lats.append(vae.encode(dl))
        assert np.all(np.isfinite(lats[-1]))
    assert np.array_equal(lats[0], lats[1])
    # planted genomes: the loss after 3 epochs is well below the untrained level
    assert first[0] < 0.9


def test_subclass_contract_autograd_route_matches_the_kernels():
    """``_encode`` / ``reparameterize`` / ``_decode`` (the methods VAELabels / VAEConcat build on,
    vamb/semisupervised_encode.py:189,438) are differentiable module code over the SAME arena the kernels train: with
    dropout off and the same noise, ``calc_loss(...)[0].backward()`` through ``forward`` gives the kernels' gradients."""
    import vamb_b200.encode as ve

    S, n, B = 6, 700, 256
    rpkm, tnfs, lens = vae_inputs(S, n, 13)
    dl = ve.make_dataloader(rpkm.copy(), tnfs.copy(), lens, batchsize=B)
    d, t, a, w = dl.dataset.tensors
    vae = ve.VAE(S, nhiddens=[96, 64], nlatent=12, dropout=0.0, seed=5)
    idx = np.random.default_rng(2).choice(n, B, replace=False)
    ti = torch.from_numpy(idx)
    vae.train()
    torch.manual_seed(77)
    do, to, ao, mu = vae(d[ti], t[ti], a[ti])
    assert mu.requires_grad and do.shape == (B, S)
    loss = vae.calc_loss(d[ti], do, t[ti], to, a[ti], ao, mu, w[ti])
    vae.zero_grad()
    loss[0].backward()
    auto = {k: p.grad.detach().clone() for k, p in vae.named_parameters()}
    torch.manual_seed(77)
    eps = torch.randn(B, 12)  # what reparameterize drew
    for bn in list(vae.encodernorms) + list(vae.decodernorms):  # undo the running-stat update of the first pass
        bn.reset_running_stats()
    losses = vae._step_injected(dl.dataset.tensors, idx, eps.numpy(), None, optimize=False)
    assert np.allclose(losses[0], float(loss[0]), rtol=2e-5)
    got = vae._grad_dict()
    for k, g in auto.items():
        assert rel(got[k].cpu().numpy(), g.cpu().numpy()) < 1e-4, k
    # eval mode / no_grad: the fused kernels, graph-less outputs
    vae.eval()
    out = vae(d[:64], t[:64], a[:64])
    assert not out[3].requires_grad
    with torch.no_grad():
        vae.train()
        out = vae(d[:64], t[:64], a[:64])
        assert not out[3].requires_grad
