"""2-GPU NCCL test of the row-sharded data-parallel VAE (skipped on single-GPU machines): replicas stay
bit-identical (same gradients after the all-reduce, same optimiser state), the loss falls, and the
per-shard encode + clustering run independently."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import vamb_b200.cluster as vc
    import vamb_b200.encode as ve
    from oracle import synth

    ab, tnf, lens = synth.make_contigs(40000, 6, seed=10 + rank)  # every rank owns its own shard
    dl = ve.make_dataloader(ab, tnf, lens, batchsize=128)
    vae = ve.VAE(6, seed=3)
    vae.enable_data_parallel()
    vae.trainmodel(dl, nepochs=3, batchsteps=[2])
    first = vae._last_epoch_losses[0]
    sd = {k: v.detach().float().cpu() for k, v in vae.state_dict().items() if "running" not in k and "tracked" not in k}
    lat = vae.encode(dl)
    clusters = 0
    for c in vc.ClusterGenerator(lat, lens, rng_seed=rank):
        clusters += 1
        if clusters >= 50:
            break
    digest = float(sum(v.double().sum() for v in sd.values()))
    flat = torch.cat([v.reshape(-1) for v in sd.values()])
    gathered = [torch.empty_like(flat).cuda() for _ in range(world)]
    dist.all_gather(gathered, flat.cuda())
    same = all(torch.equal(gathered[0], g) for g in gathered)
    q.put((rank, {"loss": first, "digest": digest, "same": bool(same), "finite": bool(np.isfinite(lat).all()),
                  "clusters": clusters, "graphs": bool(vae._use_graphs)}))
    dist.barrier()
    # CUDA graphs that captured NCCL collectives can hang NCCL's communicator teardown; the result is already
    # reported, so leave without running destructors (bench.py does the same)
    os._exit(0)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_data_parallel_replicas_stay_identical():
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert res[0]["same"] and res[1]["same"], "replicas diverged"
    assert res[0]["digest"] == res[1]["digest"]
    for r in (0, 1):
        assert res[r]["finite"] and res[r]["clusters"] > 0
        assert res[r]["loss"] < 1.2
    print("CUDA-graph capture of NCCL steps:", res[0]["graphs"])


def _worker_strong(rank, world, port, q):
    """bench.py's strong-scaling path in miniature: ONE dataset, row-sharded; data-parallel training; per-shard
    encode; all-gather of the latent shards; a single clustering of the gathered latent on rank 0."""
    import torch.distributed as dist
    from torch.utils.data import DataLoader, TensorDataset

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import vamb_b200.cluster as vc
    import vamb_b200.encode as ve
    from oracle import synth
    from vamb_b200 import parallel as par

    n = 30001  # odd on purpose: the shards differ by one row
    ab, tnf, lens = synth.make_contigs(n, 6, seed=3)
    full = ve.make_dataloader(ab, tnf, lens, batchsize=128, destroy=True)  # normalised over ALL contigs
    lo, hi = par.shard_rows(n, rank, world)
    shard = TensorDataset(*(t[lo:hi].clone() for t in full.dataset.tensors))
    dl = DataLoader(shard, batch_size=128, shuffle=True, drop_last=True)
    vae = ve.VAE(6, seed=3)
    vae.enable_data_parallel()
    vae.trainmodel(dl, nepochs=4, batchsteps=[1, 2])  # short epochs: 16- and 4-step graph chunks with NCCL inside
    lat = torch.from_numpy(vae.encode(dl)).cuda()
    allat = par.gather_rows(lat)
    out = {"rows": int(allat.shape[0]), "finite": bool(torch.isfinite(allat).all()), "loss": vae._last_epoch_losses[0],
           "graphs": bool(vae._use_graphs)}
    # every rank holds the same gathered latent, in dataset order
    digest = torch.tensor([float(allat.double().sum())], device="cuda", dtype=torch.float64)
    both = [torch.empty_like(digest) for _ in range(world)]
    dist.all_gather(both, digest)
    out["same_latent"] = bool(all(torch.equal(both[0], b) for b in both))
    out["own_rows_in_place"] = bool(torch.equal(allat[lo:hi], lat))
    if rank == 0:
        clusters = list(vc.ClusterGenerator(allat, lens, rng_seed=0, destroy=True))
        out["clustered"] = sum(len(c.members) for c in clusters)
        out["n_clusters"] = len(clusters)
    q.put((rank, out))
    dist.barrier()
    vae._graphs.clear()
    torch.cuda.synchronize()
    os._exit(0)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_strong_scaling_path_gathers_and_clusters_once():
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_strong, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for r in (0, 1):
        assert res[r]["rows"] == 30001 and res[r]["finite"] and res[r]["same_latent"] and res[r]["own_rows_in_place"]
        assert res[r]["loss"] < 1.2
    assert res[0]["clustered"] == 30001 and res[0]["n_clusters"] > 100
    print("CUDA-graph capture of NCCL steps:", res[0]["graphs"])
