#!/usr/bin/env python
"""bench.py -- contigs/sec of the vamb hot path (VAE train + encode + medoid clustering).

Contract (one JSON line on rank 0):
    python bench.py --gpus N --steps K --warmup W [--impl reference] [--scaling strong|weak] [--dump-outputs DIR]

Workload: BASELINE.json configs[1] -- 1,000,000 planted contigs x (103 TNF + 50 abundance samples), `vamb bin
default` settings (VAE 512-512-32, 300 epochs, batch 256 doubling at epochs 25/75/150/225, then
ClusterGenerator(windowsize=300, minsuccesses=15) run to exhaustion).

The timed region is exactly ONE pass of that workload, cut into K steps: step i trains epochs
[300 i / K, 300 (i + 1) / K) of the fixed schedule; the last step also encodes and clusters.  Every step is
bracketed by CUDA events on the launching stream, the K steps by a barrier + synchronize on both sides.
  value  = contigs / sum of the K step times (max over ranks), normalised dataset already resident in HBM.
  e2e    = the same metric through the public API in one more pass (make_dataloader tensors in pinned HOST
           memory -> VAE.trainmodel -> VAE.encode -> numpy latent -> ClusterGenerator -> numpy members), all
           host<->device copies inside the timed region.
Warm-up passes run the same code path with a shortened schedule (5 epochs covering all five batch sizes,
clustering capped at 300 clusters): they warm clocks, caches, the CUDA-graph captures and NCCL.

N > 1 (torchrun, one rank per GPU):
  --scaling strong (default): the SAME 1M contigs, row-sharded; ONE VAE trained data-parallel (one gradient
      all-reduce per minibatch, global batch = N x B), per-shard encode, all-gather of the latent shards over
      NVLink, ONE clustering of the gathered latent on rank 0 (the clusterer is a latency-bound sequential
      driver: "replicas only", see DESIGN.md section 6).
  --scaling weak: every rank owns its own 1M-contig sample (own genomes); same data-parallel training, encode and
      clustering per shard (Vamb splits bins per sample).

--dump-outputs DIR: after the timed pass, what its last step computed, as DIR/<name>.npy (float32 / float64, < 64 MB):
the latent of a fixed seeded sample of rows (all rows up to LATENT_SAMPLE), those row indices, the cluster ordinal of
every contig (clusters numbered in the order the generator yields them) and the medoid of every cluster.  Rank 0
writes them: with --scaling strong it clusters the gathered latent of all contigs, with --scaling weak its own sample.

--impl reference: the CPU port of the reference path (oracle/) on the host cores, ONE bounded sample of the same
workload (a few optimiser steps per batch size, encode of 50k rows, the first clusters), extrapolated over the
schedule and labelled as such.  It never imports the product package.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

METRIC = "contigs/sec (VAE train + cluster) at N=1M, S=50"
BATCHSTEPS = [25, 75, 150, 225]
LATENT_SAMPLE = 262_144  # latent rows written by --dump-outputs (32 MB at 32 dimensions)


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20, help="timed steps (>= 1): slices of the one timed pass")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--scaling", default="strong", choices=["strong", "weak"])
    ap.add_argument("--contigs", dest="n", type=int, default=1_000_000,
                    help="contigs in total (strong scaling) / per GPU (weak scaling)")
    ap.add_argument("--nsamples", type=int, default=50)
    ap.add_argument("--nepochs", type=int, default=300)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-e2e", action="store_true", help="skip the second (host-buffer) pass")
    ap.add_argument("--cpu-seconds", type=float, default=25.0, help="budget of the cpu_baseline sample")
    ap.add_argument("--time-budget", type=float, default=780.0,
                    help="wall-clock budget (s): optional legs (e2e, cpu_baseline) are skipped, and say so, when the run "
                         "would exceed it")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the latent (seeded row sample) and the clusters of the timed pass as DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    return args


def schedule(n: int, nepochs: int, batch0: int = 256):
    """[(batch, steps per epoch, epochs)] of the bin-default schedule (vamb/encode.py:383-388)."""
    out, b, prev = [], batch0, 0
    steps = [s for s in BATCHSTEPS if s < nepochs]
    for s in steps + [nepochs]:
        if s > prev:
            out.append((b, (n // b) if n > b else 1, s - prev))
        prev = s
        b *= 2
    return out


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""

    FIELDS = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
              "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
              "clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int = 0):
        self.rows, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={self.FIELDS}", "--format=csv,noheader,nounits", "-lms", "500",
                 "-i", str(self.index)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except OSError:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        for r in self.rows:
            try:
                sm.append(float(r[0]))
                mx.append(float(r[1]))
            except (ValueError, IndexError):
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "samples": len(sm), "reasons": sorted(reasons)}


T_START = time.perf_counter()


def elapsed() -> float:
    return time.perf_counter() - T_START


def log(msg: str) -> None:
    """Progress on stderr (stdout carries exactly one JSON line)."""
    print(f"[bench +{elapsed():7.1f}s] {msg}", file=sys.stderr, flush=True)


def make_workload(n, nsamples, seed):
    from oracle import synth  # synthetic planted inputs (NumPy only)

    return synth.make_contigs(n, nsamples, seed=seed)


def workload_name(args) -> str:
    """The same string on both arms, so that the `config` of the two JSON lines can be compared."""
    return (f"{args.n} contigs x (103 TNF + {args.nsamples} abundance), bin default VAE 512-512-32, {args.nepochs} "
            "epochs (batch 256 doubling at 25/75/150/225) + encode + medoid clustering to exhaustion")


def reference_threads() -> int:
    """The reference caps its BLAS/OpenMP threads at min(ncpu, 8) (vamb/__main__.py:27-40, 2221-2228); more threads
    oversubscribe these small kernels."""
    return min(os.cpu_count() or 8, 8)


def datasheet_peaks():
    """(HBM GB/s, tensor TFLOP/s, tensor peak label, HBM peak label): NVIDIA's H100 SXM data sheet (700 W card), dense
    TF32 -- these GEMMs are wgmma .tf32.  A card with a lower power limit (see "clocks") reaches less."""
    return (3350.0, 495.0, "H100 SXM data sheet, dense TF32 (not reached: an upper bound)",
            "H100 SXM data sheet HBM3 (not reached: an upper bound)")


# ---------------------------------------------------------------------------------- the GPU pass
class Ctx:
    """Per-process state of the bench: rank layout, this rank's loader, the lengths of the rows it clusters."""

    def __init__(self, args):
        self.args = args
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.rank = int(os.environ.get("RANK", "0"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        self.strong = args.scaling == "strong"

    def barrier(self):
        torch.cuda.synchronize()
        if self.world > 1:
            import torch.distributed as dist

            dist.barrier()

    def max_over_ranks(self, x: float) -> float:
        if self.world == 1:
            return x
        import torch.distributed as dist

        t = torch.tensor([x], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())


def epoch_slices(nepochs: int, k: int):
    return [(nepochs * i) // k for i in range(k + 1)]


def run_pass(ctx: Ctx, dl, lengths_cluster, nepochs, k_steps, resident: bool, max_clusters=None, batchsteps=None):
    """One pass of the hot path in `k_steps` event-timed steps.  resident=True: the dataset is bound to the device
    before the clock starts, training is driven epoch by epoch and the latent stays in HBM between encode and
    clustering; resident=False: the public API end to end (trainmodel / encode -> numpy / ClusterGenerator(numpy))."""
    import vamb_b200.cluster as vc
    import vamb_b200.encode as ve
    from vamb_b200 import parallel as par

    args = ctx.args
    bs = [b for b in (BATCHSTEPS if batchsteps is None else batchsteps) if b < nepochs]
    vae = ve.VAE(args.nsamples, seed=args.seed)
    if ctx.world > 1:
        vae.enable_data_parallel()  # one model for all shards: one gradient all-reduce per minibatch
    n_local = len(dl.dataset.tensors[0])
    if resident:
        vae._bind_dataset(dl.dataset.tensors)
    ctx.barrier()
    step_ms, phases = [], {"train": 0.0, "encode": 0.0, "cluster": 0.0}
    n_clusters = n_members = probes = evals = 0
    medoids, members = [], []  # kept for --dump-outputs only
    cluster_timing = {}
    latent_dev = None
    t_wall0 = time.perf_counter()
    edges = epoch_slices(nepochs, k_steps)
    loader = dl
    if resident:
        vae._reset_optimizer()  # trainmodel() does this itself (a new DAdaptAdam per call, vamb/encode.py:578)
    for i in range(k_steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        t0 = time.perf_counter()
        if resident:
            for epoch in range(edges[i], edges[i + 1]):
                loader = vae.trainepoch(loader, epoch, None, bs)
        elif i == 0:
            vae.trainmodel(dl, nepochs=nepochs, batchsteps=bs)  # the whole schedule in the public call
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        phases["train"] += t1 - t0
        if i == k_steps - 1:
            if resident:
                vae.eval()
                vae.sync_running_stats()
                latent = torch.empty((n_local, vae.nlatent), dtype=torch.float32, device="cuda")
                ve._lib.check(ve._L.vk_vae_encode(ve._ct.byref(vae._net), 0, n_local, 12, latent.data_ptr(), vae._stream()))
                if ctx.world > 1 and ctx.strong:
                    latent = par.gather_rows(latent)  # NVLink all-gather of the latent shards
                torch.cuda.synchronize()
            else:
                latent = vae.encode(dl)  # numpy, D2H inside
                if ctx.world > 1 and ctx.strong:
                    latent = par.gather_rows(torch.from_numpy(latent).cuda()).cpu().numpy()
            t2 = time.perf_counter()
            phases["encode"] += t2 - t1
            if ctx.world == 1 or not ctx.strong or ctx.rank == 0:
                if resident:
                    latent_dev = latent.clone()  # for the probe roofline afterwards (destroy=True normalises in place)
                gen = vc.ClusterGenerator(latent, lengths_cluster, windowsize=300, minsuccesses=15, destroy=True,
                                          rng_seed=args.seed)
                for c in gen:
                    n_clusters += 1
                    n_members += len(c.members)
                    if args.dump_outputs and ctx.rank == 0:
                        medoids.append(int(c.medoid))
                        members.append(np.asarray(c.members))
                    if max_clusters and n_clusters >= max_clusters:
                        break
                probes, evals = gen._n_probes, gen._n_evals
                cluster_timing = gen._timing()
                torch.cuda.synchronize()
            phases["cluster"] += time.perf_counter() - t2
        e1.record()
        torch.cuda.synchronize()
        step_ms.append(e0.elapsed_time(e1))
    ctx.barrier()
    t_wall = time.perf_counter() - t_wall0
    sched = schedule(n_local, nepochs)
    nl, tcm = vae._net.n_layers, vae._net.tc_min_batch

    def per_step(b):  # launches of one optimiser step (vk_vae.cu: grad_step_impl + launch_dadapt)
        base = 2 * nl + 3
        if not (tcm and b >= tcm):
            return base
        # tensor-core path: the first layer's gather draws the batch (no batch_rows launch), + weight staging + loss fold
        return base - 1 + (3 if vae._net.staging == 0 else 2 * nl + 1)

    launches = (sum(s * e * per_step(b) for b, s, e in sched)
                + ((n_local + vae._net.bmax - 1) // vae._net.bmax) * (nl + 2)
                + probes + evals + 2 * n_clusters + 1)  # probe, evaluation, (rank + selection) per cluster
    return {"step_ms": step_ms, "t_event": sum(step_ms) / 1e3, "t_wall": t_wall, "phases": phases,
            "n_clusters": n_clusters, "n_clustered": n_members, "probes": probes, "evals": evals,
            "train_steps": sum(s * e for _, s, e in sched), "launches": launches,
            "final_loss": vae._last_epoch_losses[0], "vae": vae, "latent_dev": latent_dev,
            "cluster_timing": cluster_timing, "medoids": medoids, "members": members}


def dump_outputs(outdir: str, res, n_rows: int, seed: int) -> None:
    """What the timed pass computed in its last step (see --dump-outputs), as .npy files under `outdir`."""
    os.makedirs(outdir, exist_ok=True)
    rows = np.arange(n_rows)
    if n_rows > LATENT_SAMPLE:
        rows = np.sort(np.random.default_rng(seed).choice(n_rows, LATENT_SAMPLE, replace=False))
    latent = res["latent_dev"][torch.from_numpy(rows).cuda()].cpu().numpy().astype(np.float32)
    cluster_of = np.full(n_rows, -1.0, dtype=np.float64)
    for k, m in enumerate(res["members"]):
        cluster_of[m] = k
    np.save(os.path.join(outdir, "latent_sample.npy"), latent)
    np.save(os.path.join(outdir, "latent_sample_rows.npy"), rows.astype(np.float64))
    np.save(os.path.join(outdir, "cluster_of_contig.npy"), cluster_of)
    np.save(os.path.join(outdir, "cluster_medoid.npy"), np.asarray(res["medoids"], dtype=np.float64))


def vae_roofline(vae, n, nepochs):
    """Per-launch device times of one training step at every batch size of the schedule (CUDA events on
    the launching stream) -> time share per kernel and achieved FLOP/s of the dominant one."""
    sched = schedule(n, nepochs)
    net = vae._net
    nl = net.n_layers
    dims = [(net.layers[j].k_in, net.layers[j].n_out, net.layers[j].in_kind) for j in range(nl)]
    tot = {}
    best = None
    for batch, spe, epochs in sched:
        batch = min(batch, n)
        reps = [vae._profile_step(batch) for _ in range(8)][3:]
        avg_bwd = np.mean([r["bwd"] for r in reps], axis=0)  # launch order: last layer first
        avg_fwd = np.mean([r["fwd"] for r in reps], axis=0)
        other = float(np.mean([r["batch_rows"] + r["loss"] + r["dadapt"] + r["prep"] for r in reps]))
        nsteps = spe * epochs
        tot["fwd_layer_kernel"] = tot.get("fwd_layer_kernel", 0.0) + nsteps * float(avg_fwd.sum())
        tot["bwd_layer_kernel"] = tot.get("bwd_layer_kernel", 0.0) + nsteps * float(avg_bwd.sum())
        tot["other"] = tot.get("other", 0.0) + nsteps * other
        for i, ms in enumerate(avg_bwd):
            j = nl - 1 - i
            k, nn, in_kind = dims[j]
            flops = 2.0 * batch * nn * (k + 1) + (2.0 * batch * nn * k if in_kind != 0 else 0.0)
            kname = "bwd_layer_tc_kernel" if 0 < net.tc_min_batch <= batch else "bwd_layer_kernel"
            cand = {"kernel": f"{kname}[layer {j}: {k}->{nn}, B={batch}]", "ms": float(ms),
                    "tflops": flops / (ms * 1e-3) / 1e12, "weight_ms": nsteps * float(ms)}
            if best is None or cand["weight_ms"] > best["weight_ms"]:
                best = cand
    total = sum(tot.values())
    share = {k: v / total for k, v in tot.items()}
    return best, share


def probe_roofline(latent_dev, lengths):
    """Cosine-distance probe at full N on the produced latent: algorithmic 133 B/contig / event time."""
    import vamb_b200.cluster as vc
    from vamb_b200 import _lib

    gen = vc.ClusterGenerator(latent_dev, lengths, rng_seed=0, _driver="python")
    n = gen._n_act
    state = {}

    def call(i):  # ONE launch, as the native driver issues it (mapped completion; the rank count is part of the kernel)
        gen._probe_mapped_once((i * 7919) % n, state)

    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for i in range(3):
        call(i)
    times = []
    for i in range(10):
        flush.zero_()  # > L2 (50 MB): the next probe reads from HBM
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call(i + 3)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    ms = float(np.median(times))
    nbytes = n * (4 * gen._d + 5)
    return {"kernel": "probe_kernel<32>", "ms": ms, "gbs": nbytes / (ms * 1e-3) / 1e9, "bytes": nbytes}


# ---------------------------------------------------------------------------------- CPU baseline
def cpu_baseline(abundance, tnf, lengths, nsamples, nepochs, seed, budget_s, latent=None):
    """The oracle port (torch-CPU fp32 VAE restatement with the restated DAdaptAdam + the C/NumPy clusterer) on ONE
    BOUNDED sample of the same workload, extrapolated over the bin-default schedule.  A reported baseline, not
    the optimisation target.  Imports oracle/ only."""
    from oracle import cluster_oracle as co
    from oracle import normalize as onorm
    from oracle import vae_oracle as vo

    n = len(lengths)
    threads = torch.get_num_threads()
    d, t, a, w = (torch.from_numpy(x) for x in onorm.normalize(abundance, tnf, lengths))
    orc = vo.OracleVAE(nsamples, seed=seed)
    rng = np.random.default_rng(seed)
    per_step = {}
    sched = schedule(n, nepochs)
    share = budget_s * 0.5 / max(1, len(sched))
    for batch, spe, epochs in sched:
        b = min(batch, n)
        times = []
        t_start = time.perf_counter()
        while len(times) < 3 or (time.perf_counter() - t_start < share and len(times) < 50):
            idx = torch.from_numpy(rng.integers(0, n, size=b))
            t0 = time.perf_counter()
            orc.train_step(d[idx], t[idx], a[idx], w[idx])
            times.append(time.perf_counter() - t0)
        per_step[batch] = float(np.median(times[1:]))
    t_train = sum(per_step[b] * spe * e for b, spe, e in sched)
    m = min(n, 50_000)
    t0 = time.perf_counter()
    orc.encode(d[:m], t[:m], a[:m])
    t_encode = (time.perf_counter() - t0) * n / m
    # clustering: a prefix of the clusters of the full-size latent (the reference's own max_clusters mechanism,
    # vamb/__main__.py:1289).  The reference packs the matrix after every cluster (cluster.py:318-335), so a pass
    # costs time proportional to the rows still unclustered; those fall roughly linearly from n to 0 over the
    # run, hence the mean cost per cluster is ~half the cost measured on the (full-size) prefix.
    if latent is None:
        from oracle import synth

        latent, _ = synth.make_latent(n, 32, seed=seed, spread=0.2)
    gen = co.OracleClusterGenerator(latent, lengths, windowsize=300, minsuccesses=15, rng_seed=seed)
    t0 = time.perf_counter()
    clustered = k = 0
    for c in gen:
        clustered += len(c.members)
        k += 1
        if time.perf_counter() - t0 > budget_s * 0.4:
            break
    dt = time.perf_counter() - t0
    t_cluster = 0.5 * dt * n / max(1, clustered)
    total = t_train + t_encode + t_cluster
    sample = (f"oracle port, {threads} threads (the reference's own cap min(ncpu, 8)); ONE sample: train = median of >=3 "
              f"optimiser steps per batch size {sorted(per_step)} extrapolated over {sum(s * e for _, s, e in sched)} steps; "
              f"encode = {m} rows scaled to {n}; cluster = first {k} clusters ({clustered} contigs, {dt:.1f} s) scaled to "
              f"{n} contigs x 0.5 (per-pass cost follows the linearly shrinking remainder)")
    return {"value": n / total, "unit": "contigs/s", "cores": threads, "kind": "port", "sample": sample,
            "t_train_est": t_train, "t_encode_est": t_encode, "t_cluster_est": t_cluster}


def main_reference(args, rank):
    if rank != 0:
        return
    torch.set_num_threads(reference_threads())
    ab, tnf, lens = make_workload(args.n, args.nsamples, args.seed)
    log("reference arm: one bounded sample of the workload on the host cores")
    base = cpu_baseline(ab, tnf, lens, args.nsamples, args.nepochs, args.seed, args.cpu_seconds)
    v = base["value"]
    emit_json({
        "impl": "reference", "metric": METRIC, "value": v, "unit": "contigs/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * args.n / v / max(1, args.steps),
        "higher_is_better": True, "scaling": args.scaling, "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": workload_name(args),
                   "parallelism": "cpu: the reference's own thread cap min(ncpu, 8)",
                   "note": "CPU port of the reference path (oracle/): the reference itself needs vambcore + dadaptation, "
                           "which are not in the image.  The K steps of the GPU arm are K slices of one pass; this arm "
                           "times ONE bounded sample of that pass (independent of --steps/--warmup) and extrapolates"},
        "cpu_baseline": base,
        "e2e": {"value": v, "unit": "contigs/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    })


_JSON_OUT = None


def claim_stdout() -> None:
    """stdout carries exactly ONE JSON line: keep a private handle on the real stdout for it and point file descriptor 1
    at stderr for everything else (NCCL prints its version banner to stdout at NCCL_DEBUG=WARN/VERSION; child
    processes and C libraries write to fd 1 directly)."""
    global _JSON_OUT
    sys.stdout.flush()
    _JSON_OUT = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)


def emit_json(obj) -> None:
    out = _JSON_OUT if _JSON_OUT is not None else sys.stdout
    out.write(json.dumps(obj) + "\n")
    out.flush()


def main():
    args = parse_args()
    claim_stdout()
    ctx = Ctx(args)
    if args.impl == "reference":
        return main_reference(args, ctx.rank)

    import vamb_b200.encode as ve
    from vamb_b200 import parallel as par
    from torch.utils.data import DataLoader, TensorDataset

    world, rank = ctx.world, ctx.rank
    if world > 1:
        import torch.distributed as dist

        torch.cuda.set_device(ctx.local_rank)
        dist.init_process_group("nccl", device_id=torch.device("cuda", ctx.local_rank))
    else:
        torch.cuda.set_device(0)

    if world > 1 and ctx.strong:
        # the same dataset on every rank, normalised globally (z-scores are over all contigs), then row-sharded
        ab, tnf, lens = make_workload(args.n, args.nsamples, args.seed)
        full = ve.make_dataloader(ab, tnf, lens, batchsize=256, destroy=True)
        lo, hi = par.shard_rows(args.n, rank, world)
        shard = TensorDataset(*(t[lo:hi].clone() for t in full.dataset.tensors))
        dl = DataLoader(shard, batch_size=256, shuffle=True, drop_last=(hi - lo) > 256)
        lens_cluster = lens  # rank 0 clusters the gathered latent of all contigs
        del full
        n_total = args.n
    else:
        ab, tnf, lens = make_workload(args.n, args.nsamples, args.seed + rank)
        dl = ve.make_dataloader(ab.copy(), tnf.copy(), lens, batchsize=256)
        lens_cluster = lens
        n_total = world * args.n
    log(f"workload ready: {len(dl.dataset.tensors[0])} contigs on this rank x {args.nsamples} samples")

    for i in range(args.warmup):
        log(f"warm-up pass {i + 1}/{args.warmup}")
        run_pass(ctx, dl, lens_cluster, 5, 1, resident=True, max_clusters=300, batchsteps=[1, 2, 3, 4])

    sampler = ClockSampler(ctx.local_rank)
    sampler.start()
    log(f"timed pass: {args.steps} steps (dataset resident in HBM)")
    res = run_pass(ctx, dl, lens_cluster, args.nepochs, args.steps, resident=True)
    clocks = sampler.stop()
    if args.dump_outputs and rank == 0 and res["latent_dev"] is not None:  # weak scaling: rank 0's own sample
        dump_outputs(args.dump_outputs, res, len(lens_cluster), args.seed)
        log(f"outputs of the timed pass written to {args.dump_outputs}")
    t_pass = ctx.max_over_ranks(res["t_event"])
    value = n_total / t_pass
    log(f"  {t_pass:.2f}s: train {res['phases']['train']:.2f} encode {res['phases']['encode']:.2f} cluster "
        f"{res['phases']['cluster']:.2f}; {res['n_clusters']} clusters; loss {res['final_loss']:.4f}")

    e2e = None
    if args.no_e2e:
        e2e_note = "skipped (--no-e2e)"
    elif elapsed() + 1.15 * res["t_wall"] + 60 > args.time_budget:
        e2e_note = f"skipped: would exceed --time-budget {args.time_budget:.0f}s"
    else:
        e2e_note = None
        log("end-to-end pass (pinned host buffers through the public API)")
        pinned = TensorDataset(*(t.pin_memory() for t in dl.dataset.tensors))
        dl_host = DataLoader(pinned, batch_size=256, shuffle=True, drop_last=len(pinned) > 256)
        r2 = run_pass(ctx, dl_host, lens_cluster, args.nepochs, 1, resident=False)
        t2 = ctx.max_over_ranks(r2["t_event"])
        n_loc = len(pinned)
        d_in = args.nsamples + 104
        n_clu = len(lens_cluster)
        h2d = n_loc * (d_in + 1) * 4 + n_clu * 32 * 4 + n_clu * 4  # dataset + weights; latent + lengths (clusterer)
        d2h = n_loc * 32 * 4 + n_clu * 4 + r2["probes"] * 512 + r2["evals"] * 768  # latent, ids, probe heads, densities
        e2e = {"value": n_total / t2, "unit": "contigs/s", "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h),
               "t_train": r2["phases"]["train"], "t_encode": r2["phases"]["encode"], "t_cluster": r2["phases"]["cluster"],
               "api": "make_dataloader tensors (pinned host) -> VAE.trainmodel -> VAE.encode -> numpy -> ClusterGenerator"}

    if rank == 0:
        hbm_peak, tf_peak, tf_label, hbm_label = datasheet_peaks()
        log("kernel rooflines")
        best, share = vae_roofline(res["vae"], len(dl.dataset.tensors[0]), args.nepochs)
        roof = {"bound": "tensor", "kernel": best["kernel"], "achieved": best["tflops"], "peak": tf_peak,
                "unit": "TFLOP/s", "frac": best["tflops"] / tf_peak, "traffic": None,
                "peak_source": tf_label, "time_share": share, "ms_per_launch": best["ms"],
                "note": "algorithmic FLOP of the launch (wgrad + dgrad, SURVEY 8d) / CUDA-event time of the launch; the tensor "
                        "pipe executes 3x these FLOP (3xTF32 error compensation)"}
        roof_cluster = None
        if res["latent_dev"] is not None:
            pr = probe_roofline(res["latent_dev"], lens_cluster)
            roof_cluster = {"bound": "hbm", "kernel": pr["kernel"], "achieved": pr["gbs"], "peak": hbm_peak,
                            "unit": "GB/s", "frac": pr["gbs"] / hbm_peak, "traffic": None,
                            "algorithmic_bytes": pr["bytes"], "ms_per_launch": pr["ms"],
                            "peak_source": hbm_label}
            log(f"  dominant {best['kernel']}: {best['tflops']:.1f} TFLOP/s; probe {pr['gbs']:.0f} GB/s")
        base = None
        if world == 1:
            if elapsed() + args.cpu_seconds * 1.6 + 30 > args.time_budget:
                base = {"value": None, "unit": "contigs/s", "cores": 0, "kind": "port",
                        "sample": f"skipped: would exceed --time-budget {args.time_budget:.0f}s"}
            else:
                log("cpu baseline sample")
                torch.set_num_threads(reference_threads())
                base = cpu_baseline(ab, tnf, lens, args.nsamples, args.nepochs, args.seed, args.cpu_seconds)
        mode = "strong" if (ctx.strong and world > 1) else "weak"
        par_desc = (f"dp{world}: rows of ONE {args.n}-contig dataset sharded over {world} GPUs, 1 gradient all-reduce / minibatch "
                    f"(global batch {world} x B), per-shard encode, NVLink all-gather of the latent, single clustering on rank 0"
                    if mode == "strong" and world > 1 else
                    f"dp{world}: one {args.n}-contig sample per GPU, 1 gradient all-reduce / minibatch, per-shard encode + clustering")
        out = {
            "metric": METRIC, "value": value, "unit": "contigs/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": 1e3 * t_pass / max(1, args.steps), "higher_is_better": True,
            "scaling": mode, "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": workload_name(args), "parallelism": par_desc,
                       "step": f"1/{args.steps} of one pass: {args.nepochs}/{args.steps} epochs of the schedule per step, "
                               "encode + clustering in the last step",
                       "l2": "inputs larger than L2 (620 MB dataset, 128 MB latent); the probe roofline flushes L2 between launches",
                       "warmup_workload": "same path, 5 epochs covering all 5 batch sizes, clustering capped at 300"},
            "step_ms": [round(x, 2) for x in res["step_ms"]],
            "phases_s": res["phases"], "t_pass_wall_s": res["t_wall"],
            "clusters": res["n_clusters"], "final_loss": res["final_loss"],
            "cluster_host_seconds": dict(res["cluster_timing"], probes=res["probes"], evals=res["evals"]),
            "roofline": roof, "roofline_cluster": roof_cluster, "cpu_baseline": base,
            "e2e": e2e if e2e is not None else {"value": None, "unit": "contigs/s", "h2d_bytes_per_step": 0,
                                                "d2h_bytes_per_step": 0, "note": e2e_note},
            "gpu_launches": int(res["launches"]), "clocks": clocks,
        }
        emit_json(out)
    if world > 1:
        import torch.distributed as dist

        dist.barrier()
        torch.cuda.synchronize()
        sys.stdout.flush()
        sys.stderr.flush()
        # Orderly teardown: drop the captured graphs (they hold NCCL kernels) before the communicator goes away.
        # A watchdog ends the process if the teardown blocks (seen with some NCCL builds) -- all work is done.
        threading.Timer(20.0, lambda: os._exit(0)).start()
        res["vae"]._graphs.clear()
        del res
        import gc

        gc.collect()
        torch.cuda.synchronize()
        dist.destroy_process_group()
        os._exit(0)


if __name__ == "__main__":
    main()
