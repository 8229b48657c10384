"""Gradient error against an fp64 evaluation of the same step, for the CUDA paths AND for the fp32 CPU oracle.

For B in {256, 1024, 4096} on the bin-default network (S = 50): one forward + backward with the same batch, noise and
dropout masks in (a) fp64 torch on the CPU (the yardstick), (b) the fp32 torch oracle, (c) the CUDA tensor-core path
(3xTF32), (d) the CUDA fp32 CUDA-core path.  Prints, per gradient tensor, ||g - g64|| / ||g64|| and writes the
table as JSON to $GRAD_OUT (default grad_error_fp64.json in the working directory).
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import vamb_b200.encode as ve
from oracle import vae_oracle as vo
from oracle.make_golden_vae import vae_inputs


def rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def grads_fp64(o32, d, t, a, w, eps, keeps):
    o = vo.OracleVAE(o32.nsamples, seed=0, state={k: (v.double().clone() if v.is_floating_point() else v.clone())
                                                  for k, v in o32.state.items()})
    o.nhiddens, o.alpha, o.dropout, o.beta = o32.nhiddens, o32.alpha, o32.dropout, o32.beta
    _, g, _, _ = o.grads(d.double(), t.double(), a.double(), w.double(), eps.double(), [k.double() for k in keeps])
    return g


def main():
    # GRAD_CASES="S:B,S:B,..." overrides the default sweep (S = 50 at B = 256, 1024, 4096)
    cases = [(50, 256), (50, 1024), (50, 4096)]
    if os.environ.get("GRAD_CASES"):
        cases = [tuple(int(x) for x in c.split(":")) for c in os.environ["GRAD_CASES"].split(",")]
    out = {}
    for S, B in cases:
        n = max(5000, B + 1000)
        rpkm, tnfs, lens = vae_inputs(S, n, 7)
        dl = ve.make_dataloader(rpkm.copy(), tnfs.copy(), lens, batchsize=B)
        d, t, a, w = dl.dataset.tensors
        idx = torch.from_numpy(np.random.default_rng(0).choice(n, B, replace=False))
        o = vo.OracleVAE(S, seed=2)
        torch.manual_seed(5)
        _, g32, eps, keeps = o.grads(d[idx], t[idx], a[idx], w[idx])
        g64 = grads_fp64(o, d[idx], t[idx], a[idx], w[idx], eps, keeps)
        row = {"oracle_fp32": {k: rel(g32[k].numpy(), g64[k].numpy()) for k in g64}}
        for name, tcmin, flush, staging in (("cuda_tc_3xtf32", 1, 0, 0), ("cuda_tc_3xtf32_wgrad_flush128", 1, 1, 0),
                                            ("cuda_tc_3xtf32_prep_staging", 1, 0, 1), ("cuda_fp32_ffma", 0, 0, 0)):
            vae = ve.VAE(S, seed=2)
            vae._net.tc_min_batch = tcmin
            vae._net.wgrad_flush = flush
            vae._net.staging = staging
            vae._step_injected(dl.dataset.tensors, idx.numpy(), eps.numpy(), [k.numpy() for k in keeps], optimize=False)
            got = vae._grad_dict()
            row[name] = {k: rel(got[k].cpu().numpy(), g64[k].numpy()) for k in g64}
        out[f"S{S}_B{B}"] = row
        print(f"S = {S}, B = {B}: worst tensor / median over tensors of ||g - g64|| / ||g64||")
        for name, errs in row.items():
            worst = max(errs, key=errs.get)
            print(f"  {name:36s} worst {errs[worst]:.2e} ({worst})  median {np.median(list(errs.values())):.2e}")
            if errs[worst] > 5e-5:
                print("      tensors above 5e-5:", {k: float(f"{v:.2e}") for k, v in errs.items() if v > 5e-5})
    with open(os.environ.get("GRAD_OUT", "grad_error_fp64.json"), "w") as fh:
        json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
