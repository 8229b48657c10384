"""Per-tensor gradient error of the tensor-core (3xTF32) path vs the torch-fp32 oracle (and the fp32 CUDA-core path)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import vamb_b200.encode as ve
from oracle import vae_oracle as vo
from oracle.make_golden_vae import vae_inputs

def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))

B = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
S, n = 50, 5000
rpkm, tnfs, lens = vae_inputs(S, n, 7)
dl = ve.make_dataloader(rpkm.copy(), tnfs.copy(), lens, batchsize=B)
d, t, a, w = dl.dataset.tensors
o = vo.OracleVAE(S, seed=2)
idx = torch.from_numpy(np.random.default_rng(0).choice(n, B, replace=False))
torch.manual_seed(5)
lo, grads, eps, keeps = o.grads(d[idx], t[idx], a[idx], w[idx])
for tc in (0, 1):
    vae = ve.VAE(S, seed=2)
    vae._net.tc_min_batch = 1 if tc else 0
    losses = vae._step_injected(dl.dataset.tensors, idx.numpy(), eps.numpy(), [k.numpy() for k in keeps], optimize=False)
    got = vae._grad_dict()
    print(f"B={B} tc={tc} tile_n={os.environ.get('VK_TC_TILE_N')} nsplit={os.environ.get('VK_TC_NSPLIT')} loss rel {abs(losses[0]-lo[0])/lo[0]:.2e}")
    for k, g in grads.items():
        print(f"   {k:28s} {rel(got[k].cpu().numpy(), g.numpy()):.3e}")
