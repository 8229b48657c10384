"""TEST INFRASTRUCTURE -- torch-CPU fp32 oracle for the VAE path.

A restatement of vamb/encode.py (``VAE`` forward, ``calc_loss``,
one optimiser step, ``encode``) as a small functional model over a plain
``state_dict`` whose keys/shapes equal the reference's (encode.py:226-249), so
that reference weights can be loaded and compared directly.

Random inputs are EXPLICIT: ``eps`` (reparameterisation noise, encode.py:277) and
the four dropout keep-masks (encode.py:264,292) are arguments.  When they are
``None`` they are drawn from torch's global CPU generator with the same calls, in
the same order, as the reference's forward pass -- which makes this oracle
bit-identical to the reference under ``torch.manual_seed`` (checked in
tests/test_oracle_vs_reference.py) and lets the CUDA path be tested with the very
same noise.

The optimiser is oracle/dadapt.py (restated DAdaptAdam; parity unpinned).
"""
from __future__ import annotations

from collections import OrderedDict
from math import log
from typing import Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

NTNF = 103
LEAKY_SLOPE = 0.01  # nn.LeakyReLU() default, encode.py:252
BN_EPS = 1e-5
BN_MOMENTUM = 0.1


def defaults(nsamples: int, nhiddens=None, alpha=None, dropout=0.2):
    """encode.py:188-196."""
    if alpha is None:
        alpha = 0.15 if nsamples > 1 else 0.50
    if nhiddens is None:
        nhiddens = [512, 512] if nsamples > 1 else [256, 256]
    if dropout is None:
        dropout = 0.2 if nsamples > 1 else 0.0
    return list(nhiddens), alpha, dropout


def init_state(nsamples: int, nhiddens: Sequence[int], nlatent: int, seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """Draw the initial parameters exactly as ``VAE.__init__`` does (encode.py:210-249):
    ``torch.manual_seed(seed)`` and then nn.Linear / nn.BatchNorm1d constructed in the
    reference's order (PyTorch default init consumes the global CPU generator)."""
    torch.manual_seed(seed)
    _ = torch.Generator().manual_seed(seed)  # encode.py:211-212 (does not touch the global stream)
    state: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    nin_all = nsamples + NTNF + 1
    enc_l, enc_n, dec_l, dec_n = [], [], [], []
    for nin, nout in zip([nin_all] + list(nhiddens), nhiddens):
        enc_l.append(torch.nn.Linear(nin, nout))
        enc_n.append(torch.nn.BatchNorm1d(nout))
    mu = torch.nn.Linear(nhiddens[-1], nlatent)
    rev = list(nhiddens[::-1])
    for nin, nout in zip([nlatent] + rev, rev):
        dec_l.append(torch.nn.Linear(nin, nout))
        dec_n.append(torch.nn.BatchNorm1d(nout))
    out = torch.nn.Linear(nhiddens[0], nin_all)

    def put(prefix, mod):
        for k, v in mod.state_dict().items():
            state[f"{prefix}.{k}"] = v.detach().clone()

    # registration order of the reference module (encode.py:226-249)
    for i, m in enumerate(enc_l):
        put(f"encoderlayers.{i}", m)
    for i, m in enumerate(enc_n):
        put(f"encodernorms.{i}", m)
    for i, m in enumerate(dec_l):
        put(f"decoderlayers.{i}", m)
    for i, m in enumerate(dec_n):
        put(f"decodernorms.{i}", m)
    put("mu", mu)
    put("outputlayer", out)
    return state


def param_keys(state) -> list:
    """Trainable tensors in ``module.parameters()`` order."""
    return [k for k in state if not (k.endswith("running_mean") or k.endswith("running_var") or k.endswith("num_batches_tracked"))]


def _block(x, state, lin, norm, keep, p, training):
    """encode.py:264 / :292 -- BatchNorm(Dropout(LeakyReLU(Linear(x))))."""
    h = F.linear(x, state[f"{lin}.weight"], state[f"{lin}.bias"])
    h = F.leaky_relu(h, LEAKY_SLOPE)
    if training and p > 0.0:
        if keep is None:
            # same RNG consumption and arithmetic as nn.Dropout on CPU: x * (bernoulli(1-p) / (1-p))
            keep = torch.empty_like(h).bernoulli_(1 - p)
        h = h * (keep.to(h.dtype) / (1 - p))
    h = F.batch_norm(
        h, state[f"{norm}.running_mean"], state[f"{norm}.running_var"],
        state[f"{norm}.weight"], state[f"{norm}.bias"], training, BN_MOMENTUM, BN_EPS,
    )
    if training:
        state[f"{norm}.num_batches_tracked"] += 1
    return h, keep


def forward(state, depths, tnf, abundance, nsamples: int, dropout: float, training: bool,
            eps: Optional[torch.Tensor] = None, keeps: Optional[list] = None):
    """encode.py:306-314.  Returns (depths_out, tnf_out, abundance_out, mu, eps, keeps)."""
    nenc = sum(1 for k in state if k.startswith("encoderlayers.") and k.endswith(".weight"))
    ndec = sum(1 for k in state if k.startswith("decoderlayers.") and k.endswith(".weight"))
    keeps_in = list(keeps) if keeps is not None else [None] * (nenc + ndec)
    keeps_out = []
    x = torch.cat((depths, tnf, abundance), 1)
    for i in range(nenc):
        x, k = _block(x, state, f"encoderlayers.{i}", f"encodernorms.{i}", keeps_in[i], dropout, training)
        keeps_out.append(k)
    mu = F.linear(x, state["mu.weight"], state["mu.bias"])
    if eps is None:
        eps = torch.randn(mu.size(0), mu.size(1))  # encode.py:277 (drawn in eval mode too)
    x = mu + eps
    for i in range(ndec):
        x, k = _block(x, state, f"decoderlayers.{i}", f"decodernorms.{i}", keeps_in[nenc + i], dropout, training)
        keeps_out.append(k)
    rec = F.linear(x, state["outputlayer.weight"], state["outputlayer.bias"])
    depths_out = F.softmax(rec.narrow(1, 0, nsamples), dim=1)
    tnf_out = rec.narrow(1, nsamples, NTNF)
    ab_out = rec.narrow(1, nsamples + NTNF, 1)
    return depths_out, tnf_out, ab_out, mu, eps, keeps_out


def loss_weights(nsamples: int, nlatent: int, alpha: float, beta: float):
    """encode.py:334-343."""
    ce_w = 0.0 if nsamples == 1 else ((1 - alpha) * (nsamples - 1)) / (nsamples * log(nsamples))
    ab_w = (1 - alpha) * (1 / nsamples)
    sse_w = alpha / NTNF
    kld_w = 1 / (nlatent * beta)
    return ce_w, ab_w, sse_w, kld_w


def calc_loss(depths_in, depths_out, tnf_in, tnf_out, ab_in, ab_out, mu, weights,
              nsamples, nlatent, alpha, beta):
    """encode.py:316-357.  Returns (loss, ab, ce, sse, kld) means."""
    ce_w, ab_w, sse_w, kld_w = loss_weights(nsamples, nlatent, alpha, beta)
    ab_sse = (ab_out - ab_in).pow(2).sum(dim=1)
    ce = -((depths_out + 1e-9).log() * depths_in).sum(dim=1)
    sse = (tnf_out - tnf_in).pow(2).sum(dim=1)
    kld = 0.5 * (mu.pow(2)).sum(dim=1)
    w_ab, w_ce, w_sse, w_kld = ab_sse * ab_w, ce * ce_w, sse * sse_w, kld * kld_w
    # NOTE (reference quirk, kept on purpose): the per-row losses have shape [B] while
    # ``weights`` has shape [B, 1] (encode.py:126,349), so the product broadcasts to [B, B]
    # and ``loss.mean()`` equals mean_j(l_j) * mean_i(w_i): every row is weighted by the
    # BATCH-MEAN weight, not by its own weight.
    loss = ((w_ce + w_ab + w_sse) + w_kld) * weights
    return loss.mean(), w_ab.mean(), w_ce.mean(), w_sse.mean(), w_kld.mean()


class OracleVAE:
    """Stateful convenience wrapper: parameters + restated DAdaptAdam."""

    def __init__(self, nsamples, nhiddens=None, nlatent=32, alpha=None, beta=200.0, dropout=0.2, seed=0,
                 state=None):
        self.nsamples, self.nlatent, self.beta = nsamples, nlatent, beta
        self.nhiddens, self.alpha, self.dropout = defaults(nsamples, nhiddens, alpha, dropout)
        self.state = state if state is not None else init_state(nsamples, self.nhiddens, nlatent, seed)
        self.params = [self.state[k] for k in param_keys(self.state)]
        self.opt = None

    def load_reference_state(self, sd):
        for k in self.state:
            self.state[k].copy_(sd[k])

    def grads(self, depths, tnf, ab, weights, eps=None, keeps=None):
        """One forward+backward in train mode.  Returns (losses5, {key: grad}, eps, keeps)."""
        for p in self.params:
            p.requires_grad_(True)
            p.grad = None
        d_out, t_out, a_out, mu, eps, keeps = forward(
            self.state, depths, tnf, ab, self.nsamples, self.dropout, True, eps, keeps
        )
        losses = calc_loss(depths, d_out, tnf, t_out, ab, a_out, mu, weights.reshape(-1, 1),
                           self.nsamples, self.nlatent, self.alpha, self.beta)
        losses[0].backward()
        g = {k: self.state[k].grad.detach().clone() for k in param_keys(self.state)}
        for p in self.params:
            p.requires_grad_(False)
        return [float(x.detach()) for x in losses], g, eps, keeps

    def train_step(self, depths, tnf, ab, weights, eps=None, keeps=None):
        """encode.py:401-419 with the restated optimiser."""
        from .dadapt import DAdaptAdam

        losses, g, eps, keeps = self.grads(depths, tnf, ab, weights, eps, keeps)
        if self.opt is None:
            self.opt = DAdaptAdam(self.params, decouple=True)
        for k, p in zip(param_keys(self.state), self.params):
            p.grad = g[k]
        self.opt.step()
        return losses, eps, keeps

    @property
    def d(self) -> float:
        return self.opt.param_groups[0]["d"] if self.opt is not None else 1e-6

    def encode(self, depths, tnf, ab, batch: int = 256) -> np.ndarray:
        """encode.py:442-484: eval-mode mu for every row, then mask the low 12 mantissa bits."""
        n = len(depths)
        out = np.empty((n, self.nlatent), dtype=np.float32)
        with torch.no_grad():
            for i in range(0, n, batch):
                sl = slice(i, min(n, i + batch))
                mu = forward(self.state, depths[sl], tnf[sl], ab[sl], self.nsamples, self.dropout, False,
                             eps=torch.zeros(sl.stop - sl.start, self.nlatent))[3]
                out[sl] = mu.numpy()
        raw = out.copy()
        u = out.view(np.uint32)
        u &= ~np.uint32(2 ** 12 - 1)  # vambtools.py:324-330
        return out, raw
