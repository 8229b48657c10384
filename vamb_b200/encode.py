__doc__ = """Encode a depths matrix and a tnf matrix to latent representation on H100.

Drop-in for ``vamb.encode`` (RasmussenLab/vamb, vamb/encode.py): ``make_dataloader``,
``set_batchsize`` and ``VAE`` keep the reference's names, arguments, attributes,
``state_dict`` layout, exceptions and return types.  What differs is where the work runs:

  * the normalised dataset is uploaded to HBM once; minibatches are drawn on the device by
    an epoch-keyed pseudo-random permutation (no DataLoader worker, no per-step H2D);
  * one optimiser step = 15 hand-written sm_90a kernel launches (vamb_b200/csrc/vk_vae.cu)
    -- batch gather, fused Linear+LeakyReLU+Dropout+BatchNorm forward, loss, fused
    backward, single-pass D-Adaptation Adam -- replayed from CUDA graphs, with the five
    loss scalars accumulated on the device and read once per epoch;
  * ``encode`` runs the eval-mode encoder in large batches and masks the low mantissa bits
    in the epilogue of the mu layer.

Usage is the reference's:
>>> vae = VAE(nsamples=6)
>>> dataloader = make_dataloader(depths, tnf, lengths)
>>> vae.trainmodel(dataloader)
>>> latent = vae.encode(dataloader)
"""

import ctypes as _ct
import os as _os
from math import log as _log
from pathlib import Path
from typing import IO, Optional, Union

import numpy as _np
import torch as _torch
import torch.distributed as _dist
from torch import Tensor
from torch import nn as _nn
from torch.nn.functional import softmax as _softmax
from torch.utils.data import DataLoader as _DataLoader
from torch.utils.data.dataset import TensorDataset as _TensorDataset

from . import _lib
from . import parallel as _par
from . import vambtools as _vambtools

try:  # the reference logs through loguru; fall back to the std logger when it is absent
    from loguru import logger
except ImportError:  # pragma: no cover
    import logging

    logger = logging.getLogger("vamb_b200")

_warned = set()


def _warn_once(msg: str) -> None:
    if msg not in _warned:
        _warned.add(msg)
        logger.warning(msg)


_MAX_BATCH = 8192  # rows of the activation workspaces (training batches double up to 4096)
_GRAPH_CHUNKS = (128, 16, 4)  # optimiser steps per captured CUDA graph, largest first
_WGRAD_FLUSH = 0  # default of vk_vae.wgrad_flush: the plain chain is fp32-grade against fp64 (tools/grad_error_fp64.py)
_USE_TMA = 1  # default of vk_vae.use_tma (both feeds are checked by tests/test_vae_gpu.py, test_tc_gpu.py)
_TC_MIN_BATCH = 128  # batches >= this run their GEMMs on the wgmma tensor-core path (0 = never)


def set_batchsize(data_loader: _DataLoader, batch_size: int, n_obs: int, encode=False) -> _DataLoader:
    """Copy of the loader with another batch size (vamb/encode.py:33-50).  With ``encode`` the
    copy neither shuffles nor drops the last partial batch."""
    return _DataLoader(
        dataset=data_loader.dataset,
        batch_size=batch_size,
        shuffle=not encode,
        drop_last=not encode and (n_obs > batch_size),
        num_workers=1 if encode else data_loader.num_workers,
        pin_memory=data_loader.pin_memory,
        collate_fn=data_loader.collate_fn,
    )


def make_dataloader(
    abundance: _np.ndarray,
    tnf: _np.ndarray,
    lengths: _np.ndarray,
    batchsize: int = 256,
    destroy: bool = False,
    cuda: bool = False,
) -> _DataLoader:
    """Normalise abundance / TNF and wrap them for the VAE (vamb/encode.py:53-146).

    The four tensors of ``loader.dataset.tensors`` -- depths [N, S] (rows sum to 1), tnf
    [N, 103] (column z-scores), total abundance [N, 1] (z-scored log), weights [N, 1] (mean
    1) -- are the contract; ``VAE.trainmodel`` uploads them to the GPU once.  The object is
    a genuine ``torch.utils.data.DataLoader`` so that code that inspects or iterates it
    (e.g. the TaxVamb models) keeps working.
    """
    if not isinstance(abundance, _np.ndarray) or not isinstance(tnf, _np.ndarray):
        raise ValueError("TNF and abundance must be Numpy arrays")
    if batchsize < 1:
        raise ValueError(f"Batch size must be minimum 1, not {batchsize}")
    if len(abundance) != len(tnf) or len(tnf) != len(lengths):
        raise ValueError("Lengths of abundance, TNF and lengths arrays must be the same")
    if not (abundance.dtype == tnf.dtype == _np.float32):
        raise ValueError("TNF and abundance must be Numpy arrays of dtype float32")

    if not destroy:
        abundance = abundance.copy()
        tnf = tnf.copy()

    # every sample (column) is scaled to one million
    per_sample = abundance.sum(axis=0)
    if _np.any(per_sample == 0):
        raise ValueError(
            "One or more samples have zero depth in all sequences, so cannot be depth normalized"
        )
    abundance *= 1_000_000 / per_sample
    total_abundance = abundance.sum(axis=1)

    # rows become compositions; an all-zero row becomes uniform
    n_samples = abundance.shape[1]
    is_zero = total_abundance == 0
    abundance[is_zero] = 1 / n_samples
    divisor = total_abundance.copy()
    divisor[is_zero] = 1.0
    abundance /= divisor.reshape((-1, 1))

    total_abundance = _np.log(total_abundance.clip(min=0.001))
    _vambtools.zscore(total_abundance, inplace=True)
    _vambtools.zscore(tnf, axis=0, inplace=True)
    total_abundance.shape = (len(total_abundance), 1)

    # contig weights: max(log(length) - 5, 2), rescaled to mean 1
    lengths = (lengths).astype(_np.float32)
    weights = _np.log(lengths).astype(_np.float32) - 5.0
    weights[weights < 2.0] = 2.0
    weights *= len(weights) / weights.sum()
    weights.shape = (len(weights), 1)

    dataset = _TensorDataset(
        _torch.from_numpy(abundance),
        _torch.from_numpy(tnf),
        _torch.from_numpy(total_abundance),
        _torch.from_numpy(weights),
    )
    return _DataLoader(
        dataset=dataset,
        batch_size=batchsize,
        drop_last=(len(abundance) > batchsize),
        shuffle=True,
        num_workers=4 if cuda else 1,
        pin_memory=cuda,
    )


def reference_epoch_noise(n_seq: int, batch: int, drop_last: bool, nhiddens, nlatent: int, dropout: float):
    """Yield (batch_idx, eps, keeps) for one epoch, consuming torch's global CPU generator exactly as one epoch of
    the reference does: ``iter(DataLoader)`` draws the worker base seed and then the RandomSampler seed
    (torch/utils/data/dataloader.py ``_BaseDataLoaderIter.__init__``, sampler.py ``RandomSampler.__iter__``), the
    permutation comes from a private generator seeded with the latter, and every step draws its dropout masks
    (``empty_like(h).bernoulli_(1 - p)``, one per hidden block in forward order) and ``randn(B, nlatent)`` between
    the encoder and the decoder (vamb/encode.py:264, 277, 292).  Pinned against the live reference by
    tests/test_oracle_vs_reference.py."""
    _torch.empty((), dtype=_torch.int64).random_()
    sampler_seed = int(_torch.empty((), dtype=_torch.int64).random_().item())
    g = _torch.Generator()
    g.manual_seed(sampler_seed)
    perm = _torch.randperm(n_seq, generator=g)
    nb = n_seq // batch if drop_last else (n_seq + batch - 1) // batch
    p = float(dropout)
    for i in range(nb):
        idx = perm[i * batch:(i + 1) * batch]
        b = len(idx)
        keeps = []
        for h in nhiddens:
            keeps.append(_torch.empty(b, h).bernoulli_(1 - p) if p > 0 else None)
        eps = _torch.randn(b, nlatent)
        for h in list(nhiddens)[::-1]:
            keeps.append(_torch.empty(b, h).bernoulli_(1 - p) if p > 0 else None)
        yield idx, eps, keeps


# ---------------------------------------------------------------------- ctypes mirrors
_MAXL = 10


class _VkCtl(_ct.Structure):
    _fields_ = [
        ("d", _ct.c_double), ("num_w", _ct.c_double), ("loss_sums", _ct.c_double * 5), ("wbar", _ct.c_double),
        ("step", _ct.c_int64), ("epoch_step0", _ct.c_int64), ("n_loss_steps", _ct.c_int64),
        ("seed", _ct.c_uint64), ("epoch", _ct.c_int32), ("tickets", _ct.c_int32 * (2 * _MAXL + 4)),
        ("barrier_gen", _ct.c_int32 * (2 * _MAXL)),
    ]


class _VkLayer(_ct.Structure):
    _fields_ = [
        ("k_in", _ct.c_int32), ("n_out", _ct.c_int32), ("kind", _ct.c_int32), ("in_kind", _ct.c_int32),
        ("w_off", _ct.c_int64), ("b_off", _ct.c_int64), ("g_off", _ct.c_int64), ("beta_off", _ct.c_int64),
        ("running_mean", _ct.c_void_p), ("running_var", _ct.c_void_p), ("num_batches_tracked", _ct.c_void_p),
        ("act", _ct.c_void_p), ("dact", _ct.c_void_p), ("fwd_part", _ct.c_void_p), ("bwd_part", _ct.c_void_p),
        ("bn_a", _ct.c_void_p), ("bn_c", _ct.c_void_p), ("bn_mean", _ct.c_void_p), ("bn_rstd", _ct.c_void_p),
        ("bn_m1", _ct.c_void_p), ("bn_m2", _ct.c_void_p),
        ("bn_bA", _ct.c_void_p), ("bn_bB", _ct.c_void_p), ("bn_bC", _ct.c_void_p),
        ("xop_hi", _ct.c_void_p), ("xop_lo", _ct.c_void_p), ("xt_hi", _ct.c_void_p), ("xt_lo", _ct.c_void_p),
        ("dy_hi", _ct.c_void_p), ("dy_lo", _ct.c_void_p), ("dyt_hi", _ct.c_void_p), ("dyt_lo", _ct.c_void_p),
        ("w_hi", _ct.c_void_p), ("w_lo", _ct.c_void_p), ("wt_hi", _ct.c_void_p), ("wt_lo", _ct.c_void_p),
    ]


class _VkVae(_ct.Structure):
    _fields_ = [
        ("n_layers", _ct.c_int32), ("nsamples", _ct.c_int32), ("ntnf", _ct.c_int32), ("nlatent", _ct.c_int32),
        ("d_in", _ct.c_int32), ("bmax", _ct.c_int32),
        ("dropout", _ct.c_float), ("slope", _ct.c_float),
        ("ce_w", _ct.c_float), ("ab_w", _ct.c_float), ("sse_w", _ct.c_float), ("kld_w", _ct.c_float),
        ("n_rows", _ct.c_int64), ("data", _ct.c_void_p), ("weights", _ct.c_void_p),
        ("n_params", _ct.c_int64),
        ("params", _ct.c_void_p), ("grads", _ct.c_void_p), ("exp_avg", _ct.c_void_p),
        ("exp_avg_sq", _ct.c_void_p), ("s", _ct.c_void_p),
        ("z", _ct.c_void_p), ("batch_rows", _ct.c_void_p), ("opt_part", _ct.c_void_p), ("loss_part", _ct.c_void_p),
        ("ctl", _ct.c_void_p),
        ("layers", _VkLayer * _MAXL),
        ("data_ld", _ct.c_int32), ("tc_min_batch", _ct.c_int32), ("grad_slab", _ct.c_int64),
        ("n_grad_slabs", _ct.c_int32), ("staging", _ct.c_int32),
        ("use_tma", _ct.c_int32), ("wgrad_flush", _ct.c_int32),
    ]


class _VkInject(_ct.Structure):
    _fields_ = [("batch_idx", _ct.c_void_p), ("eps", _ct.c_void_p), ("keep", _ct.c_void_p * _MAXL)]


_L = _lib.lib
for _name, _args in {
    "vk_vae_train_step": [_ct.POINTER(_VkVae), _ct.c_int, _ct.POINTER(_VkInject), _ct.c_void_p],
    "vk_vae_grad_step": [_ct.POINTER(_VkVae), _ct.c_int, _ct.POINTER(_VkInject), _ct.c_void_p],
    "vk_vae_forward": [_ct.POINTER(_VkVae), _ct.c_int64, _ct.c_int, _ct.c_int, _ct.c_int, _ct.POINTER(_VkInject), _ct.c_void_p],
    "vk_vae_encode": [_ct.POINTER(_VkVae), _ct.c_int64, _ct.c_int64, _ct.c_int, _ct.c_void_p, _ct.c_void_p],
    "vk_vae_prepare_eval": [_ct.POINTER(_VkVae), _ct.c_void_p],
    "vk_vae_dadapt_step": [_ct.POINTER(_VkVae), _ct.c_void_p],
    "vk_vae_profile_step": [_ct.POINTER(_VkVae), _ct.c_int, _ct.POINTER(_VkInject), _ct.POINTER(_ct.c_float),
                            _ct.POINTER(_ct.c_int), _ct.c_int, _ct.POINTER(_ct.c_int), _ct.c_void_p],
}.items():
    getattr(_L, _name).argtypes = _args
    getattr(_L, _name).restype = _ct.c_int
_L.vk_vae_init_device.argtypes = []
_L.vk_vae_init_device.restype = _ct.c_int
_L.vk_vae_sizeof.argtypes = [_ct.c_int]
_L.vk_vae_sizeof.restype = _ct.c_int64
for _i, _cls in enumerate((_VkVae, _VkLayer, _VkCtl, _VkInject)):
    if _L.vk_vae_sizeof(_i) != _ct.sizeof(_cls):
        raise ImportError(f"vamb_b200: struct {_cls.__name__} is out of sync with include/vamb_b200.h")

_KIND_HIDDEN, _KIND_MU, _KIND_OUT = 0, 1, 2
_IN_DATA, _IN_BN, _IN_Z = 0, 1, 2


class VAE(_nn.Module):
    """Variational autoencoder, subclass of torch.nn.Module.

    Instantiate with:
        nsamples: Number of samples in abundance matrix
        nhiddens: list of n_neurons in the hidden layers [None=Auto]
        nlatent: Number of neurons in the latent layer [32]
        alpha: Approximate starting TNF/(CE+TNF) ratio in loss. [None = Auto]
        beta: Multiply KLD by the inverse of this value [200]
        dropout: Probability of dropout on forward pass [0.2]
        cuda: accepted for API compatibility -- this implementation always runs on the GPU
        seed: seed of the parameter initialisation (CPU generator, as in the reference) and
              of the on-device Philox streams (shuffling, dropout, reparameterisation noise)

    vae.trainmodel(dataloader, nepochs batchsteps, modelfile)
        Trains the model, returning None

    vae.encode(self, data_loader):
        Encodes the data in the data loader and returns the encoded matrix.

    If alpha or dropout is None and there is only one sample, they are set to
    0.99 and 0.0, respectively
    """

    def __init__(
        self,
        nsamples: int,
        nhiddens: Optional[list[int]] = None,
        nlatent: int = 32,
        alpha: Optional[float] = None,
        beta: float = 200.0,
        dropout: Optional[float] = 0.2,
        cuda: bool = False,
        seed: int = 0,
    ):
        # argument checks of vamb/encode.py:182-208, same order and messages
        if nlatent < 1:
            raise ValueError(f"Minimum 1 latent neuron, not {nlatent}")
        if nsamples < 1:
            raise ValueError(f"nsamples must be > 0, not {nsamples}")
        if alpha is None:
            alpha = 0.15 if nsamples > 1 else 0.50
        if nhiddens is None:
            nhiddens = [512, 512] if nsamples > 1 else [256, 256]
        if dropout is None:
            dropout = 0.2 if nsamples > 1 else 0.0
        if any(i < 1 for i in nhiddens):
            raise ValueError(f"Minimum 1 neuron per layer, not {min(nhiddens)}")
        if beta <= 0:
            raise ValueError(f"beta must be > 0, not {beta}")
        if not (0 < alpha < 1):
            raise ValueError(f"alpha must be 0 < alpha < 1, not {alpha}")
        if not (0 <= dropout < 1):
            raise ValueError(f"dropout must be 0 <= dropout < 1, not {dropout}")
        if 2 * len(nhiddens) + 2 > _MAXL:
            raise ValueError(f"at most {(_MAXL - 2) // 2} hidden layers are supported")

        if not cuda:
            # The reference's default (cuda=False) selects its CPU path.  This implementation has none -- it IS the
            # GPU path -- so the flag cannot be honoured; say so once instead of silently ignoring it.
            _warn_once("vamb_b200.encode.VAE always runs on the GPU (sm_90a); cuda=False is not honoured")

        # Parameters are drawn by CPU torch in the reference's construction order
        # (vamb/encode.py:210-249) so that the same seed gives the same initial weights.
        _torch.manual_seed(seed)
        self.rng = _torch.Generator()
        self.rng.manual_seed(seed)
        super(VAE, self).__init__()

        self.usecuda = True
        self.nsamples = nsamples
        self.ntnf = 103
        self.alpha = alpha
        self.beta = beta
        self.nhiddens = nhiddens
        self.nlatent = nlatent
        self.dropout = dropout
        self._seed = int(seed)
        self._bmax = _MAX_BATCH  # rows of the activation workspaces; grown on demand by _ensure_capacity
        # Parity mode: draw batch order, dropout masks and reparameterisation noise from torch's GLOBAL CPU generator
        # with the reference's own calls in the reference's order (vamb/encode.py:210, 264, 277, 292 + the two draws of
        # iter(DataLoader)) and inject them, so that a training run follows the CPU reference's trajectory for the same
        # ``seed``.  Slow (host RNG + H2D per step); the default draws everything on the device (Philox).
        self.strict_rng = _os.environ.get("VAMB_B200_STRICT_RNG", "0") not in ("", "0")

        self.encoderlayers = _nn.ModuleList()
        self.encodernorms = _nn.ModuleList()
        self.decoderlayers = _nn.ModuleList()
        self.decodernorms = _nn.ModuleList()
        nin_all = self.nsamples + self.ntnf + 1
        for nin, nout in zip([nin_all] + self.nhiddens, self.nhiddens):
            self.encoderlayers.append(_nn.Linear(nin, nout))
            self.encodernorms.append(_nn.BatchNorm1d(nout))
        self.mu = _nn.Linear(self.nhiddens[-1], self.nlatent)
        for nin, nout in zip([self.nlatent] + self.nhiddens[::-1], self.nhiddens[::-1]):
            self.decoderlayers.append(_nn.Linear(nin, nout))
            self.decodernorms.append(_nn.BatchNorm1d(nout))
        self.outputlayer = _nn.Linear(self.nhiddens[0], nin_all)
        self.relu = _nn.LeakyReLU()
        self.softplus = _nn.Softplus()
        self.dropoutlayer = _nn.Dropout(p=self.dropout)

        _lib.require_device()  # no CPU path
        self.cuda()
        self._build_device_state()

    # ------------------------------------------------------------------ device state
    def _build_device_state(self) -> None:
        dev = next(self.parameters()).device
        f32 = dict(dtype=_torch.float32, device=dev)
        self._keep = {}  # tensors referenced by raw pointer from the C structs

        # flat parameter arena in module.parameters() order; parameters become views of it
        offsets, total = {}, 0
        for name, p in self.named_parameters():
            offsets[name] = total
            total += (p.numel() + 3) // 4 * 4
        arena = _torch.zeros(total, **f32)
        for name, p in self.named_parameters():
            view = arena[offsets[name]:offsets[name] + p.numel()].view_as(p)
            view.copy_(p.data)
            p.data = view
        self._arena = arena
        self._offsets = offsets
        self._n_slabs = 8  # split-K partial-gradient slabs of the tensor-core wgrad (slab 0 = the gradient)
        self._grads_all = _torch.zeros(self._n_slabs * total, **f32)
        self._grads = self._grads_all[:total]
        self._exp_avg = _torch.zeros(total, **f32)
        self._exp_avg_sq = _torch.zeros(total, **f32)
        self._s = _torch.zeros(total, **f32)

        bmax = self._bmax
        n_rt = (bmax + 31) // 32
        net = _VkVae()
        L = len(self.nhiddens)
        net.n_layers = 2 * L + 2
        net.nsamples, net.ntnf, net.nlatent = self.nsamples, self.ntnf, self.nlatent
        net.d_in = self.nsamples + self.ntnf + 1
        net.bmax = bmax
        net.dropout, net.slope = float(self.dropout), 0.01
        ce_w = 0.0 if self.nsamples == 1 else ((1 - self.alpha) * (self.nsamples - 1)) / (self.nsamples * _log(self.nsamples))
        net.ce_w, net.ab_w = ce_w, (1 - self.alpha) * (1 / self.nsamples)
        net.sse_w, net.kld_w = self.alpha / self.ntnf, 1 / (self.nlatent * self.beta)
        net.n_params = total
        net.grad_slab, net.n_grad_slabs = total, self._n_slabs
        net.data_ld = (net.d_in + 3) // 4 * 4
        net.tc_min_batch = _TC_MIN_BATCH
        # 0: the GEMM kernels stage the next GEMM's operands themselves; 1: separate prep launches (same results)
        net.staging = int(_os.environ.get("VAMB_B200_STAGING", "0"))
        # weight operand of the forward / dgrad GEMMs through TMA (cp.async.bulk.tensor) or the cp.async ring
        net.use_tma = int(_os.environ.get("VAMB_B200_TMA", str(_USE_TMA)))
        # wgrad: cut the truncating tensor-core accumulation chain every 128 batch rows (fp32 register sums)
        net.wgrad_flush = int(_os.environ.get("VAMB_B200_WGRAD_FLUSH", str(_WGRAD_FLUSH)))
        with _torch.cuda.device(dev):
            _lib.check(_L.vk_vae_init_device())  # side stream / events of the training step (once per device)
        for field, t in (("params", arena), ("grads", self._grads), ("exp_avg", self._exp_avg),
                         ("exp_avg_sq", self._exp_avg_sq), ("s", self._s)):
            setattr(net, field, t.data_ptr())

        def buf(name, *shape, dtype=_torch.float32):
            t = _torch.zeros(*shape, dtype=dtype, device=dev)
            self._keep[name] = t
            return t.data_ptr()

        net.z = buf("z", bmax, self.nlatent)
        net.batch_rows = buf("batch_rows", bmax, dtype=_torch.int64)
        # partial sums: two doubles per 1024-parameter block of the optimiser + one per 32 batch rows (weight fold); four
        # doubles per 8-row block of the loss kernel (include/vamb_b200.h: vk_vae.opt_part / loss_part)
        net.opt_part = buf("opt_part", 2 * ((total + 1023) // 1024) + bmax // 32 + 8, dtype=_torch.float64)
        net.loss_part = buf("loss_part", 4 * ((bmax + 31) // 32 * 32 // 8) + 64, dtype=_torch.float64)
        self._ctl = _torch.zeros(_ct.sizeof(_VkCtl), dtype=_torch.uint8, device=dev)
        net.ctl = self._ctl.data_ptr()

        specs = []  # (prefix of the Linear, BatchNorm module or None, kind, in_kind)
        for i in range(L):
            specs.append((f"encoderlayers.{i}", self.encoderlayers[i], self.encodernorms[i], f"encodernorms.{i}",
                          _KIND_HIDDEN, _IN_DATA if i == 0 else _IN_BN))
        specs.append(("mu", self.mu, None, None, _KIND_MU, _IN_BN))
        for i in range(L):
            specs.append((f"decoderlayers.{i}", self.decoderlayers[i], self.decodernorms[i], f"decodernorms.{i}",
                          _KIND_HIDDEN, _IN_Z if i == 0 else _IN_BN))
        specs.append(("outputlayer", self.outputlayer, None, None, _KIND_OUT, _IN_BN))
        for j, (lname, lin, bn, bname, kind, in_kind) in enumerate(specs):
            ly = net.layers[j]
            ly.k_in, ly.n_out, ly.kind, ly.in_kind = lin.in_features, lin.out_features, kind, in_kind
            ly.w_off, ly.b_off = offsets[f"{lname}.weight"], offsets[f"{lname}.bias"]
            ly.g_off = ly.beta_off = -1
            n = lin.out_features
            ly.act = buf(f"act{j}", bmax, n)
            ly.dact = buf(f"dact{j}", bmax, n)
            if bn is not None:
                ly.g_off, ly.beta_off = offsets[f"{bname}.weight"], offsets[f"{bname}.bias"]
                ly.running_mean = bn.running_mean.data_ptr()
                ly.running_var = bn.running_var.data_ptr()
                ly.num_batches_tracked = bn.num_batches_tracked.data_ptr()
                ly.fwd_part = buf(f"fp{j}", n_rt * 2 * n, dtype=_torch.float64)
                ly.bwd_part = buf(f"bp{j}", n_rt * 2 * n, dtype=_torch.float64)
                for f in ("bn_a", "bn_c", "bn_mean", "bn_rstd", "bn_m1", "bn_m2", "bn_bA", "bn_bB", "bn_bC"):
                    setattr(ly, f, buf(f"{f}{j}", n))
            # tensor-core operand staging (see include/vamb_b200.h): zero-initialised, padded
            k = lin.in_features
            r32 = lambda v: (v + 31) // 32 * 32
            r128 = lambda v: (v + 127) // 128 * 128
            for name, rows, cols in (("xop", bmax, r32(k)), ("xt", r128(k + 1), bmax), ("dy", bmax, r32(n)),
                                     ("dyt", r128(n), bmax), ("w", r128(n), r32(k)), ("wt", r128(k), r32(n))):
                setattr(ly, f"{name}_hi", buf(f"{name}_hi{j}", rows, cols))
                # weights: the tf32 remainders are written once per step by prep_weights and fetched by TMA;
                # activations: the GEMM derives them in shared memory
                setattr(ly, f"{name}_lo", buf(f"{name}_lo{j}", rows, cols) if name in ("w", "wt") else None)
        self._net = net
        self._dataset = None  # (data [N, d_in], weights [N]) resident on the device
        self._ctl_f64 = self._ctl[: (_ct.sizeof(_VkCtl) // 8) * 8].view(_torch.float64)
        self._ctl_i64 = self._ctl[: (_ct.sizeof(_VkCtl) // 8) * 8].view(_torch.int64)
        self._ctl_i32 = self._ctl[: (_ct.sizeof(_VkCtl) // 4) * 4].view(_torch.int32)
        self._reset_optimizer()
        seed64 = (self._seed * 0x9E3779B97F4A7C15 + 0x1234567) & 0x7FFFFFFFFFFFFFFF
        self._ctl_i64[_VkCtl.seed.offset // 8] = seed64
        self._graphs = {}
        self._dp_group = None
        self._use_graphs = True

    def _stream(self) -> int:
        return _torch.cuda.current_stream().cuda_stream

    def _ensure_capacity(self, rows: int) -> None:
        """Grow the activation workspaces to hold ``rows`` batch rows (the reference has no batch cap:
        ``-t 1024`` with four batchsteps reaches 16384).  Parameters and BatchNorm buffers are carried over;
        the optimiser state is reset, so this is only called before training starts."""
        if rows <= self._net.bmax:
            return
        self._bmax = (int(rows) + 127) // 128 * 128
        dataset, group, use_graphs = self._dataset, self._dp_group, self._use_graphs
        seed = int(self._ctl_i64[_VkCtl.seed.offset // 8].item())  # carries the per-rank perturbation
        self._build_device_state()  # copies the current parameter values into the new arena
        self._dp_group, self._use_graphs = group, use_graphs
        self._ctl_i64[_VkCtl.seed.offset // 8] = seed
        if dataset is not None:
            self._dataset = dataset
            self._net.data, self._net.weights, self._net.n_rows = dataset[1].data_ptr(), dataset[2].data_ptr(), len(dataset[2])

    def _reset_optimizer(self) -> None:
        "A fresh DAdaptAdam(params, decouple=True) (vamb/encode.py:578): zero state, d = 1e-6."
        for t in (self._exp_avg, self._exp_avg_sq, self._s):
            t.zero_()
        self._ctl_f64[_VkCtl.d.offset // 8] = 1e-6
        self._ctl_f64[_VkCtl.num_w.offset // 8] = 0.0
        self._reset_loss_sums()

    def _reset_loss_sums(self) -> None:
        o = _VkCtl.loss_sums.offset // 8
        self._ctl_f64[o:o + 5] = 0.0
        self._ctl_i64[_VkCtl.n_loss_steps.offset // 8] = 0

    def _read_loss_sums(self):
        o = _VkCtl.loss_sums.offset // 8
        sums = self._ctl_f64[o:o + 5].cpu().tolist()
        n = int(self._ctl_i64[_VkCtl.n_loss_steps.offset // 8].item())
        return sums, n

    @property
    def dadapt_d(self) -> float:
        "Current D-Adaptation distance estimate (``optimizer.param_groups[0]['d']`` in the reference)."
        return float(self._ctl_f64[_VkCtl.d.offset // 8].item())

    def _bind_dataset(self, tensors) -> int:
        """Upload (depths, tnf, abundance, weights) once: [N, S | 103 | 1] rows + weights."""
        depths, tnf, ab, w = tensors
        # the cache is keyed on the source tensors themselves (kept alive here, so their addresses cannot be
        # recycled) and their in-place version counters, not on raw addresses
        src = (depths, tnf, ab, w)
        key = tuple(t._version for t in src)
        if (self._dataset is not None and all(a is b for a, b in zip(self._dataset[3], src))
                and self._dataset[0] == key):
            return len(depths)
        dev = self._arena.device
        n = len(depths)
        data = _torch.zeros((n, self._net.data_ld), dtype=_torch.float32, device=dev)
        s = self.nsamples
        data[:, :s] = depths.to(dev, non_blocking=True)
        data[:, s:s + self.ntnf] = tnf.to(dev, non_blocking=True)
        data[:, s + self.ntnf:s + self.ntnf + 1] = ab.reshape(n, 1).to(dev, non_blocking=True)
        weights = w.reshape(n).to(dev).contiguous()
        self._dataset = (key, data, weights, src)
        self._net.data, self._net.weights, self._net.n_rows = data.data_ptr(), weights.data_ptr(), n
        self._graphs = {}
        return n

    # ------------------------------------------------------------------ reference API
    # Subclass contract (SURVEY 8b): the TaxVamb encoders subclass VAE and call ``self._encode``,
    # ``self.reparameterize`` and ``self._decode`` on their OWN concatenated inputs, inside their own autograd
    # training loops (vamb/semisupervised_encode.py:189, 438).  These three methods are therefore ordinary
    # differentiable module code over the registered layers -- whose parameters are views of the arena the kernels
    # train, so both routes always see the same weights.  The hot path (trainmodel / encode) never goes through them.
    def _encode(self, tensor: Tensor) -> Tensor:
        "vamb/encode.py:259-273: BatchNorm(Dropout(LeakyReLU(Linear))) per hidden layer, then ``mu``."
        tensor = tensor.to(self._arena.device)
        for encoderlayer, encodernorm in zip(self.encoderlayers, self.encodernorms):
            tensor = encodernorm(self.dropoutlayer(self.relu(encoderlayer(tensor))))
        return self.mu(tensor)

    def reparameterize(self, mu: Tensor) -> Tensor:
        "vamb/encode.py:276-286 (noise from the global torch CPU generator, moved to the device, as in the reference)."
        epsilon = _torch.randn(mu.size(0), mu.size(1)).to(mu.device)
        epsilon.requires_grad = True
        return mu + epsilon

    def _decode(self, tensor: Tensor) -> tuple[Tensor, Tensor, Tensor]:
        "vamb/encode.py:288-304: decoder blocks, output layer, softmax over the first ``nsamples`` outputs."
        tensor = tensor.to(self._arena.device)
        for decoderlayer, decodernorm in zip(self.decoderlayers, self.decodernorms):
            tensor = decodernorm(self.dropoutlayer(self.relu(decoderlayer(tensor))))
        reconstruction = self.outputlayer(tensor)
        depths_out = _softmax(reconstruction.narrow(1, 0, self.nsamples), dim=1)
        tnf_out = reconstruction.narrow(1, self.nsamples, self.ntnf)
        abundance_out = reconstruction.narrow(1, self.nsamples + self.ntnf, 1)
        return depths_out, tnf_out, abundance_out

    def forward(self, depths: Tensor, tnf: Tensor, abundance: Tensor) -> tuple[Tensor, Tensor, Tensor, Tensor]:
        """(depths_out, tnf_out, abundance_out, mu) for explicit input tensors (vamb/encode.py:306-314), in train or
        eval mode according to ``self.training``.

        In training mode with autograd enabled the call goes through the differentiable module route
        (``_encode`` -> ``reparameterize`` -> ``_decode``) so that ``calc_loss(...)[0].backward()`` works for callers
        that run their own optimiser; otherwise (eval mode or ``torch.no_grad()``) it runs the fused kernels and the
        outputs carry no graph.  Outputs are returned on the device of the inputs."""
        if self.training and _torch.is_grad_enabled():
            src = depths.device
            tensor = _torch.cat((depths, tnf, abundance.reshape(len(depths), -1)), 1)
            mu = self._encode(tensor)
            d_out, t_out, a_out = self._decode(self.reparameterize(mu))
            return d_out.to(src), t_out.to(src), a_out.to(src), mu.to(src)
        out = self._forward_tensors(depths, tnf, abundance)
        return out[0], out[1], out[2], out[3]

    def _forward_tensors(self, depths, tnf, abundance, inject=None, training=None):
        dev = self._arena.device
        b = len(depths)
        if b > self._net.bmax:
            raise ValueError(f"at most {self._net.bmax} rows per forward call")
        src_dev = depths.device
        pad = _torch.zeros((b, self._net.data_ld - self._net.d_in), dtype=_torch.float32, device=dev)
        data = _torch.cat((depths.to(dev), tnf.to(dev), abundance.reshape(b, -1).to(dev), pad), 1).float().contiguous()
        weights = _torch.ones(b, dtype=_torch.float32, device=dev)
        tmp = _VkVae.from_buffer_copy(self._net)
        tmp.data, tmp.weights, tmp.n_rows = data.data_ptr(), weights.data_ptr(), b
        training = self.training if training is None else training
        if not training:
            _lib.check(_L.vk_vae_prepare_eval(_ct.byref(tmp), self._stream()))
        _lib.check(_L.vk_vae_forward(_ct.byref(tmp), 0, b, 1 if training else 0, 0,
                                     _ct.byref(inject) if inject is not None else None, self._stream()))
        nl = tmp.n_layers
        rec = self._keep[f"act{nl - 1}"][:b].clone()
        mu = self._keep[f"act{len(self.nhiddens)}"][:b].clone()
        s = self.nsamples
        depths_out = _softmax(rec[:, :s], dim=1)
        tnf_out = rec[:, s:s + self.ntnf]
        ab_out = rec[:, s + self.ntnf:]
        _torch.cuda.current_stream().synchronize()
        return tuple(t.to(src_dev) for t in (depths_out, tnf_out, ab_out, mu))

    def calc_loss(self, depths_in, depths_out, tnf_in, tnf_out, abundance_in, abundance_out, mu, weights):
        """The composite loss as a plain tensor expression (vamb/encode.py:316-357), including
        its [B] x [B, 1] broadcast: loss = mean_j(l_j) * mean_i(w_i)."""
        ab_sse = (abundance_out - abundance_in).pow(2).sum(dim=1)
        ce = -((depths_out + 1e-9).log() * depths_in).sum(dim=1)
        sse = (tnf_out - tnf_in).pow(2).sum(dim=1)
        kld = 0.5 * (mu.pow(2)).sum(dim=1)
        net = self._net
        weighed_ab, weighed_ce = ab_sse * net.ab_w, ce * net.ce_w
        weighed_sse, weighed_kld = sse * net.sse_w, kld * net.kld_w
        loss = ((weighed_ce + weighed_ab + weighed_sse) + weighed_kld) * weights
        return (loss.mean(), weighed_ab.mean(), weighed_ce.mean(), weighed_sse.mean(), weighed_kld.mean())

    # ------------------------------------------------------------------ test / parity hooks
    def _hidden_layer_ids(self) -> list:
        L = len(self.nhiddens)
        return list(range(L)) + [L + 1 + i for i in range(L)]

    def _step_injected(self, tensors, batch_idx, eps=None, keeps=None, optimize=True):
        """One training step on explicit rows with host-supplied noise (parity tests):
        ``eps`` [B, nlatent], ``keeps`` = one [B, n_out] 0/1 array per hidden block in forward
        order.  Returns the five per-step loss values (loss, ab, ce, sse, kld)."""
        self._bind_dataset(tensors)
        self.train()
        dev = self._arena.device
        hold = []
        inj = _VkInject()
        idx = _torch.as_tensor(_np.asarray(batch_idx), dtype=_torch.int64).to(dev)
        hold.append(idx)
        inj.batch_idx = idx.data_ptr()
        if eps is not None:
            e = _torch.as_tensor(_np.asarray(eps), dtype=_torch.float32).to(dev).contiguous()
            hold.append(e)
            inj.eps = e.data_ptr()
        if keeps is not None:
            for j, k in zip(self._hidden_layer_ids(), keeps):
                if k is None:
                    continue
                t = _torch.as_tensor(_np.asarray(k), dtype=_torch.uint8).to(dev).contiguous()
                hold.append(t)
                inj.keep[j] = t.data_ptr()
        self._reset_loss_sums()
        fn = _L.vk_vae_train_step if optimize else _L.vk_vae_grad_step
        _lib.check(fn(_ct.byref(self._net), len(idx), _ct.byref(inj), self._stream()))
        _torch.cuda.current_stream().synchronize()
        sums, _ = self._read_loss_sums()
        return sums

    def _profile_step(self, batch: int) -> dict:
        """Per-launch device times (ms) of one training step at ``batch`` (dataset must be bound).
        ``fwd`` / ``bwd`` are per layer (backward: last layer first); ``prep`` = operand staging."""
        cap = 96
        ms = (_ct.c_float * cap)()
        kinds = (_ct.c_int * cap)()
        n = _ct.c_int(0)
        _lib.check(_L.vk_vae_profile_step(_ct.byref(self._net), batch, None, ms, kinds, cap, _ct.byref(n), self._stream()))
        out = {"batch_rows": 0.0, "fwd": [], "loss": 0.0, "bwd": [], "dadapt": 0.0, "prep": 0.0, "n_launches": n.value}
        for i in range(n.value):
            k, v = kinds[i], float(ms[i])
            if k == 1:
                out["fwd"].append(v)
            elif k == 3:
                out["bwd"].append(v)
            else:
                out[{0: "batch_rows", 2: "loss", 4: "dadapt", 5: "prep"}[k]] += v
        return out

    def _grad_dict(self) -> dict:
        "Gradients of the last step, keyed like ``named_parameters()``."
        return {name: self._grads[off:off + p.numel()].view_as(p).clone()
                for (name, p), off in ((kv, self._offsets[kv[0]]) for kv in self.named_parameters())}

    def _encode_device(self, tensors, mask_bits: int = 12) -> _np.ndarray:
        n = self._bind_dataset(tensors)
        self.eval()
        out = _torch.empty((n, self.nlatent), dtype=_torch.float32, device=self._arena.device)
        _lib.check(_L.vk_vae_encode(_ct.byref(self._net), 0, n, mask_bits, out.data_ptr(), self._stream()))
        return out.cpu().numpy()

    # ------------------------------------------------------------------ training
    def _one_step(self, batch: int) -> None:
        if self._dp_group is None:
            _lib.check(_L.vk_vae_train_step(_ct.byref(self._net), batch, None, self._stream()))
        else:
            # row-sharded data parallelism (SURVEY 8e): local gradients, ONE all-reduce (average) of the
            # packed gradient arena over NCCL / NVLink, then the identical optimiser step on every rank
            _lib.check(_L.vk_vae_grad_step(_ct.byref(self._net), batch, None, self._stream()))
            _par.allreduce_mean_(self._grads, self._dp_group)
            _lib.check(_L.vk_vae_dadapt_step(_ct.byref(self._net), self._stream()))

    def _graph_for(self, batch: int, chunk: int):
        """The captured graph of ``chunk`` optimiser steps at ``batch`` (None when capture is unavailable).
        Capture executes nothing; the steps run at replay."""
        key = (batch, chunk)
        g = self._graphs.get(key)
        if g is not None or not self._use_graphs:
            return g
        g = _torch.cuda.CUDAGraph()
        try:
            with _torch.cuda.graph(g):
                for _ in range(chunk):
                    self._one_step(batch)
            self._graphs[key] = g
            return g
        except Exception:
            if self._dp_group is None:
                raise
            self._use_graphs = False  # this NCCL build cannot be captured: run the steps eagerly
            _torch.cuda.synchronize()
            return None

    def _run_steps(self, batch: int, nsteps: int) -> None:
        """``nsteps`` optimiser steps at batch size ``batch`` through replayed CUDA graphs: chunks of 128, then
        16, then 4 steps (short epochs -- row shards, large batches -- still run from graphs), the rest eagerly."""
        done = 0
        if self._use_graphs and nsteps > _GRAPH_CHUNKS[-1]:
            if ("warm", batch) not in self._graphs:
                self._one_step(batch)  # first use of this batch size: one step outside capture
                done += 1
                _torch.cuda.current_stream().synchronize()
                self._graphs[("warm", batch)] = True
            for chunk in _GRAPH_CHUNKS:
                if nsteps - done < chunk:
                    continue
                g = self._graph_for(batch, chunk)
                while g is not None and nsteps - done >= chunk:
                    g.replay()
                    done += chunk
        for _ in range(nsteps - done):
            self._one_step(batch)

    # ------------------------------------------------------------------ multi-GPU (row-sharded data parallel)
    def enable_data_parallel(self, group=None) -> None:
        """Train this replica as one rank of a data-parallel group: every rank binds its own row shard of
        the dataset; each optimiser step all-reduces (averages) the gradient arena once.  Parameters start
        identical (same CPU seed) and stay identical; dropout / noise / shuffling streams are per rank;
        BatchNorm batch statistics are per GPU and the running statistics are averaged before
        ``encode`` / ``save`` (``sync_running_stats``).  ``torch.distributed`` must be initialised (NCCL)."""
        if not _dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised")
        self._dp_group = group if group is not None else _dist.group.WORLD
        rank = _dist.get_rank(self._dp_group)
        so = _VkCtl.seed.offset // 8
        self._ctl_i64[so] = int(self._ctl_i64[so].item()) ^ ((rank + 1) * 0x2545F4914F6CDD1D & 0x7FFFFFFFFFFFFFFF)
        self._graphs = {}

    def sync_running_stats(self) -> None:
        "Average the BatchNorm running statistics over the data-parallel group."
        if self._dp_group is None:
            return
        _par.average_running_stats_(list(self.encodernorms) + list(self.decodernorms), self._dp_group)

    def _run_epoch_strict(self, n_seq: int, batch: int, drop_last: bool) -> None:
        dev = self._arena.device
        for idx, eps, keeps in reference_epoch_noise(n_seq, batch, drop_last, self.nhiddens, self.nlatent, self.dropout):
            hold = [idx.to(dev), eps.to(dev).contiguous()]
            inj = _VkInject()
            inj.batch_idx, inj.eps = hold[0].data_ptr(), hold[1].data_ptr()
            for j, k in zip(self._hidden_layer_ids(), keeps):
                if k is not None:
                    t = k.to(_torch.uint8).to(dev).contiguous()
                    hold.append(t)
                    inj.keep[j] = t.data_ptr()
            _lib.check(_L.vk_vae_train_step(_ct.byref(self._net), len(idx), _ct.byref(inj), self._stream()))
            _torch.cuda.current_stream().synchronize()  # `hold` must outlive the step

    def trainepoch(self, data_loader: _DataLoader, epoch: int, optimizer, batchsteps: list[int]) -> _DataLoader:
        """One pass over the data (vamb/encode.py:359-440).  ``optimizer`` is accepted for
        signature compatibility; the D-Adaptation state lives on the device."""
        n_seq = len(data_loader.dataset.tensors[0])
        if n_seq < 2:
            raise ValueError(
                "Cannot train on a dataset with fewer than 2 sequences, but got "
                f"{n_seq} sequences. "
                "If you are trying to fit a DL model to this few sequences, "
                "something probably went wrong in your pipeline."
            )
        self.train()
        if epoch in batchsteps:
            data_loader = set_batchsize(data_loader, data_loader.batch_size * 2, n_seq)
        self._bind_dataset(data_loader.dataset.tensors)
        batch = data_loader.batch_size if n_seq > data_loader.batch_size else n_seq
        if batch > self._net.bmax:
            raise ValueError(
                f"batch size {batch} exceeds the workspace capacity {self._net.bmax}: call trainmodel(), which sizes the "
                "workspaces for the whole schedule before the first epoch"
            )
        nsteps = len(data_loader)  # N // batch with drop_last, else 1
        if self._dp_group is not None:
            nsteps = _par.agree_min(nsteps, self._dp_group, self._arena.device)  # every rank takes the same steps

        self._ctl_i32[_VkCtl.epoch.offset // 4] = int(epoch)
        so = _VkCtl.step.offset // 8
        self._ctl_i64[_VkCtl.epoch_step0.offset // 8] = self._ctl_i64[so]
        self._reset_loss_sums()
        if self.strict_rng and self._dp_group is None:
            self._run_epoch_strict(n_seq, batch, bool(data_loader.drop_last))
        else:
            self._run_steps(batch, nsteps)
        sums, n = self._read_loss_sums()  # the only host synchronisation of the epoch
        n = max(n, 1)
        logger.info(
            "\t\tEpoch: {:>3}  Loss: {:.5e}  CE: {:.5e}  AB: {:.5e}  SSE: {:.5e}  KLD: {:.5e}  Batchsize: {:>4}".format(
                epoch + 1, sums[0] / n, sums[2] / n, sums[1] / n, sums[3] / n, sums[4] / n, data_loader.batch_size,
            )
        )
        self._last_epoch_losses = tuple(x / n for x in sums)
        self.eval()
        return data_loader

    def encode(self, data_loader) -> _np.ndarray:
        """Encode a data loader to a latent representation with VAE

        Input: data_loader: As generated by train_vae

        Output: A (n_contigs x n_latent) Numpy array of latent repr.
        """
        self.eval()
        self.sync_running_stats()
        n = self._bind_dataset(data_loader.dataset.tensors)
        dev = self._arena.device
        out = _torch.empty((n, self.nlatent), dtype=_torch.float32, device=dev)
        _lib.check(_L.vk_vae_encode(_ct.byref(self._net), 0, n, 12, out.data_ptr(), self._stream()))
        # a NumPy array that owns its memory, so that callers may resize it (vamb/encode.py:459-462)
        latent = _np.empty((n, self.nlatent), dtype=_np.float32)
        _torch.from_numpy(latent).copy_(out)
        return latent

    def save(self, filehandle):
        """Saves the VAE to a path or binary opened file. Load with VAE.load

        Input: Path or binary opened filehandle
        Output: None
        """
        self.sync_running_stats()  # data-parallel: BatchNorm running statistics are per GPU until averaged
        state = {
            "nsamples": self.nsamples,
            "alpha": self.alpha,
            "beta": self.beta,
            "dropout": self.dropout,
            "nhiddens": self.nhiddens,
            "nlatent": self.nlatent,
            "state": {k: v.detach().cpu().clone() for k, v in self.state_dict().items()},
        }
        _torch.save(state, filehandle)

    @classmethod
    def load(cls, path: Union[IO[bytes], str], cuda: bool = False, evaluate: bool = True):
        """Instantiates a VAE from a model file.

        Inputs:
            path: Path to model file as created by functions VAE.save or
                  VAE.trainmodel.
            cuda: accepted for API compatibility (the network always lives on the GPU)
            evaluate: Return network in evaluation mode [True]

        Output: VAE with weights and parameters matching the saved network.
        """
        dictionary = _torch.load(path, map_location=lambda storage, loc: storage, weights_only=True)
        vae = cls(
            dictionary["nsamples"], dictionary["nhiddens"], dictionary["nlatent"], dictionary["alpha"],
            dictionary["beta"], dictionary["dropout"], cuda,
        )
        vae.load_state_dict(dictionary["state"])  # copies into the arena views in place
        if evaluate:
            vae.eval()
        return vae

    def trainmodel(
        self,
        dataloader: _DataLoader,
        nepochs: int = 500,
        batchsteps: Optional[list[int]] = [25, 75, 150, 300],
        modelfile: Union[None, str, Path, IO[bytes]] = None,
    ):
        """Train the autoencoder from depths array and tnf array.

        Inputs:
            dataloader: DataLoader made by make_dataloader
            nepochs: Train for this many epochs before encoding [500]
            batchsteps: None or double batchsize at these epochs [25, 75, 150, 300]
            modelfile: Save models to this file if not None [None]

        Output: None
        """
        if nepochs < 1:
            raise ValueError(f"Minimum 1 epoch, not {nepochs}")
        if batchsteps is None:
            batchsteps_set: set[int] = set()
        else:
            batchsteps = list(batchsteps)
            if not all(isinstance(i, int) for i in batchsteps):
                raise ValueError("All elements of batchsteps must be integers")
            if max(batchsteps, default=0) >= nepochs:
                raise ValueError("Max batchsteps must not equal or exceed nepochs")
            batchsteps_set = set(batchsteps)

        ncontigs, nsamples = dataloader.dataset.tensors[0].shape
        # the largest batch the schedule will reach must fit the workspaces BEFORE any epoch runs (the batch
        # doubles at every batchstep, vamb/encode.py:383-388); grow them now instead of failing at epoch 300
        self._ensure_capacity(min(ncontigs, dataloader.batch_size * 2 ** len(batchsteps_set)))
        self._reset_optimizer()  # the reference builds a new DAdaptAdam per trainmodel call

        logger.info("\tNetwork properties:")
        logger.info(f"\t    CUDA: {self.usecuda}")
        logger.info(f"\t    Alpha: {self.alpha}")
        logger.info(f"\t    Beta: {self.beta}")
        logger.info(f"\t    Dropout: {self.dropout}")
        logger.info(f"\t    N hidden: {', '.join(map(str, self.nhiddens))}")
        logger.info(f"\t    N latent: {self.nlatent}")
        logger.info("\tTraining properties:")
        logger.info(f"\t    N epochs: {nepochs}")
        logger.info(f"\t    Starting batch size: {dataloader.batch_size}")
        batchsteps_string = ", ".join(map(str, sorted(batchsteps_set))) if batchsteps_set else "None"
        logger.info(f"\t    Batchsteps: {batchsteps_string}")
        logger.info(f"\t    N sequences: {ncontigs}")
        logger.info(f"\t    N samples: {nsamples}")

        for epoch in range(nepochs):
            dataloader = self.trainepoch(dataloader, epoch, None, sorted(batchsteps_set))

        if modelfile is not None:
            try:
                self.save(modelfile)
            except Exception:
                pass
        return None
