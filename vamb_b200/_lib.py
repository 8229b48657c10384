"""ctypes binding of the C ABI declared in include/vamb_b200.h.

There is NO CPU fallback: importing this module without a loadable ``_vk.so`` raises, and
``require_device()`` raises unless ``cuda:0`` is an sm_90 (H100) GPU.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_int64, c_uint8, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
# VAMB_B200_SO selects another build of the same library (tools/step_timeline.py uses the stamped one)
_SO = os.environ.get("VAMB_B200_SO") or os.path.join(_HERE, "_vk.so")

VK_ABI_VERSION = 2
VK_NBINS = 60
VK_MAX_CAND = 32
VK_LIST_CAND = 64
VK_EVAL_SUBS = 4
VK_EVAL_SCRATCH_U64 = VK_EVAL_SUBS * VK_LIST_CAND * 16  # device accumulator words of vk_eval_candidates_lists
VK_PROBE_INLINE = 2040

# byte offsets inside vk_probe_header (include/vamb_b200.h)
HDR_DENSITY_LO = 0
HDR_DENSITY_HI = 8
HDR_HIST = 16
HDR_NWITHIN = 16 + 8 * VK_NBINS
HDR_NLT = HDR_NWITHIN + 4
HDR_NNL = HDR_NWITHIN + 8
HDR_RANK = HDR_NWITHIN + 12
HDR_WITHIN = HDR_NWITHIN + 16
HDR_SIZE = HDR_WITHIN + 4 * VK_PROBE_INLINE


class VkError(RuntimeError):
    pass


def _load() -> ctypes.CDLL:
    if not os.path.isfile(_SO):
        # the extension is built in-tree by __graft_entry__.build(); try once here so that a
        # fresh checkout works, but never fall back to anything else.
        from . import build as _build

        _build.build()
    lib = ctypes.CDLL(_SO)
    lib.vk_last_error.restype = c_char_p
    lib.vk_abi_version.restype = c_int
    if lib.vk_abi_version() != VK_ABI_VERSION:
        raise ImportError(f"{_SO}: ABI version {lib.vk_abi_version()} != {VK_ABI_VERSION}; rebuild")
    return lib


lib = _load()

_p = c_void_p  # device / pinned pointers are passed as integers (tensor.data_ptr())

_SIGNATURES = {
    "vk_check_device": [],
    "vk_normalize_rows": [_p, c_int64, c_int, _p],
    "vk_check_normalized": [_p, c_int64, c_int, c_float, _p, _p],
    "vk_probe": [_p, _p, _p, c_int64, c_int, c_int64, c_float, _p, _p, _p, _p, _p, _p],
    "vk_probe_sync": [_p, _p, _p, c_int64, c_int, c_int64, c_float, _p, _p, _p, _p, _p, _p, _p],
    "vk_probe_mapped": [_p, _p, _p, c_int64, c_int, c_int64, c_float, _p, _p, _p, _p, _p, _p, _p, _p, c_int32, _p, _p],
    "vk_eval_candidates_sync": [_p, _p, c_int, _p, _p, c_int32, c_float, POINTER(c_int32), c_int, _p, _p, _p],
    "vk_eval_candidates_mapped": [_p, _p, c_int, _p, _p, c_int32, c_float, POINTER(c_int32), c_int, _p, _p, _p, _p,
                                  c_int32, _p],
    "vk_eval_candidates_lists": [_p, _p, c_int, _p, _p, c_int32, c_float, POINTER(c_int32), c_int, c_int32, c_uint64, c_uint64,
                                 _p, _p, _p, _p,
                                 c_int32, _p, _p, c_int32, _p],
    "vk_select_members_sync": [_p, _p, c_int32, c_float, _p, _p, _p, _p, c_int32, _p],
    "vk_mask_clear": [_p, _p, c_int32, _p],
    "vk_compact_rows_sync": [_p, _p, _p, _p, c_int64, c_int, _p, _p, _p, _p, _p, POINTER(c_int64), _p],
    "vk_distances": [_p, c_int64, c_int, c_int64, _p, _p],
    "vk_tc_gemm_test": [_p, c_int, _p, _p, c_int, _p, c_int, c_int, c_int, c_int, c_int, c_int, _p],
    "vk_lane_major_index": [c_int, c_int, c_int],
    "vk_tnf_project": [_p, _p, _p, c_int64, c_int, _p],
}


def _bind():
    for name, argtypes in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = the .so does not export a declared symbol
        fn.argtypes = argtypes
        fn.restype = c_int


_bind()
lib.vk_lane_major_index.restype = c_int64


# bound (with argtypes) in vamb_b200/encode.py next to the ctypes mirrors of their structs
_VAE_SYMBOLS = [
    "vk_vae_sizeof", "vk_vae_train_step", "vk_vae_grad_step", "vk_vae_forward", "vk_vae_encode",
    "vk_vae_prepare_eval", "vk_vae_dadapt_step", "vk_vae_profile_step", "vk_vae_init_device",
    # bound in vamb_b200/_cluster_native.py
    "vk_cluster_create", "vk_cluster_next", "vk_cluster_next_block", "vk_cluster_stats", "vk_cluster_timing", "vk_cluster_destroy", "vk_cluster_rng_selftest", "vk_cluster_sizeof",
]
for _name in _VAE_SYMBOLS:
    getattr(lib, _name)  # AttributeError = stale .so


def declared_symbols() -> list:
    """Every entry point include/vamb_b200.h declares (checked by the CPU test-suite)."""
    return ["vk_last_error", "vk_abi_version"] + list(_SIGNATURES) + _VAE_SYMBOLS


def check(status: int) -> None:
    if status != 0:
        raise VkError(lib.vk_last_error().decode("utf-8", "replace"))


_device_ok = False


def require_device() -> None:
    """Fail loudly unless an H100 (sm_90) GPU and the CUDA extension are usable."""
    global _device_ok
    if _device_ok:
        return
    import torch

    if not torch.cuda.is_available():
        raise VkError(
            "vamb_b200 has no CPU path: a CUDA device (sm_90, H100) is required "
            "(torch.cuda.is_available() is False)"
        )
    check(lib.vk_check_device())
    _device_ok = True
