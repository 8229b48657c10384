"""TEST INFRASTRUCTURE -- import the UNMODIFIED reference hot-path files.

Loads vamb/{vambtools,encode,cluster}.py of a checkout of RasmussenLab/vamb
(named by the environment variable VAMB_REFERENCE_ROOT) by file path under a
stub ``vamb`` package (the real ``vamb/__init__.py`` needs an installed dist and
compiled wheels), after injecting two shims into ``sys.modules``:
``vambcore`` (oracle/vambcore_shim.py) and ``dadaptation`` (oracle/dadapt.py).

Only the oracle/make_golden*.py scripts use it: the tests compare with what
those scripts recorded under tests/golden/.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("VAMB_REFERENCE_ROOT", "")
_PKG = "vamb"
_cached = None


def available() -> bool:
    return bool(REFERENCE_ROOT) and os.path.isfile(os.path.join(REFERENCE_ROOT, "vamb", "cluster.py"))


def load():
    """Return a namespace with ``.vambtools``, ``.encode``, ``.cluster`` = the reference modules."""
    global _cached
    if _cached is not None:
        return _cached
    if not available():
        raise FileNotFoundError(f"set VAMB_REFERENCE_ROOT to a checkout of RasmussenLab/vamb (now {REFERENCE_ROOT!r})")

    from . import dadapt, vambcore_shim

    saved = {k: sys.modules.get(k) for k in (_PKG, "vambcore", "dadaptation")}
    sys.modules["vambcore"] = vambcore_shim
    sys.modules["dadaptation"] = dadapt
    pkg = types.ModuleType(_PKG)
    pkg.__path__ = []  # mark as package
    sys.modules[_PKG] = pkg
    mods = {}
    try:
        for name in ("vambtools", "encode", "cluster"):
            full = f"{_PKG}.{name}"
            spec = importlib.util.spec_from_file_location(
                full, os.path.join(REFERENCE_ROOT, "vamb", f"{name}.py")
            )
            mod = importlib.util.module_from_spec(spec)
            sys.modules[full] = mod
            spec.loader.exec_module(mod)
            setattr(pkg, name, mod)
            mods[name] = mod
    finally:
        # leave the reference modules reachable only through the returned namespace,
        # so that the product package can never pick them up by accident
        for name in ("vambtools", "encode", "cluster"):
            sys.modules.pop(f"{_PKG}.{name}", None)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    # quiet the reference's loguru chatter (one line per epoch)
    try:
        from loguru import logger

        logger.disable("vamb")
    except Exception:
        pass
    _cached = types.SimpleNamespace(**mods)
    return _cached
