"""Loader for the in-tree sm_90a extension (``baton_b200/_C.so``).

The extension is the product: on a machine with a CUDA device every op in
``baton_b200.ops`` runs its hand-written kernel and a missing/unloadable
extension is a hard error (no silent eager fallback).  On a GPU-less host the
module still imports (``nvcc`` cross-compiles there) but is never called.

``load()`` returns a thin proxy that counts kernel launches per entry point
(``launch_counts()``); the counts taken while a CUDA graph is being captured are
what ``bench.py`` multiplies out to report ``gpu_launches``.
"""
from __future__ import annotations

import importlib
import os
from collections import Counter

_RAW = None
_PROXY = None
_COUNTS: Counter = Counter()

# entry points that enqueue more than one kernel/memset node
_EXTRA_NODES = {"colsum": 1}


class _Counting:
    """Attribute proxy over the pybind module: every call bumps a per-op counter."""

    def __init__(self, mod):
        object.__setattr__(self, "_mod", mod)
        object.__setattr__(self, "_cache", {})

    def __getattr__(self, name):
        cache = object.__getattribute__(self, "_cache")
        fn = cache.get(name)
        if fn is None:
            target = getattr(object.__getattribute__(self, "_mod"), name)
            if callable(target):
                def fn(*a, __t=target, __n=name, **k):
                    _COUNTS[__n] += 1
                    return __t(*a, **k)
            else:
                fn = target
            cache[name] = fn
        return fn


def load(build_if_missing: bool = False):
    global _RAW, _PROXY
    if _PROXY is not None:
        return _PROXY
    import torch  # noqa: F401  (libtorch must be loaded before the extension)
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = os.path.join(here, "_C.so")
    if not os.path.exists(so) and build_if_missing:
        from .. import build_ext
        build_ext.build()
    try:
        if os.environ.get("BATON_TRACE") == "1":
            # kernel-timeline build (BATON_BUILD_TRACE=1 python -m baton_b200.build_ext): same module, -DB200_TRACE
            from importlib import machinery, util
            path = os.path.join(here, "_C_trace.so")
            loader = machinery.ExtensionFileLoader("_C", path)
            spec = util.spec_from_file_location("_C", path, loader=loader)
            _RAW = util.module_from_spec(spec)
            loader.exec_module(_RAW)
        else:
            _RAW = importlib.import_module("baton_b200._C")
    except Exception as exc:  # pragma: no cover - exercised only on broken installs
        raise RuntimeError(
            "baton_b200._C (sm_90a kernels) is not available: {!r}. "
            "Run `python -m baton_b200.build_ext`.".format(exc)) from exc
    _PROXY = _Counting(_RAW)
    return _PROXY


def available() -> bool:
    try:
        load()
        return True
    except Exception:
        return False


def launch_counts() -> Counter:
    """Kernel launches issued through the extension since import, by entry point."""
    return Counter(_COUNTS)


def total_launches() -> int:
    return sum(v + _EXTRA_NODES.get(k, 0) * v for k, v in _COUNTS.items())
