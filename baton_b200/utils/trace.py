"""In-graph kernel timeline.

CUDA events cannot see inside a replayed CUDA graph and ``ncu`` serialises launches with cold caches, so neither
tells where a captured local-SGD step (one graph launch = thousands of kernels) spends its time.  A trace build
of the extension (``BATON_BUILD_TRACE=1 python -m baton_b200.build_ext`` -> ``_C_trace.so``, loaded when
``BATON_TRACE=1``) makes CTA 0 of every kernel stamp ``%globaltimer`` when it becomes resident and again when its
programmatic dependencies have completed (``csrc/pdl.cuh``).  The difference between consecutive "dependencies
done" stamps is the critical-path time of the earlier kernel *as it ran inside the graph*.

    tr = KernelTrace(capacity=1 << 16); tr.start(); graph.replay(); torch.cuda.synchronize()
    for row in tr.summary(): print(row)

The reference has no tracing at all (SURVEY.md section 5); this is its "tracing / profiling" subsystem,
together with ``metrics.phase`` (NVTX ranges + CUDA-event timers).
"""
from __future__ import annotations

import collections
import os
import re
from typing import Callable, Dict, List, Tuple

import torch

_TUS = ["?", "gemm_wgmma", "gemm_fp8", "quant", "attention", "im2col_tma", "gemm_simt", "fedavg", "elementwise",
        "conv", "norm", "loss", "conv_halo", "dropout"]
_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "csrc")
_NAME_CACHE: Dict[int, str] = {}


POINT_BASE = 5_000_000_000      # TRACE_POINT() stamps (intra-kernel): tag = POINT_BASE + tu * 100000 + line


def point_label(tag: int) -> str:
    """Label of an intra-kernel stamp = the comment on its source line."""
    tu, line = divmod(int(tag) - POINT_BASE, 100000)
    try:
        with open(os.path.join(_CSRC, _TUS[tu] + ".cu")) as f:
            src = f.readlines()
        text = src[line - 1]
        return text.split("//", 1)[1].strip() if "//" in text else "{}:{}".format(_TUS[tu], line)
    except (OSError, IndexError):
        return "point {}:{}".format(tu, line)


def kernel_name(tag: int) -> str:
    """``tag = tu * 100000 + line`` -> name of the ``__global__`` function enclosing that source line."""
    tag = abs(int(tag))
    if tag in _NAME_CACHE:
        return _NAME_CACHE[tag]
    tu, line = divmod(tag, 100000)
    name = "{}:{}".format(_TUS[tu] if tu < len(_TUS) else tu, line)
    try:
        with open(os.path.join(_CSRC, _TUS[tu] + ".cu")) as f:
            src = f.readlines()
        for i in range(min(line, len(src)) - 1, -1, -1):
            if "__global__" in src[i]:
                m = re.search(r"(\w+)\s*\(", " ".join(s.strip() for s in src[i:i + 4]).split("__global__", 1)[1]
                              .replace("__launch_bounds__", " ").replace("__cluster_dims__", " "))
                # skip attribute argument lists such as (GEMM_THREADS, 1)
                cands = re.findall(r"([A-Za-z_]\w*)\s*\(", " ".join(s.strip() for s in src[i:i + 4]))
                cands = [c for c in cands if c not in ("__launch_bounds__", "__cluster_dims__")]
                if cands:
                    name = cands[0]
                elif m:
                    name = m.group(1)
                break
    except OSError:
        pass
    _NAME_CACHE[tag] = name
    return name


def timeline_rows(records: List[Tuple[int, int]], name: Callable[[int], str] = kernel_name) -> List[dict]:
    """Rows of :meth:`KernelTrace.timeline` from time-sorted ``(t_ns, tag)`` records.  The "resident" stamp
    (griddep_launch_dependents) and the "dependencies done" stamp (griddep_wait) of one launch sit on different source
    lines, so their tags differ: they are paired per kernel NAME, first resident stamp to first dependencies-done stamp."""
    resident = collections.defaultdict(collections.deque)
    rows = []
    for t, tag in records:
        if abs(tag) >= POINT_BASE:
            continue
        k = name(tag)
        if tag < 0:
            resident[k].append(t)
        else:
            pre = resident[k].popleft() if resident[k] else t
            rows.append({"t_ns": t, "tag": tag, "name": k, "early_ns": t - pre})
    for a, b in zip(rows, rows[1:]):
        a["slot_ns"] = b["t_ns"] - a["t_ns"]
    if rows:
        rows[-1]["slot_ns"] = 0
    return rows


class KernelTrace:
    def __init__(self, capacity: int = 1 << 16, device=None):
        from ..ops._ext import load
        self.C = load()
        self.device = torch.device(device or "cuda:0")
        self.capacity = capacity
        self.buf = torch.zeros(2 + 2 * capacity, dtype=torch.int64, device=self.device)
        self.buf[1] = capacity
        self.enabled = False

    def start(self) -> bool:
        self.buf[0] = 0
        self.enabled = bool(self.C.trace_set(self.buf))
        return self.enabled

    def stop(self) -> None:
        torch.cuda.synchronize(self.device)
        self.C.trace_set(None)

    def records(self) -> List[Tuple[int, int]]:
        """``[(t_ns, tag)]`` sorted by time (tag < 0: CTA 0 resident, tag > 0: dependencies complete)."""
        torch.cuda.synchronize(self.device)
        host = self.buf.cpu()
        n = min(int(host[0]), self.capacity)
        rec = host[2: 2 + 2 * n].view(n, 2).tolist()
        rec.sort()
        return [(int(t), int(tag)) for t, tag in rec]

    def timeline(self) -> List[dict]:
        """One row per kernel: start of its critical-path slot (dependencies done), the slot length (until the next
        kernel's dependencies are done) and how long before that its first CTA was already resident (PDL overlap)."""
        return timeline_rows(self.records())

    def points(self) -> List[Tuple[int, str]]:
        """``[(t_ns, label)]`` of everything in time order: kernel starts (``> name``) and intra-kernel TRACE_POINTs."""
        out = []
        for t, tag in self.records():
            if tag >= POINT_BASE:
                out.append((t, "    . " + point_label(tag)))
            elif tag > 0:
                out.append((t, "> " + kernel_name(tag)))
            else:
                out.append((t, "  (resident) " + kernel_name(tag)))
        return out

    def summary(self, skip_first: int = 0) -> List[str]:
        rows = self.timeline()[skip_first:]
        tot = collections.defaultdict(float)
        cnt = collections.Counter()
        early = collections.defaultdict(float)
        for r in rows:
            tot[r["name"]] += r["slot_ns"]
            cnt[r["name"]] += 1
            early[r["name"]] += r["early_ns"]
        total = sum(tot.values()) or 1.0
        out = ["kernels {}  critical-path total {:.1f} us".format(len(rows), total / 1e3)]
        for n, t in sorted(tot.items(), key=lambda kv: -kv[1]):
            out.append("{:9.1f} us {:5.1f}%  n={:5d}  avg slot {:6.2f} us  avg resident-before-deps {:5.2f} us  {}".format(
                t / 1e3, 100 * t / total, cnt[n], t / cnt[n] / 1e3, early[n] / cnt[n] / 1e3, n))
        return out
