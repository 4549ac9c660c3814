"""Structured per-round metrics and phase tracing.

The reference's observability is 23 ``print`` calls (e.g. manager.py:73,117,
131-132).  This module provides:

  * ``RoundMetrics`` -- an in-memory JSON-able log of round records (wall time,
    participants, samples, bytes moved, device-timed phases) and of evaluations of
    the global model, served by the manager at ``GET /{name}/metrics``;
  * ``phase`` -- a context manager that opens an NVTX range (when CUDA is
    present) and records host wall time, used around broadcast / local-train /
    upload-reduce;
  * ``DeviceTimer`` -- CUDA-event timing on the launching stream, the only kind
    of number the benchmarks report (max over ranks is taken by the caller).
"""
from __future__ import annotations

import contextlib
import json
import logging
import time
from typing import Dict, List, Optional

log = logging.getLogger("baton_b200.metrics")


class RoundMetrics:
    def __init__(self, name: str, max_records: int = 4096):
        self.name = name
        self.records: List[dict] = []
        self.evals: List[dict] = []         # held-out loss / accuracy of the global model, oldest first
        self.max_records = max_records
        self.counters: Dict[str, float] = {}

    def incr(self, key: str, by: float = 1.0) -> None:
        self.counters[key] = self.counters.get(key, 0.0) + by

    def add(self, **record) -> dict:
        record.setdefault("t", time.time())
        self.records.append(record)
        if len(self.records) > self.max_records:
            del self.records[: len(self.records) - self.max_records]
        log.info("round %s", json.dumps(record, default=str))
        return record

    def add_eval(self, **record) -> dict:
        record.setdefault("t", time.time())
        self.evals.append(record)
        if len(self.evals) > self.max_records:
            del self.evals[: len(self.evals) - self.max_records]
        log.info("eval %s", json.dumps(record, default=str))
        return record

    def summary(self) -> dict:
        walls = [r["wall_s"] for r in self.records if "wall_s" in r]
        samples = sum(r.get("n_samples", 0) for r in self.records)
        total = sum(walls)
        return {
            "name": self.name,
            "rounds": len(self.records),
            "rounds_per_s": (len(walls) / total) if total > 0 else None,
            "samples_per_s": (samples / total) if total > 0 else None,
            "counters": dict(self.counters),
            "last": self.records[-1] if self.records else None,
            "evals": list(self.evals),
        }


@contextlib.contextmanager
def phase(name: str, sink: Optional[dict] = None):
    """NVTX range + host wall-clock for a round phase."""
    pushed = False
    try:
        import torch
        if torch.cuda.is_available():
            torch.cuda.nvtx.range_push(name)
            pushed = True
    except Exception:  # pragma: no cover
        pushed = False
    t0 = time.perf_counter()
    try:
        yield
    finally:
        dt = time.perf_counter() - t0
        if pushed:
            import torch
            torch.cuda.nvtx.range_pop()
        if sink is not None:
            sink[name] = sink.get(name, 0.0) + dt


class DeviceTimer:
    """CUDA-event stopwatch on the current stream; ``elapsed_ms`` synchronises
    on the stop event only."""

    def __init__(self):
        import torch
        self._torch = torch
        self._start = torch.cuda.Event(enable_timing=True)
        self._stop = torch.cuda.Event(enable_timing=True)
        self._armed = False

    def start(self, stream=None) -> "DeviceTimer":
        self._start.record(stream) if stream is not None else self._start.record()
        self._armed = True
        return self

    def stop(self, stream=None) -> "DeviceTimer":
        self._stop.record(stream) if stream is not None else self._stop.record()
        return self

    def elapsed_ms(self) -> float:
        if not self._armed:
            return 0.0
        self._stop.synchronize()
        return float(self._start.elapsed_time(self._stop))
