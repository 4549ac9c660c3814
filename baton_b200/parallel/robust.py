"""Byzantine-robust aggregation: coordinate-wise median and trimmed mean (Yin et al., ICML 2018).

For the ``P`` participating clients of a round and their deltas ``d_k = theta_k - global`` (fp32, as decoded from the
wire), every element ``i`` of the float arena sorts ``d_1[i] .. d_P[i]`` in a total order (-inf < ... < -0 < +0 < ...
< +inf < NaN, every NaN canonicalised to one positive quiet NaN) into ``x[0] <= ... <= x[P-1]`` and takes

    median        x[P/2] for odd P, 0.5 * (x[(P-1)/2] + x[P/2]) for even P       (numpy's median, not torch's lower one)
    trimmed mean  (x[b] + x[b+1] + ... + x[P-b-1]) / (P - 2b),  b = floor(beta * P),  added in ascending order from 0

in fp32 with IEEE round-to-nearest, then ``global += result``.  ``P = 0`` changes nothing; ``P = 1`` gives that client's
delta.  The statistic is UNWEIGHTED over clients, as Flower's FedMedian / FedTrimmedAvg: a sample count is whatever a
client says it is, and weighting by it would hand the outcome to any client that claims a large one.  Integer buffers
keep the max-over-participants policy, and the reported loss stays the sample-weighted mean (a metric, not the update).

At most ``MAX_ROBUST_CLIENTS`` = 32 participants per round: the fused collective's tile owner sorts every element's
values in registers.  :func:`robust_combine` is the host implementation (the oracle of the tests and the CPU / gloo
path); ``csrc/fedavg.cu`` (``fedavg_allreduce_robust_kernel``) computes the same bits on an fp32 wire.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List

import torch

MAX_ROBUST_CLIENTS = 32
KINDS = ("median", "trimmed_mean")
AGGREGATORS = ("mean",) + KINDS


def check_robust(kind: str, trim_ratio: float) -> float:
    """Validate ``(kind, beta)``: ``kind`` in ``KINDS`` and ``0 <= beta < 0.5`` (finite)."""
    if kind not in KINDS:
        raise ValueError("robust aggregator must be one of {}, got {!r}".format(KINDS, kind))
    beta = float(trim_ratio)
    if not (0.0 <= beta < 0.5):
        raise ValueError("trim_ratio must satisfy 0 <= trim_ratio < 0.5, got {!r}".format(trim_ratio))
    return beta


def check_aggregator(aggregator: str, trim_ratio: float) -> float:
    """Validate an engine / config ``aggregator`` (``"mean"`` or a robust kind) and its ``trim_ratio``."""
    if aggregator not in AGGREGATORS:
        raise ValueError("aggregator must be one of {}, got {!r}".format(AGGREGATORS, aggregator))
    beta = float(trim_ratio)
    if not (0.0 <= beta < 0.5):
        raise ValueError("trim_ratio must satisfy 0 <= trim_ratio < 0.5, got {!r}".format(trim_ratio))
    return beta


@dataclass
class RobustConfig:
    """``kind``: ``"median"`` or ``"trimmed_mean"``; ``trim_ratio`` = beta, the fraction trimmed at EACH end (read only
    by the trimmed mean)."""
    kind: str = "median"
    trim_ratio: float = 0.1

    def __post_init__(self):
        self.trim_ratio = check_robust(self.kind, self.trim_ratio)

    @property
    def kind_id(self) -> int:
        return KINDS.index(self.kind)

    def trim_count(self, p: int) -> int:
        """``b = floor(beta * P)`` (0 for the median)."""
        return trim_count(self.trim_ratio, p) if self.kind == "trimmed_mean" else 0

    def trim_table(self) -> List[int]:
        """``b`` for ``P = 0 .. 32``: the collective reads its round's entry."""
        return [self.trim_count(p) for p in range(MAX_ROBUST_CLIENTS + 1)]

    def to_dict(self) -> dict:
        return {"kind": self.kind, "trim_ratio": self.trim_ratio}


def trim_count(beta: float, p: int) -> int:
    return int(math.floor(float(beta) * int(p)))


def check_participants(n: int) -> None:
    if n > MAX_ROBUST_CLIENTS:
        raise ValueError("robust aggregation takes at most {} participants per round, got {}".format(
            MAX_ROBUST_CLIENTS, n))


def _keys(x: torch.Tensor) -> torch.Tensor:
    """Order-preserving int64 keys of fp32 values (uint32 sign-flip key; NaN canonicalised above +inf)."""
    u = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    u = torch.where(torch.isnan(x), torch.full_like(u, 0x7FC00000), u)
    neg = (u & 0x80000000) != 0
    return torch.where(neg, u ^ 0xFFFFFFFF, u | 0x80000000)


@torch.no_grad()
def robust_combine(stacked: torch.Tensor, cfg: RobustConfig) -> torch.Tensor:
    """The robust statistic of ``stacked`` (fp32 ``[P, n]``, one row per participant) per column: fp32 ``[n]``.
    ``P = 0`` gives zeros.  Sequential fp32 adds in sorted order, IEEE division: the kernel's bits on an fp32 wire."""
    x = stacked.to(torch.float32)
    if x.dim() != 2:
        raise ValueError("robust_combine takes a [P, n] stack")
    p, n = x.shape
    check_participants(p)
    if p == 0:
        return torch.zeros(n, dtype=torch.float32, device=x.device)
    x = torch.where(torch.isnan(x), torch.full_like(x, float("nan")), x)
    order = torch.argsort(_keys(x), dim=0, stable=True)
    s = torch.gather(x, 0, order)
    s = torch.where(torch.isnan(s), torch.full_like(s, float("nan")), s)
    if cfg.kind == "median":
        if p % 2:
            return s[p // 2].clone()
        return (s[(p - 1) // 2] + s[p // 2]) * 0.5
    b = cfg.trim_count(p)
    acc = torch.zeros(n, dtype=torch.float32, device=x.device)
    for j in range(b, p - b):
        acc = acc + s[j]
    return acc / torch.tensor(float(p - 2 * b), dtype=torch.float32, device=x.device)
