"""Byzantine-robust aggregation: coordinate-wise median and trimmed mean (Yin et al., ICML 2018), and Multi-Krum
(Blanchard et al., NeurIPS 2017; El Mhamdi et al., ICML 2018).

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
path); ``csrc/fedavg.cu`` (``fedavg_round_kernel<WIRE, FedAvgRobustArgs>``) computes the same bits on an fp32 wire.

Multi-Krum (``kind="krum"``, ``krum_f`` = f Byzantine clients assumed, ``krum_m`` = m clients kept) works on whole
updates instead of coordinates.  With ``D[i][j] = sum_e (d_i[e] - d_j[e])^2`` over the float arena (a non-finite
``D`` counts as +inf), ``k = max(1, P - f - 2)`` capped at ``P - 1``, and ``score_i`` the sum of the ``k`` smallest
``D[i][j]`` (``j != i``) added in ascending order in fp64 (0 when ``P = 1``), the clients are ordered by ``(score,
segment position)`` and the first ``m = clamp(krum_m or P - f, 1, P)`` are kept.  The update is the trimmed mean with
``b = 0`` over the kept rows (their plain mean, added in ascending order, so it depends only on the kept values).
``krum_m = 1`` is classic Krum.  Blanchard's guarantee needs ``P > 2f + 2``: the engine and the configuration reject a
planned participant count below ``2f + 3``, but a round that arrives with fewer participants still runs with the
clamped ``k`` and ``m`` above.  :func:`krum_select` is the host selection; the fused collective
(``fedavg_round_kernel<WIRE, FedAvgKrumArgs>``) computes ``D`` from fp32 partial sums per chunk, fp64 across chunks, so its scores
agree with the host's to rounding and its kept mean is bitwise the host's for the same kept set.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

MAX_ROBUST_CLIENTS = 32
KINDS = ("median", "trimmed_mean", "krum")
AGGREGATORS = ("mean",) + KINDS


def check_robust(kind: str, trim_ratio: float) -> float:
    """Validate ``(kind, beta)``: ``kind`` in ``KINDS`` and ``0 <= beta < 0.5`` (finite)."""
    if kind not in KINDS:
        raise ValueError("robust aggregator must be one of {}, got {!r}".format(KINDS, kind))
    beta = float(trim_ratio)
    if not (0.0 <= beta < 0.5):
        raise ValueError("trim_ratio must satisfy 0 <= trim_ratio < 0.5, got {!r}".format(trim_ratio))
    return beta


def check_krum(krum_f, krum_m) -> Tuple[int, Optional[int]]:
    """Validate Multi-Krum's ``f`` (an int >= 0) and ``m`` (None or an int >= 1)."""
    if isinstance(krum_f, bool) or not isinstance(krum_f, int) or krum_f < 0:
        raise ValueError("krum_f must be an int >= 0, got {!r}".format(krum_f))
    if krum_m is not None and (isinstance(krum_m, bool) or not isinstance(krum_m, int) or krum_m < 1):
        raise ValueError("krum_m must be None or an int >= 1, got {!r}".format(krum_m))
    return krum_f, krum_m


def check_krum_participants(planned: int, krum_f: int) -> None:
    """Blanchard's condition ``n > 2f + 2`` on the planned participant count of a round."""
    if int(planned) < 2 * int(krum_f) + 3:
        raise ValueError("Krum with f={} needs at least 2f + 3 = {} participants per round, {} are planned".format(
            krum_f, 2 * krum_f + 3, planned))


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
    """``kind``: ``"median"``, ``"trimmed_mean"`` or ``"krum"``; ``trim_ratio`` = beta, the fraction trimmed at EACH
    end (read only by the trimmed mean); ``krum_f`` / ``krum_m``: Multi-Krum's assumed Byzantine clients and kept
    clients (``None``: ``P - f``; read only by Krum)."""
    kind: str = "median"
    trim_ratio: float = 0.1
    krum_f: int = 0
    krum_m: Optional[int] = None

    def __post_init__(self):
        self.trim_ratio = check_robust(self.kind, self.trim_ratio)
        self.krum_f, self.krum_m = check_krum(self.krum_f, self.krum_m)

    @property
    def kind_id(self) -> int:
        return KINDS.index(self.kind)

    def trim_count(self, p: int) -> int:
        """``b = floor(beta * P)`` (0 for the median and for Krum's kept mean)."""
        return trim_count(self.trim_ratio, p) if self.kind == "trimmed_mean" else 0

    def trim_table(self) -> List[int]:
        """``b`` for ``P = 0 .. 32``: the collective reads its round's entry."""
        return [self.trim_count(p) for p in range(MAX_ROBUST_CLIENTS + 1)]

    def krum_k(self, p: int) -> int:
        """Neighbours summed into a score: ``max(1, P - f - 2)`` capped at ``P - 1`` (0 for ``P <= 1``)."""
        return min(max(1, int(p) - self.krum_f - 2), max(int(p) - 1, 0))

    def krum_kept(self, p: int) -> int:
        """Clients kept: ``clamp(krum_m or P - f, 1, P)`` (0 for ``P = 0``)."""
        if p <= 0:
            return 0
        m = self.krum_m if self.krum_m is not None else int(p) - self.krum_f
        return min(max(m, 1), int(p))

    def krum_tables(self) -> Tuple[List[int], List[int]]:
        """``k`` and ``m`` for ``P = 0 .. 32``: the Krum collective reads its round's entries."""
        r = range(MAX_ROBUST_CLIENTS + 1)
        return [self.krum_k(p) for p in r], [self.krum_kept(p) for p in r]

    def to_dict(self) -> dict:
        if self.kind == "krum":
            return {"kind": "krum", "f": self.krum_f, "m": self.krum_m}
        return {"kind": self.kind, "trim_ratio": self.trim_ratio}

    @classmethod
    def from_dict(cls, d: dict) -> "RobustConfig":
        """Inverse of :meth:`to_dict` (the seated planes' plan)."""
        if d["kind"] == "krum":
            m = d.get("m")
            return cls("krum", krum_f=int(d.get("f", 0)), krum_m=int(m) if m is not None else None)
        return cls(str(d["kind"]), float(d["trim_ratio"]))


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
def krum_select(stacked: torch.Tensor, cfg: RobustConfig) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Multi-Krum's selection over ``stacked`` (fp32 ``[P, n]``, rows in segment order): ``(D, scores, kept)`` --
    the fp64 ``[P, P]`` squared distances (non-finite: +inf, diagonal 0), the fp64 ``[P]`` scores and the bool
    ``[P]`` mask of the ``m`` kept rows (lowest ``(score, position)``).  Everything on the host, in fp64."""
    x = stacked.to(torch.float32)
    if x.dim() != 2:
        raise ValueError("krum_select takes a [P, n] stack")
    p = x.shape[0]
    check_participants(p)
    x = x.detach().double()
    D = torch.zeros(p, p, dtype=torch.float64)
    for i in range(p):
        for j in range(i + 1, p):
            d = float(((x[i] - x[j]) ** 2).sum())
            D[i, j] = D[j, i] = d if math.isfinite(d) else math.inf
    k = cfg.krum_k(p)
    scores = torch.zeros(p, dtype=torch.float64)
    for i in range(p):
        row = sorted(float(D[i, j]) for j in range(p) if j != i)
        acc = 0.0
        for v in row[:k]:
            acc += v
        scores[i] = acc
    order = sorted(range(p), key=lambda i: (float(scores[i]), i))
    kept = torch.zeros(p, dtype=torch.bool)
    kept[order[: cfg.krum_kept(p)]] = True
    return D, scores, kept


@torch.no_grad()
def robust_combine(stacked: torch.Tensor, cfg: RobustConfig) -> torch.Tensor:
    """The robust statistic of ``stacked`` (fp32 ``[P, n]``, one row per participant) per column: fp32 ``[n]``.
    ``P = 0`` gives zeros.  Sequential fp32 adds in sorted order, IEEE division: the kernel's bits on an fp32 wire.
    Krum: the trimmed mean with ``b = 0`` over the rows :func:`krum_select` keeps."""
    x = stacked.to(torch.float32)
    if x.dim() != 2:
        raise ValueError("robust_combine takes a [P, n] stack")
    p, n = x.shape
    check_participants(p)
    if p == 0:
        return torch.zeros(n, dtype=torch.float32, device=x.device)
    if cfg.kind == "krum":
        kept = krum_select(x, cfg)[2].to(x.device)
        return robust_combine(x[kept], RobustConfig("trimmed_mean", 0.0))
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
