"""Top-k sparsified client uploads with error feedback (Stich et al., NeurIPS 2018; Karimireddy et al., ICML 2019).

Each participating client ``i`` uploads only the ``k`` largest-magnitude entries of its update and carries the rest
into its next round in a residual ``e_i`` (fp32 over the arena, kept on the rank that hosts the client, zeros the first
time it takes part):

    u   = fl32(fl32(theta - global) + e_i)          (each operation rounded separately; without error feedback
                                                     u = theta - global)
    S   = the first k elements in the order  key = |u| descending, then arena index ascending
    e_i = u off S, 0 on S                            (so u == topk(u) + e_i exactly in fp32)

``k = max(1, ceil(ratio * n_float))``, ``n_float`` being the float ``state_dict`` elements (parameters and BatchNorm
running statistics, without the arena's padding).  The key is the 31-bit magnitude pattern ``bits(u) & 0x7FFFFFFF``;
every NaN gets the key of the canonical quiet NaN, ``0x7FC00000``, above +inf.  The round's update is the
sample-weighted mean of the clients' ``topk(u)``, cast through the session's wire dtype; the wire cast is not fed back.

This module holds the configuration, the per-client residuals and the host implementation of the rule:
:func:`topk_select` / :func:`topk_ef_` (the oracle of the tests and the selection of :class:`NcclSession`) and
:func:`topk_combine`, which reproduces the fused collective's reduce (``fedavg_round_kernel<WIRE, FedAvgTopkArgs>``).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import torch

GRANULE = 1024          # elements per row of the sparse wire format (= the collective's FLAG_GRANULE)
NAN_KEY = 0x7FC00000


@dataclass(frozen=True)
class TopKConfig:
    """``ratio`` in ``(0, 1]``: the share of the float elements each client uploads; ``error_feedback``: carry the
    unsent remainder in a per-client residual."""
    ratio: float
    error_feedback: bool = True

    def __post_init__(self):
        r = self.ratio
        if isinstance(r, bool) or not isinstance(r, (int, float)) or not math.isfinite(float(r)) or not (0.0 < r <= 1.0):
            raise ValueError("topk_ratio must be in (0, 1], got {!r}".format(r))
        object.__setattr__(self, "ratio", float(r))
        object.__setattr__(self, "error_feedback", bool(self.error_feedback))

    def k(self, n_float: int) -> int:
        return max(1, math.ceil(self.ratio * int(n_float)))


def n_float(arena) -> int:
    """Float ``state_dict`` elements of an arena, without its alignment padding."""
    return sum(s.numel for s in arena.slots.values())


class TopKState:
    """Per-client residuals ``e_i`` of one rank (fp32 over the arena), allocated as zeros on first use."""

    def __init__(self, n: int, device):
        self.n = int(n)
        self.device = torch.device(device)
        self.e: Dict[int, torch.Tensor] = {}

    def residual(self, cid: int) -> torch.Tensor:
        e = self.e.get(cid)
        if e is None:
            e = self.e[cid] = torch.zeros(self.n, dtype=torch.float32, device=self.device)
        return e


def topk_keys(u: torch.Tensor) -> torch.Tensor:
    """int64 selection keys of fp32 ``u``: the 31-bit magnitude pattern, NaN -> ``NAN_KEY`` (above +inf)."""
    bits = u.contiguous().view(torch.int32).to(torch.int64) & 0x7FFFFFFF
    return torch.where(bits > 0x7F800000, torch.full_like(bits, NAN_KEY), bits)


def topk_select(u: torch.Tensor, k: int) -> torch.Tensor:
    """Indices (ascending) of the first ``k`` elements of ``u`` by key descending, ties by ascending index."""
    k = int(k)
    if not (1 <= k <= u.numel()):
        raise ValueError("k must be in 1..{}, got {}".format(u.numel(), k))
    key = topk_keys(u.reshape(-1))
    order = torch.sort(key, descending=True, stable=True).indices     # stable: equal keys keep ascending index
    return torch.sort(order[:k]).values


@torch.no_grad()
def topk_ef_(theta: torch.Tensor, global_w: torch.Tensor, e: Optional[torch.Tensor], k: int) -> Tuple[torch.Tensor,
                                                                                                    torch.Tensor]:
    """One client's selection: ``u = (theta - global) + e`` (``e`` None: no error feedback), ``S = topk(u)``; ``e``
    becomes ``u`` off ``S`` and 0 on it (in place).  Returns ``(idx, u[idx])`` with ``idx`` ascending."""
    u = theta - global_w
    if e is not None:
        u = u + e
    idx = topk_select(u, k)
    vals = u[idx].clone()
    if e is not None:
        e.copy_(u)
        e[idx] = 0.0
    return idx, vals


def wire_torch_dtype(wire_dtype: str) -> torch.dtype:
    return {"fp32": torch.float32, "bf16": torch.bfloat16}[wire_dtype]


def topk_combine(per_rank_sparse: Sequence[Optional[Tuple[torch.Tensor, torch.Tensor]]], weights: Sequence[float],
                 n: int, wire_dtype: str = "fp32") -> torch.Tensor:
    """The fused top-k reduce on the host: ``per_rank_sparse[r] = (idx, values)`` (values already in the wire dtype,
    None for a rank without upload), ``weights[r] = w_r`` (fp32).  Every element starts at +0 and takes
    ``acc = fl32(w_r * x + acc)`` in rank order, skipping ``w_r == 0`` and absent entries; the result is cast to the wire
    dtype and returned as fp32.  The fused multiply-add is computed in fp64: the product of two fp32 values is exact
    there, and the one rounding of the sum to fp32 is then the rounding ``fmaf`` makes, except in the rare case where
    the fp64 sum itself rounds to a value halfway between two fp32 numbers."""
    acc = torch.zeros(int(n), dtype=torch.float64)
    for sp, w in zip(per_rank_sparse, weights):
        w = float(torch.tensor(float(w), dtype=torch.float32))
        if sp is None or w == 0.0:
            continue
        idx, vals = sp
        idx = idx.cpu()
        x = vals.float().cpu().double()
        acc[idx] = (x * w + acc[idx]).float().double()
    return acc.float().to(wire_torch_dtype(wire_dtype)).float()


def sparse_upload_bytes(n: int, entries: int, wire_dtype: str) -> int:
    """Bytes of one sparse upload: the row pointers, then a 16-bit offset and a value per entry."""
    vb = 4 if wire_dtype == "fp32" else 2
    return 4 * (int(n) // GRANULE + 1) + int(entries) * (2 + vb)
