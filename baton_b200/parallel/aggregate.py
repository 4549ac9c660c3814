"""FedAvg aggregation algebra (host-visible entry points).

Parity target: ``Experiment.end_round`` (reference manager.py:113-132):

    N = sum_k n_k
    for every key of the global state_dict:  value[:] = sum_k(sd_k[key] * n_k) / N
    loss_history[e] = sum_k(loss_k[e] * n_k) / N     for e in range(n_epoch)

The reduction is written into the *live* storage of the global model, covers
every ``state_dict`` entry (buffers included), and is a no-op when N == 0.

Integer buffers (``num_batches_tracked``; quirk 16) cannot go through the float
formula; the policy here is ``max`` over participants (every client advanced the
counter by its own step count; the max is the furthest-advanced replica and
keeps BatchNorm's ``momentum=None`` mode monotone).  ``int_policy='mean'`` gives
the rounded weighted mean instead.

On CUDA tensors the float path runs the hand-written multi-source weighted-sum
kernel (``ops.weighted_sum_``) instead of K temporaries per key.
"""
from __future__ import annotations

from typing import List, Mapping, Optional, Sequence

import torch


def client_weights(n_samples: Sequence[float]) -> List[float]:
    """Normalised FedAvg weights ``n_k / N`` (all zeros when N == 0)."""
    total = float(sum(n_samples))
    if total <= 0:
        return [0.0 for _ in n_samples]
    return [float(n) / total for n in n_samples]


def _reduce_float(dst: torch.Tensor, srcs: List[torch.Tensor], weights: List[float]) -> None:
    if dst.is_cuda:
        from ..ops import weighted_sum_
        weighted_sum_(dst, srcs, weights)
        return
    acc = torch.zeros_like(dst, dtype=torch.float32 if dst.dtype != torch.float64 else torch.float64)
    for s, w in zip(srcs, weights):
        acc.add_(s.to(device=dst.device, dtype=acc.dtype), alpha=w)
    dst.copy_(acc.to(dst.dtype))


def _reduce_int(dst: torch.Tensor, srcs: List[torch.Tensor], weights: List[float], policy: str) -> None:
    stack = torch.stack([s.to(device=dst.device, dtype=torch.int64).reshape(dst.shape) for s in srcs])
    if policy == "max":
        out = stack.max(dim=0).values
    elif policy == "mean":
        w = torch.tensor(weights, dtype=torch.float64, device=dst.device).view(-1, *([1] * dst.dim()))
        out = (stack.to(torch.float64) * w).sum(0).round().to(torch.int64)
    elif policy == "keep":
        return
    else:
        raise ValueError("unknown int_policy {!r}".format(policy))
    dst.copy_(out.to(dst.dtype))


@torch.no_grad()
def fedavg_into(global_state: Mapping[str, torch.Tensor],
                client_states: Sequence[Mapping[str, torch.Tensor]],
                n_samples: Sequence[float], *, int_policy: str = "max",
                strict: bool = True) -> bool:
    """Sample-weighted mean of ``client_states`` written in place into
    ``global_state``.  Returns False (and touches nothing) when N == 0."""
    if len(client_states) != len(n_samples):
        raise ValueError("client_states and n_samples differ in length")
    weights = client_weights(n_samples)
    if not any(weights):
        return False
    keep = [i for i, w in enumerate(weights) if w > 0.0]
    for key, value in global_state.items():
        srcs, ws = [], []
        for i in keep:
            sd = client_states[i]
            if key not in sd:
                if strict:
                    raise KeyError("client state_dict is missing {!r}".format(key))
                continue
            srcs.append(sd[key])
            ws.append(weights[i])
        if not srcs:
            continue
        if not strict and len(srcs) != len(keep):
            tot = sum(ws)
            ws = [w / tot for w in ws]
        if value.is_floating_point() or value.is_complex():
            _reduce_float(value, srcs, ws)
        else:
            _reduce_int(value, srcs, ws, int_policy)
    return True


@torch.no_grad()
def dp_fedavg_into(global_state: Mapping[str, torch.Tensor], client_states: Sequence[Mapping[str, torch.Tensor]], *,
                   clip: float, noise_multiplier: float, seed: int, round_index: int,
                   int_policy: str = "max") -> List[float]:
    """DP-FedAvg (``parallel/dp.py``) written in place into ``global_state``: every client's update ``Delta_k`` is its
    float entries minus the global ones, taken as ONE vector in ``global_state`` order; ``s_k = min(1, clip /
    ||Delta_k||)`` (0 when not finite -- the client still counts in m); ``global += (sum_k s_k Delta_k + sigma C z) / m``
    with uniform weights and ``z`` the Philox stream ``(seed, round_index)`` over the same element order.  Integer
    entries follow ``int_policy`` over all clients.  Computed in float64, cast once.  Returns the clip factors."""
    from .dp import check_dp, norm_to_factor, normals
    import math
    clip, sigma = check_dp(clip, noise_multiplier)
    m = len(client_states)
    if m == 0:
        return []
    fkeys = [k for k, v in global_state.items() if v.is_floating_point()]
    for sd in client_states:
        missing = [k for k in global_state if k not in sd]
        if missing:
            raise KeyError("client state_dict is missing {!r}".format(missing[0]))
    deltas = []
    for sd in client_states:
        deltas.append([sd[k].detach().to(device="cpu", dtype=torch.float64).reshape(-1)
                       - global_state[k].detach().to(device="cpu", dtype=torch.float64).reshape(-1) for k in fkeys])
    factors = []
    for d in deltas:
        sq = sum(float(t.pow(2).sum()) for t in d)
        factors.append(norm_to_factor(math.sqrt(sq) if math.isfinite(sq) else float("nan"), clip))
    n_total = sum(global_state[k].numel() for k in fkeys)
    z = torch.from_numpy(normals(seed, round_index, n_total)) if sigma > 0.0 else None
    off = 0
    for i, k in enumerate(fkeys):
        g = global_state[k]
        acc = torch.zeros(g.numel(), dtype=torch.float64)
        for d, sk in zip(deltas, factors):
            if sk != 0.0:
                acc.add_(d[i], alpha=sk)
        if z is not None:
            acc.add_(z[off: off + g.numel()], alpha=sigma * clip)
        off += g.numel()
        new = g.detach().to(device="cpu", dtype=torch.float64).reshape(-1) + acc / m
        g.copy_(new.reshape(g.shape).to(device=g.device, dtype=g.dtype))
    for k, v in global_state.items():
        if not v.is_floating_point():
            _reduce_int(v, [sd[k] for sd in client_states], [1.0 / m] * m, int_policy)
    return factors


def fedavg_loss_history(loss_histories: Sequence[Sequence[float]], n_samples: Sequence[float],
                        n_epoch: Optional[int] = None) -> List[float]:
    """Per-epoch sample-weighted loss (manager.py:127-130).  A client that
    reported fewer than ``n_epoch`` entries (early stop) simply does not
    contribute to the missing epochs; the weights are renormalised."""
    if n_epoch is None:
        n_epoch = max((len(h) for h in loss_histories), default=0)
    out: List[float] = []
    for e in range(n_epoch):
        num = 0.0
        den = 0.0
        for hist, n in zip(loss_histories, n_samples):
            if e < len(hist) and n > 0:
                num += float(hist[e]) * float(n)
                den += float(n)
        if den > 0:
            out.append(num / den)
    return out


@torch.no_grad()
def robust_into(global_state: Mapping[str, torch.Tensor], client_states: Sequence[Mapping[str, torch.Tensor]], cfg,
                int_policy: str = "max") -> bool:
    """Coordinate-wise median / trimmed mean or Multi-Krum (``parallel/robust.py``, ``cfg`` a ``RobustConfig``) written
    in place into ``global_state``: every client's delta is its float entries minus the global ones in fp32, taken in
    ``global_state`` order; ``global += robust_combine(deltas)``, unweighted over clients.  Krum's distances span every
    float entry, so it takes two passes: the first selects the kept clients over the concatenated deltas, the second
    applies their plain mean key by key.  Integer entries follow ``int_policy`` over all clients.  Returns False (and
    touches nothing) without clients."""
    from .robust import RobustConfig, check_participants, krum_select, robust_combine
    m = len(client_states)
    if m == 0:
        return False
    check_participants(m)
    for sd in client_states:
        missing = [k for k in global_state if k not in sd]
        if missing:
            raise KeyError("client state_dict is missing {!r}".format(missing[0]))
    if cfg.kind == "krum":
        floats = [k for k, g in global_state.items() if g.is_floating_point()]
        flat = torch.cat([torch.stack([sd[k].detach().to(device="cpu", dtype=torch.float32).reshape(-1)
                                       - global_state[k].detach().to(device="cpu", dtype=torch.float32).reshape(-1)
                                       for sd in client_states]) for k in floats], 1)
        kept = krum_select(flat, cfg)[2].tolist()
        rows = [sd for sd, keep in zip(client_states, kept) if keep]
        cfg = RobustConfig("trimmed_mean", 0.0)
    else:
        rows = client_states
    for k, g in global_state.items():
        if not g.is_floating_point():
            continue
        g32 = g.detach().to(device="cpu", dtype=torch.float32).reshape(-1)
        stack = torch.stack([sd[k].detach().to(device="cpu", dtype=torch.float32).reshape(-1) - g32
                             for sd in rows])
        new = g32 + robust_combine(stack, cfg)
        g.copy_(new.reshape(g.shape).to(device=g.device, dtype=g.dtype))
    for k, v in global_state.items():
        if not v.is_floating_point():
            _reduce_int(v, [sd[k] for sd in client_states], [1.0 / m] * m, int_policy)
    return True
