"""Personalized federated learning: client-local ``state_dict`` entries (FedBN, FedPer).

``FederatedEngine(local_keys=...)`` keeps some float ``state_dict`` entries with each client instead of averaging them:

* ``"bn"`` -- FedBN (Li et al., ICLR 2021): every ``ops.nn.BatchNorm2d``'s ``weight``, ``bias``, ``running_mean`` and
  ``running_var``;
* ``"head"`` -- FedPer (Arivazhagan et al., 2019): the entries under the model's ``head`` prefix (ResNet ``fc``, BERT
  ``classifier``, ``MLP2`` ``fc2``);
* any ``state_dict`` key or ``fnmatch`` pattern, mixed with the presets, e.g. ``("bn", "head")``.

Integer buffers (``num_batches_tracked``) stay shared.  The arena lays the local entries out as one contiguous range
``[lo, hi)`` of whole 1024-element granules (``ParamArena(local=...)``) that the collective never reads or writes, so
every swap below is a slice copy.  :class:`LocalStore` holds the initial values of the range and one fp32 vector per
hosted client that has taken part, ``4 (hi - lo)`` bytes each.
"""
from __future__ import annotations

import fnmatch
from dataclasses import replace
from typing import Dict, List, Sequence, Union

import torch
from torch import nn


def _float_keys(model: nn.Module) -> List[str]:
    return [k for k, v in model.state_dict().items() if v.is_floating_point()]


def resolve_local_keys(model: nn.Module, local_keys: Union[str, Sequence[str]]) -> List[str]:
    """The float ``state_dict`` keys that ``local_keys`` names, in ``state_dict`` order.  ``ValueError`` for a preset or
    pattern that matches nothing, a model without a head under ``"head"``, and a set that covers every float entry."""
    items = [local_keys] if isinstance(local_keys, str) else list(local_keys)
    if not items or not all(isinstance(x, str) for x in items):
        raise ValueError("local_keys takes 'bn', 'head', state_dict keys or fnmatch patterns, got {!r}".format(local_keys))
    floats = _float_keys(model)
    chosen = set()
    for item in items:
        if item == "bn":
            from ..ops.nn import BatchNorm2d
            prefixes = [name + "." for name, m in model.named_modules() if isinstance(m, BatchNorm2d)]
            hit = [k for k in floats if any(k.startswith(p) for p in prefixes)]
        elif item == "head":
            head = getattr(model, "head", None)
            if not head:
                raise ValueError("local_keys='head' needs a model with a head prefix; {} has none".format(
                    type(model).__name__))
            hit = [k for k in floats if k.startswith(head + ".")]
            if hit and len(hit) == len(floats):
                raise ValueError("local_keys='head': the head {!r} of {} is the whole model".format(
                    head, type(model).__name__))
        else:
            hit = [k for k in floats if fnmatch.fnmatchcase(k, item)]
        if not hit:
            raise ValueError("local_keys entry {!r} matches no float state_dict entry".format(item))
        chosen.update(hit)
    if len(chosen) == len(floats):
        raise ValueError("local_keys cover every float state_dict entry: nothing would be shared")
    return [k for k in floats if k in chosen]


class LocalStore:
    """The client-local range ``[lo, hi)`` of an arena: its initial values and one vector per hosted client."""

    def __init__(self, arena, keys: Sequence[str]):
        if arena.local_range is None:
            raise ValueError("the arena has no client-local range")
        self.arena = arena
        self.keys = list(keys)
        self.lo, self.hi = arena.local_range
        self.init = arena.theta[self.lo: self.hi].clone()
        self.clients: Dict[int, torch.Tensor] = {}

    def values(self, cid: int) -> torch.Tensor:
        """Client ``cid``'s vector (live): the initial values until it has taken part."""
        return self.clients.get(int(cid), self.init)

    @torch.no_grad()
    def swap_in(self, cid: int) -> None:
        """Load client ``cid``'s entries into the replica: theta, global_w (FedProx's anchor), the bf16 shadow, and a
        zero momentum over the local parameters (a client starts every round without momentum)."""
        a, lo, hi = self.arena, self.lo, self.hi
        v = self.clients.get(int(cid))
        if v is None:
            v = self.clients[int(cid)] = self.init.clone()
        a.theta[lo:hi].copy_(v)
        self.refresh()

    @torch.no_grad()
    def refresh(self) -> None:
        """The replica already holds its client's entries in theta (one client per GPU): copy them into global_w and
        the bf16 shadow, and zero the momentum over the local parameters."""
        a, lo, hi = self.arena, self.lo, self.hi
        a.global_w[lo:hi].copy_(a.theta[lo:hi])
        if a.theta_bf16 is not None:
            a.theta_bf16[lo:hi].copy_(a.theta[lo:hi])
        if a.momentum is not None and a.n_param > lo:
            a.momentum[lo: a.n_param].zero_()

    @torch.no_grad()
    def swap_out(self, cid: int) -> None:
        """Keep what client ``cid``'s training left in the replica's local range."""
        v = self.clients.get(int(cid))
        if v is None:
            v = self.clients[int(cid)] = torch.empty_like(self.init)
        v.copy_(self.arena.theta[self.lo: self.hi])

    def entries(self, cid: int) -> Dict[str, torch.Tensor]:
        """``{key: tensor}`` copies of client ``cid``'s local entries, shaped as in ``state_dict``."""
        return self._unflatten(self.values(cid))

    def initial_entries(self) -> Dict[str, torch.Tensor]:
        """``{key: tensor}`` copies of the initial values: what a client starts from."""
        return self._unflatten(self.init)

    def _unflatten(self, v: torch.Tensor) -> Dict[str, torch.Tensor]:
        a = self.arena
        out = {}
        for k in self.keys:
            s = a.slots[k]
            flat = v[s.offset - self.lo: s.offset - self.lo + s.numel].clone()
            out[k] = a._view(flat, replace(s, offset=0))
        return out
