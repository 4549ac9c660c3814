"""Flat parameter arena.

Every floating ``state_dict`` entry of a model (parameters first, then float
buffers such as BatchNorm running statistics) is re-homed into ONE contiguous
fp32 buffer at a fixed, 8-element-aligned offset; integer buffers
(``num_batches_tracked``) go to a small int64 side arena.  The module's
parameters/buffers become views, so ``state_dict()`` / ``load_state_dict()`` and
the checkpoint layout are unchanged (reference: the global model is addressed by
``state_dict`` keys, manager.py:78,123) while

* the optimizer is one kernel over ``theta[:n_param]`` (``ops.fused_sgd``),
* the FedAvg collective is one kernel over ``theta[:n]`` (parameters AND
  running statistics -- the reference averages every entry, manager.py:123),
* gradients (``grad``), momentum, the bf16 shadow weights consumed by the GEMMs
  (``theta_bf16``) and the frozen global copy used for delta uploads
  (``global_w``) are parallel flat buffers with identical offsets on every rank.

With client-local entries (FedBN / FedPer, ``parallel/personal.py``) the slots are reordered so that those entries
form one 1024-aligned range ``local_range`` that the collective skips; see :class:`ParamArena`.  Frozen parameters
(``requires_grad=False``, e.g. the base weights of a LoRA model) form the 1024-aligned range ``frozen_range`` right
after the trainable ones: they have no gradient or optimizer state, and the collective skips them too.

Conv weights keep their logical ``[Cout, Cin, KH, KW]`` shape with channels_last
strides, i.e. they are physically ``[Cout, KH, KW, Cin]`` in the arena.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, Iterable, Optional, Tuple

import torch
from torch import nn

ALIGN = 8  # elements: 16 B for bf16, 32 B for fp32 -> every view satisfies TMA / vector alignment
LOCAL_ALIGN = 1024  # edges of the client-local range: no wire vector, fp8 block or collective granule crosses one


@dataclass
class Slot:
    name: str
    offset: int
    numel: int
    shape: Tuple[int, ...]
    channels_last: bool
    is_param: bool


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class ParamArena:
    def __init__(self, model: nn.Module, device=None, *, momentum: bool = False, bf16_shadow: bool = True,
                 keep_global: bool = True, theta_storage: Optional[torch.Tensor] = None, total_align: int = 2048,
                 local: Iterable[str] = ()):
        """``local``: names of float ``state_dict`` entries that stay with each client (``parallel/personal.py``).  They
        are laid out as one contiguous range ``local_range = (lo, hi)`` of whole 1024-element granules that straddles
        ``n_param``: ``[shared params | pad][local params | local float buffers | pad][shared float buffers]``.
        Without them the layout is parameters, then float buffers, and ``local_range`` is None.

        Parameters with ``requires_grad=False`` are laid out as ``frozen_range = (lo, hi)`` of whole 1024-element
        granules: ``[trainable params | pad][frozen params | pad][float buffers]`` with ``n_param = lo``, so the gradient,
        momentum, AdamW and server-optimizer state cover the trainable parameters only while ``theta``, ``global_w`` and
        the bf16 shadow hold everything.  Without frozen parameters ``frozen_range`` is None and the layout unchanged."""
        self.model = model
        params = [(n, p) for n, p in model.named_parameters()]
        device = torch.device(device) if device is not None else (params[0][1].device if params else torch.device("cpu"))
        self.device = device
        self.slots: "OrderedDict[str, Slot]" = OrderedDict()
        self.int_slots: "OrderedDict[str, Tuple[int, int]]" = OrderedDict()
        local = frozenset(local)
        seen = set()
        uniq = []
        for name, p in params:
            if id(p) not in seen:
                seen.add(id(p))
                uniq.append((name, p))
        bufs = []
        ioff = 0
        for name, b in model.named_buffers():
            if name.split(".")[-1] in getattr(self._owner(name), "_non_persistent_buffers_set", ()):
                continue
            if b.is_floating_point():
                bufs.append((name, b))
            else:
                self.int_slots[name] = (ioff, b.numel())
                ioff += b.numel()
        unknown = sorted(local - {n for n, _ in uniq} - {n for n, _ in bufs})
        if unknown:
            raise ValueError("local entries must be float state_dict entries of their own, got {}".format(unknown))

        def place(items, off, is_param):
            for name, t in items:
                self.slots[name] = Slot(name, off, t.numel(), tuple(t.shape), is_param and t.dim() == 4, is_param)
                off = _round_up(off + t.numel(), ALIGN)
            return off

        frozen = [x for x in uniq if not x[1].requires_grad]
        if frozen:
            reason = getattr(model, "frozen_params_unsupported", None)
            if reason:
                raise ValueError(reason)
            if local:
                raise ValueError("frozen parameters with client-local entries are not supported: the collective skips "
                                 "one range")
            uniq = [x for x in uniq if x[1].requires_grad]
        off = place([x for x in uniq if x[0] not in local], 0, True)
        self.local_range: Optional[Tuple[int, int]] = None
        self.frozen_range: Optional[Tuple[int, int]] = None
        if local:
            lo = off = _round_up(off, LOCAL_ALIGN)
            off = place([x for x in uniq if x[0] in local], off, True)
        if frozen:
            self.n_param = lo = _round_up(off, LOCAL_ALIGN)
            off = _round_up(place(frozen, lo, True), LOCAL_ALIGN)
            self.frozen_range = (lo, off)
        else:
            self.n_param = _round_up(off, ALIGN)
            off = self.n_param
        if local:
            off = _round_up(place([x for x in bufs if x[0] in local], off, False), LOCAL_ALIGN)
            self.local_range = (lo, off)
        off = place([x for x in bufs if x[0] not in local], off, False)
        self.n = _round_up(max(off, ALIGN), total_align)   # padded so tiles / vectors never straddle the end
        self.n_int = ioff
        if (local or frozen) and self.n % LOCAL_ALIGN:
            raise ValueError("local entries and frozen parameters need total_align to be a multiple of {}".format(
                LOCAL_ALIGN))

        if theta_storage is not None:
            assert theta_storage.numel() >= self.n and theta_storage.dtype == torch.float32
            self.theta = theta_storage[: self.n]
            self.theta.zero_()
        else:
            self.theta = torch.zeros(self.n, dtype=torch.float32, device=device)
        self.grad = torch.zeros(self.n_param, dtype=torch.float32, device=device)
        self.momentum = torch.zeros(self.n_param, dtype=torch.float32, device=device) if momentum else None
        self.adam_v = None            # AdamW second moment over the parameters, allocated by the first AdamW run
        # server optimizer state over the parameters (parallel/server_opt.py), allocated by a session built with
        # server_opt=; server_v stays None for FedAvgM
        self.server_m = None
        self.server_v = None
        self.theta_bf16 = torch.zeros(self.n, dtype=torch.bfloat16, device=device) if bf16_shadow else None
        self.global_w = torch.zeros(self.n, dtype=torch.float32, device=device) if keep_global else None
        self.int_arena = torch.zeros(max(self.n_int, 1), dtype=torch.int64, device=device)
        self._adopt()

    @property
    def skip_range(self) -> Optional[Tuple[int, int]]:
        """The one range the collective skips: the client-local range or the frozen range (never both), or None."""
        return self.local_range if self.local_range is not None else self.frozen_range

    @property
    def n_shared(self) -> int:
        """Elements the collective carries: ``n`` minus the skipped range (a multiple of 1024 when there is one)."""
        if self.skip_range is None:
            return self.n
        lo, hi = self.skip_range
        return self.n - (hi - lo)

    # ------------------------------------------------------------------
    def _owner(self, qualified: str) -> nn.Module:
        mod = self.model
        parts = qualified.split(".")[:-1]
        for p in parts:
            mod = getattr(mod, p)
        return mod

    def _view(self, flat: torch.Tensor, slot: Slot) -> torch.Tensor:
        v = flat[slot.offset: slot.offset + slot.numel]
        if slot.channels_last:
            co, ci, kh, kw = slot.shape
            return v.view(co, kh, kw, ci).permute(0, 3, 1, 2)
        return v.view(slot.shape)

    @torch.no_grad()
    def _adopt(self) -> None:
        for name, slot in self.slots.items():
            owner = self._owner(name)
            leaf = name.split(".")[-1]
            view = self._view(self.theta, slot)
            if slot.is_param:
                p = getattr(owner, leaf)
                view.copy_(p.detach().to(self.device))
                p.data = view
                p.grad = self._view(self.grad, slot) if slot.offset < self.n_param else None
                if self.theta_bf16 is not None:
                    sh = self.theta_bf16[slot.offset: slot.offset + slot.numel]
                    sh = sh.view(slot.shape[0], -1) if len(slot.shape) >= 2 else sh.view(slot.shape)
                    # plain attribute (not a registered buffer): stays out of state_dict
                    object.__setattr__(owner, leaf + "_bf16", sh)
            else:
                b = getattr(owner, leaf)
                view.copy_(b.detach().to(self.device))
                owner._buffers[leaf] = view
        for name, (ioff, n) in self.int_slots.items():
            owner = self._owner(name)
            leaf = name.split(".")[-1]
            b = getattr(owner, leaf)
            view = self.int_arena[ioff: ioff + n].view(b.shape)
            view.copy_(b.detach().to(self.device))
            owner._buffers[leaf] = view
        self.sync_shadow()
        if self.global_w is not None:
            self.global_w.copy_(self.theta)

    # ------------------------------------------------------------------
    @torch.no_grad()
    def sync_shadow(self) -> None:
        """Refresh the bf16 shadow from the fp32 master (after load_state_dict etc.)."""
        if self.theta_bf16 is None:
            return
        if self.theta.is_cuda:
            from ..ops import functional as F
            F.cast(self.theta, torch.bfloat16, out=self.theta_bf16)
        else:
            self.theta_bf16.copy_(self.theta.to(torch.bfloat16))

    @torch.no_grad()
    def commit_global(self) -> None:
        """Declare the current weights to be the global model (start of training / after a
        manual ``load_state_dict``)."""
        if self.global_w is not None:
            self.global_w.copy_(self.theta)
        self.sync_shadow()

    def zero_grad(self) -> None:
        self.grad.zero_()

    def first_weight_slot(self) -> Optional[Slot]:
        for s in self.slots.values():
            if s.is_param and len(s.shape) >= 2:
                return s
        return None

    def nbytes(self) -> Dict[str, int]:
        out = {"theta": self.theta.numel() * 4, "grad": self.grad.numel() * 4}
        if self.momentum is not None:
            out["momentum"] = self.momentum.numel() * 4
        if self.adam_v is not None:
            out["adam_v"] = self.adam_v.numel() * 4
        if self.server_m is not None:
            out["server_m"] = self.server_m.numel() * 4
        if self.server_v is not None:
            out["server_v"] = self.server_v.numel() * 4
        if self.theta_bf16 is not None:
            out["theta_bf16"] = self.theta_bf16.numel() * 2
        if self.global_w is not None:
            out["global_w"] = self.global_w.numel() * 4
        return out

    def describe(self) -> str:
        return "ParamArena(n={}, n_param={}, n_int={}, tensors={}, device={})".format(
            self.n, self.n_param, self.n_int, len(self.slots), self.device)
