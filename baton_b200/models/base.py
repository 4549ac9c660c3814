"""The user-model contract of the federation.

Parity target: demo ``Model`` (reference demo.py:15-49): an ``nn.Module`` with
  * ``name``      -- experiment name shared by manager and workers (demo.py:16),
  * ``__hash__``  -- hash of the (key, shape) signature so both sides derive the
                     same fallback name (demo.py:26-27),
  * ``train(X, y, n_epoch=32, lr=0.001, batch_size=32, verbose=True)``
                  -- the local-SGD loop, returning per-epoch losses (demo.py:29-49).

The reference overrides ``nn.Module.train(mode)`` to do this (quirk 11).
``FederatedModule.train`` keeps that call shape *and* the stock meaning:
``model.train()`` / ``model.train(False)`` still toggle training mode, while
``model.train(X, y, n_epoch=...)`` runs local SGD.  The loop is also available
under the unambiguous name ``local_train``.
"""
from __future__ import annotations

from typing import List, Optional

import torch
from torch import nn

from ..train import run_local_sgd


class FederatedModule(nn.Module):
    name: Optional[str] = None
    loss_kind = "mse"
    default_lr = 0.001
    default_batch_size = 32
    default_momentum = 0.0
    default_weight_decay = 0.0
    default_prox_mu = 0.0          # FedProx coefficient (0: plain SGD)
    default_optimizer = "sgd"      # local optimizer: "sgd" or "adamw" (betas / eps: local_train keywords)
    head = None                    # state_dict prefix of the classifier head (local_keys="head"), None: no head

    def signature(self):
        return tuple((k, *v.shape) for k, v in self.state_dict().items())

    def __hash__(self):
        return hash(self.signature())

    def __eq__(self, other):
        return self is other

    # -- local SGD ------------------------------------------------------------
    def local_train(self, X, y, n_epoch: int = 32, lr: Optional[float] = None,
                    batch_size: Optional[int] = None, verbose: bool = False, **kw) -> List[float]:
        lr = self.default_lr if lr is None else lr
        batch_size = self.default_batch_size if batch_size is None else batch_size
        kw.setdefault("momentum", self.default_momentum)
        kw.setdefault("weight_decay", self.default_weight_decay)
        kw.setdefault("prox_mu", self.default_prox_mu)
        kw.setdefault("optimizer", self.default_optimizer)
        trainer = getattr(self, "_graphed_trainer", None)
        if X.is_cuda and trainer is not None:
            return trainer.run(X, y, n_epoch=n_epoch, lr=lr, batch_size=batch_size, **kw)
        return run_local_sgd(self, X, y, n_epoch=n_epoch, lr=lr, batch_size=batch_size,
                             loss=self.loss_kind, verbose=verbose, **kw)

    def train(self, *args, **kwargs):  # noqa: D401 - dual-purpose by design
        """``train()`` / ``train(bool)`` -> ``nn.Module.train``;
        ``train(X, y, n_epoch=...)`` -> local SGD (reference contract)."""
        if not args and not kwargs:
            return nn.Module.train(self, True)
        if args and isinstance(args[0], bool) and len(args) == 1 and not kwargs:
            return nn.Module.train(self, args[0])
        if "mode" in kwargs and len(kwargs) == 1 and not args:
            return nn.Module.train(self, kwargs["mode"])
        return self.local_train(*args, **kwargs)
