"""SCAFFOLD control variates (Karimireddy et al., ICML 2020) of one rank of the SPMD engine.

``c`` is the server control variate, replicated on every rank; ``c_i`` is client ``i``'s, kept on the rank that hosts
it and allocated (as zeros) the first time the client takes part.  All are fp32 over the arena's parameters
(``n_param`` elements, 4 bytes each per hosted client).  Per hosted participant of a round:

    corr = c - c_i                                  (before it trains; every SGD step adds corr to the gradient)
    dc   = (global - theta) / (K eta) - c           (after its K local steps at learning rate eta: option II)
    c_i += dc ;  up (+)= dc                         (up: this rank's upload of the control-variate segment)

and the round's collective applies ``c += (sum over ranks of up) / N``.  On CUDA both steps are one kernel each
(``csrc/elementwise.cu``); on CPU they are the same formulas in PyTorch.
"""
from __future__ import annotations

from typing import Dict

import torch


class ScaffoldState:
    def __init__(self, n_param: int, device):
        self.n = int(n_param)
        self.device = torch.device(device)
        self.c = torch.zeros(self.n, dtype=torch.float32, device=self.device)
        self.c_i: Dict[int, torch.Tensor] = {}
        self.corr = torch.zeros(self.n, dtype=torch.float32, device=self.device)   # read by the trainers' SGD kernels
        self.up = torch.zeros(self.n, dtype=torch.float32, device=self.device)     # the rank's summed dc

    def client(self, cid: int) -> torch.Tensor:
        ci = self.c_i.get(cid)
        if ci is None:
            ci = self.c_i[cid] = torch.zeros(self.n, dtype=torch.float32, device=self.device)
        return ci

    @torch.no_grad()
    def begin_client(self, cid: int) -> None:
        """``corr = c - c_i`` for the client about to train."""
        ci = self.client(cid)
        if self.device.type == "cuda":
            from ..ops import functional as F
            F.scaffold_corr(self.corr, self.c, ci)
        else:
            torch.sub(self.c, ci, out=self.corr)

    @torch.no_grad()
    def end_client(self, cid: int, arena, k_steps: int, lr: float, first: bool) -> None:
        """After the client trained ``k_steps`` SGD steps at ``lr`` (before the replica is reset): ``dc``, ``c_i +=
        dc`` and ``up = dc`` (``first`` hosted participant of the round) or ``up += dc``."""
        ci = self.client(cid)
        inv = 1.0 / (float(k_steps) * float(lr))
        g, t = arena.global_w[: self.n], arena.theta[: self.n]
        if self.device.type == "cuda":
            from ..ops import functional as F
            F.scaffold_dc(self.up, ci, self.c, g, t, inv, first=first)
            return
        dc = (g - t) * inv - self.c
        ci.add_(dc)
        if first:
            self.up.copy_(dc)
        else:
            self.up.add_(dc)
