"""Server-side optimizers: FedAvgM, FedAdagrad, FedYogi and FedAdam (Hsu et al. 2019; Reddi et al., "Adaptive
Federated Optimization", ICLR 2021, Algorithm 2).

The round's aggregate ``d`` (the pseudo-gradient: the mean, DP, robust or Krum update the collective applies today)
drives a stateful step on the global model ``x``, per parameter element, with state ``m = 0`` and ``v = tau^2`` at
the start and no bias correction:

    avgm     m = b1*m + d                                   x = x + lr*m
    adagrad  m = b1*m + (1-b1)*d;  v = v + d*d               x = x + lr*m / (sqrt(v) + tau)
    yogi     m as adagrad;  v = v - (1-b2)*(d*d)*sign(v - d*d)   as adagrad
    adam     m as adagrad;  v = b2*v + (1-b2)*(d*d)          as adagrad

Every operation is rounded separately, left to right as written, with ``sign(0) = 0``.  The fp32 coefficients
``b1, 1-b1, b2, 1-b2, lr, tau`` are computed once in fp64 and cast (:meth:`ServerOptConfig.coefficients`); the fused
collective (``csrc/fedavg.cu``, the ``SOPT`` instantiations) uses the same values with ``__fmul_rn`` / ``__fadd_rn`` /
``__fsqrt_rn`` / ``__fdiv_rn``, so for the same ``d`` it equals :func:`server_step_` bit for bit (up to the device's
flush of denormal results to zero).

The step covers the parameters only, ``[0, n_param)`` of the arena: float buffers (BatchNorm running statistics)
keep ``global += d`` -- an adaptive step on a running variance can drive it negative -- and the integer arena keeps its
max.  A round whose total weight is zero leaves the model and the state unchanged.  The step post-processes the
aggregate, so it changes nothing in DP-FedAvg's privacy accounting.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional, Tuple

import torch

KINDS = ("avgm", "adagrad", "yogi", "adam")


def check_server_opt(kind: str, lr, b1, b2, tau) -> Tuple[float, float, float, float]:
    """Validate ``kind`` in ``KINDS``, finite ``lr > 0`` and ``tau > 0``, and ``0 <= b1, b2 < 1``."""
    if kind not in KINDS:
        raise ValueError("server_opt must be one of {}, got {!r}".format(KINDS, kind))
    if lr is None:
        raise ValueError("a server optimizer needs server_lr: it has no default")
    out = []
    for name, x in (("server_lr", lr), ("server_tau", tau)):
        x = float(x)
        if not (math.isfinite(x) and x > 0.0):
            raise ValueError("{} must be finite and > 0, got {!r}".format(name, x))
        out.append(x)
    for name, x in (("server_beta1", b1), ("server_beta2", b2)):
        x = float(x)
        if not (0.0 <= x < 1.0):
            raise ValueError("{} must satisfy 0 <= beta < 1, got {!r}".format(name, x))
        out.append(x)
    lr, tau, b1, b2 = out
    return lr, b1, b2, tau


@dataclass
class ServerOptConfig:
    """``kind``: ``"avgm"``, ``"adagrad"``, ``"yogi"`` or ``"adam"``; ``lr``: the server learning rate (required);
    ``b1`` / ``b2``: the moment decays (``avgm`` reads only ``b1``); ``tau``: the adaptivity floor (``v`` starts at
    ``tau^2``)."""
    kind: str
    lr: float
    b1: float = 0.9
    b2: float = 0.99
    tau: float = 1e-3

    def __post_init__(self):
        self.lr, self.b1, self.b2, self.tau = check_server_opt(self.kind, self.lr, self.b1, self.b2, self.tau)

    @property
    def kind_id(self) -> int:
        return KINDS.index(self.kind)

    @property
    def needs_v(self) -> bool:
        return self.kind != "avgm"

    def coefficients(self) -> Tuple[float, ...]:
        """``(b1, 1-b1, b2, 1-b2, lr, tau)``: computed in fp64, rounded to fp32 (returned as Python floats holding the
        fp32 values): the collective and :func:`server_step_` read the same six numbers."""
        c = torch.tensor([self.b1, 1.0 - self.b1, self.b2, 1.0 - self.b2, self.lr, self.tau], dtype=torch.float64)
        return tuple(float(x) for x in c.to(torch.float32))

    def v0(self) -> float:
        """Initial second moment ``tau^2`` (fp64, then fp32)."""
        return float(torch.tensor(self.tau * self.tau, dtype=torch.float64).to(torch.float32))

    def init_state(self, n: int, device) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """Fresh ``(m, v)`` over ``n`` parameters: ``m = 0``, ``v = tau^2`` (``None`` for ``avgm``)."""
        m = torch.zeros(n, dtype=torch.float32, device=device)
        v = torch.full((n,), self.v0(), dtype=torch.float32, device=device) if self.needs_v else None
        return m, v

    def to_dict(self) -> dict:
        return {"kind": self.kind, "lr": self.lr, "b1": self.b1, "b2": self.b2, "tau": self.tau}

    @classmethod
    def from_dict(cls, d: dict) -> "ServerOptConfig":
        """Inverse of :meth:`to_dict`."""
        return cls(str(d["kind"]), float(d["lr"]), float(d.get("b1", 0.9)), float(d.get("b2", 0.99)),
                   float(d.get("tau", 1e-3)))


@torch.no_grad()
def server_step_(x: torch.Tensor, d: torch.Tensor, m: torch.Tensor, v: Optional[torch.Tensor],
                 cfg: ServerOptConfig) -> None:
    """One server step in place over fp32 tensors of the same shape: ``m``, ``v`` (``None`` for ``avgm``) and ``x``
    updated from the aggregate ``d`` in the order of the module docstring, every operation rounded separately.  The
    host implementation: the oracle of the tests and the step of :class:`NcclSession` and the ``http`` manager plane."""
    c = [torch.tensor(t, dtype=torch.float32, device=x.device) for t in cfg.coefficients()]
    b1, omb1, b2, omb2, lr, tau = c
    d = d.to(torch.float32)
    if cfg.kind == "avgm":
        m.copy_(torch.add(torch.mul(b1, m), d))
        x.copy_(torch.add(x, torch.mul(lr, m)))
        return
    m.copy_(torch.add(torch.mul(b1, m), torch.mul(omb1, d)))
    dd = torch.mul(d, d)
    if cfg.kind == "adagrad":
        v.copy_(torch.add(v, dd))
    elif cfg.kind == "yogi":
        v.copy_(torch.sub(v, torch.mul(torch.mul(omb2, dd), torch.sign(torch.sub(v, dd)))))
    else:
        v.copy_(torch.add(torch.mul(b2, v), torch.mul(omb2, dd)))
    # the correctly rounded fp32 square root: torch's vectorised fp32 sqrt on the CPU is not, the fp64 one rounded to
    # fp32 is (53 >= 2 * 24 + 2 bits, so the double rounding is exact)
    sq = torch.sqrt(v.double()).to(torch.float32)
    x.copy_(torch.add(x, torch.div(torch.mul(lr, m), torch.add(sq, tau))))


@torch.no_grad()
def apply_update_(global_w: torch.Tensor, d: torch.Tensor, n_param: int, m: torch.Tensor, v: Optional[torch.Tensor],
                  cfg: ServerOptConfig) -> None:
    """The apply phase of a server-optimizer round over a whole arena: :func:`server_step_` on ``[0, n_param)`` and
    ``global += d`` on the float buffers behind it."""
    server_step_(global_w[:n_param], d[:n_param], m, v, cfg)
    if global_w.numel() > n_param:
        global_w[n_param:].add_(d[n_param:])
