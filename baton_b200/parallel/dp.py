"""Client-level differential privacy for FedAvg (DP-FedAvg, McMahan et al., ICLR 2018).

For every participating client ``k`` of a round, ``Delta_k = theta_k - global`` over the whole float arena (parameters
and float buffers), ``s_k = min(1, C / ||Delta_k||_2)`` (0 when the norm is not finite -- the client still counts), and

    global <- global + (sum_k s_k Delta_k + sigma C z) / m,        m = number of participants,

with uniform weights and ``z[i]`` a pure function of ``(seed, round, i)``: Philox4x32-10 (key ``(seed_lo, seed_hi)``,
counter ``(q_lo, q_hi, round, 0)``, ``q = i // 4``) and Box-Muller, as in ``csrc/dp.cuh``.  This module holds the
configuration, the host sampler (test oracle and the noise of the host paths) and the RDP accountant.
"""
from __future__ import annotations

import math
import secrets
from dataclasses import dataclass, field
from typing import Dict, Iterable, Optional, Sequence, Tuple

import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF


@dataclass
class DPConfig:
    """``clip`` = C, ``noise_multiplier`` = sigma (noise std on the sum of clipped updates: sigma * C).

    ``seed=None`` draws a fresh 64-bit Philox key per process (``secrets.randbits(64)``).  Anyone who knows the seed can
    regenerate and subtract the noise, which voids the guarantee: pass an explicit seed only for tests and reproductions.
    In a multi-process job every rank must use the same key, so the SPMD engine takes rank 0's."""
    clip: float
    noise_multiplier: float = 0.0
    seed: Optional[int] = field(default=None)

    def __post_init__(self):
        self.clip, self.noise_multiplier = check_dp(self.clip, self.noise_multiplier)
        if self.clip <= 0.0:
            raise ValueError("DP needs a clip norm > 0, got {!r}".format(self.clip))
        if self.seed is None:
            self.seed = secrets.randbits(64)
        self.seed = int(self.seed) & 0xFFFFFFFFFFFFFFFF

    @property
    def noise_std(self) -> float:
        """Standard deviation of the noise on the SUM of the clipped updates."""
        return self.noise_multiplier * self.clip


def check_dp(clip: float, noise_multiplier: float) -> Tuple[float, float]:
    """Validate ``(C, sigma)``: both finite and >= 0, and noise needs a clip norm (the sensitivity).  ``C = 0`` means
    DP is off."""
    clip, nm = float(clip), float(noise_multiplier)
    for name, v in (("dp_clip", clip), ("dp_noise_multiplier", nm)):
        if not (0.0 <= v < float("inf")):
            raise ValueError("{} must be a finite number >= 0, got {!r}".format(name, v))
    if nm > 0.0 and clip == 0.0:
        raise ValueError("dp_noise_multiplier > 0 needs dp_clip > 0 (the noise is scaled by the clip norm)")
    return clip, nm


# ---------------------------------------------------------------------------------------------------- host sampler
def philox4x32_10(counter: np.ndarray, key: Tuple[int, int]) -> np.ndarray:
    """Philox4x32-10 of uint32 counters ``[..., 4]`` under ``key = (k0, k1)``; returns uint32 ``[..., 4]``."""
    c = [counter[..., j].astype(np.uint64) for j in range(4)]
    k0, k1 = np.uint64(key[0] & _MASK), np.uint64(key[1] & _MASK)
    m0, m1, mask = np.uint64(M0), np.uint64(M1), np.uint64(_MASK)
    for _ in range(10):
        p0, p1 = c[0] * m0, c[2] * m1
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & mask, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & mask]
        k0, k1 = (k0 + np.uint64(W0)) & mask, (k1 + np.uint64(W1)) & mask
    return np.stack(c, axis=-1).astype(np.uint32)


def normals(seed: int, round_index: int, n: int, start: int = 0) -> np.ndarray:
    """``z[start : start + n]`` of the stream ``(seed, round)`` in float64 (the kernel computes the same in fp32)."""
    if n <= 0:
        return np.zeros(0, dtype=np.float64)
    q0, q1 = start // 4, (start + n + 3) // 4
    q = np.arange(q0, q1, dtype=np.uint64)
    ctr = np.stack([q & np.uint64(_MASK), q >> np.uint64(32), np.full_like(q, round_index & _MASK),
                    np.zeros_like(q)], axis=-1)
    x = philox4x32_10(ctr, (seed & _MASK, (seed >> 32) & _MASK)).astype(np.float64)
    u = (x + 0.5) * 2.0 ** -32
    r0, r1 = np.sqrt(-2.0 * np.log(u[:, 0])), np.sqrt(-2.0 * np.log(u[:, 2]))
    a0, a1 = 2.0 * np.pi * u[:, 1], 2.0 * np.pi * u[:, 3]
    z = np.stack([r0 * np.cos(a0), r0 * np.sin(a0), r1 * np.cos(a1), r1 * np.sin(a1)], axis=-1).reshape(-1)
    off = start - 4 * q0
    return z[off: off + n]


def norm_to_factor(norm: float, clip: float) -> float:
    """``min(1, C / norm)``; 0 for a norm that is not finite."""
    if not math.isfinite(norm):
        return 0.0
    return 1.0 if norm <= clip else float(clip) / norm


def clip_factor(delta, clip: float) -> Tuple[float, float]:
    """``(s, ||delta||_2)`` of one client's update (a tensor or a sequence of tensors), the norm in float64."""
    import torch
    parts = [delta] if isinstance(delta, torch.Tensor) else list(delta)
    sq = sum(float(p.detach().double().pow(2).sum()) for p in parts)
    norm = math.sqrt(sq) if math.isfinite(sq) else float("nan")
    return norm_to_factor(norm, clip), norm


# ---------------------------------------------------------------------------------------------------- accountant
# RDP of the sampled Gaussian mechanism (Mironov, Talwar, Zhang 2019): integer orders by the binomial expansion of
# A_alpha, fractional orders by the two-sided series; composition adds RDP over rounds; (epsilon, delta) by the
# conversion of Balle et al. 2020 (Theorem 21), as Opacus reports it.
DEFAULT_ORDERS = tuple([1.0 + x / 10.0 for x in range(1, 100)] + [float(a) for a in range(12, 64)])


def _log_add(a: float, b: float) -> float:
    lo, hi = min(a, b), max(a, b)
    if lo == -math.inf:
        return hi
    return hi + math.log1p(math.exp(lo - hi))


def _log_sub(a: float, b: float) -> float:
    if b == -math.inf:
        return a
    if a <= b:
        return -math.inf          # the series terms cancel to below the precision
    return a + math.log1p(-math.exp(b - a))


def _log_erfc(x: float) -> float:
    if x < 20.0:
        return math.log(math.erfc(x))
    # asymptotic expansion: erfc(x) ~ exp(-x^2) / (x sqrt(pi)) (1 - 1/(2x^2) + 3/(4x^4) - 15/(8x^6))
    x2 = x * x
    return -x2 - math.log(x) - 0.5 * math.log(math.pi) + math.log1p(-0.5 / x2 + 0.75 / x2 ** 2 - 1.875 / x2 ** 3)


def _log_binom(n: float, k: int) -> Tuple[float, float]:
    """(log |C(n, k)|, sign) for real n >= 0 and integer k >= 0."""
    if k == 0:
        return 0.0, 1.0
    sign = 1.0
    logc = 0.0
    for j in range(k):
        t = (n - j) / (j + 1)
        if t == 0.0:
            return -math.inf, 0.0
        if t < 0:
            sign = -sign
        logc += math.log(abs(t))
    return logc, sign


def _log_a_int(q: float, sigma: float, alpha: int) -> float:
    out = -math.inf
    for i in range(alpha + 1):
        lc, _ = _log_binom(alpha, i)
        term = lc + i * math.log(q) + (alpha - i) * math.log1p(-q) + (i * i - i) / (2.0 * sigma ** 2)
        out = _log_add(out, term)
    return out


def _log_a_frac(q: float, sigma: float, alpha: float) -> float:
    log_a0 = log_a1 = -math.inf
    z0 = sigma ** 2 * math.log(1.0 / q - 1.0) + 0.5
    i = 0
    while True:
        lc, sign = _log_binom(alpha, i)
        j = alpha - i
        log_t0 = lc + i * math.log(q) + j * math.log1p(-q)
        log_t1 = lc + j * math.log(q) + i * math.log1p(-q)
        log_e0 = math.log(0.5) + _log_erfc((i - z0) / (math.sqrt(2.0) * sigma))
        log_e1 = math.log(0.5) + _log_erfc((z0 - j) / (math.sqrt(2.0) * sigma))
        log_s0 = log_t0 + (i * i - i) / (2.0 * sigma ** 2) + log_e0
        log_s1 = log_t1 + (j * j - j) / (2.0 * sigma ** 2) + log_e1
        if sign > 0:
            log_a0, log_a1 = _log_add(log_a0, log_s0), _log_add(log_a1, log_s1)
        elif sign < 0:
            log_a0, log_a1 = _log_sub(log_a0, log_s0), _log_sub(log_a1, log_s1)
        i += 1
        if max(log_s0, log_s1) < -30 or i > 10000:
            break
    return _log_add(log_a0, log_a1)


def rdp_sampled_gaussian(q: float, sigma: float, alpha: float) -> float:
    """Renyi DP of order ``alpha`` of ONE round: Gaussian noise ``sigma`` (in units of the sensitivity), each client
    included with probability ``q``."""
    q, sigma, alpha = float(q), float(sigma), float(alpha)
    if q <= 0.0:
        return 0.0
    if sigma <= 0.0:
        return math.inf
    if q >= 1.0:
        return alpha / (2.0 * sigma ** 2)
    if math.isinf(alpha):
        return math.inf
    if float(alpha).is_integer():
        log_a = _log_a_int(q, sigma, int(alpha))
    else:
        log_a = _log_a_frac(q, sigma, alpha)
    return log_a / (alpha - 1.0)


def epsilon_from_rdp(rdp: Sequence[float], orders: Sequence[float], delta: float) -> Tuple[float, float]:
    """Best ``(epsilon, order)`` over the orders (Balle et al. 2020, Theorem 21)."""
    if not (0.0 < delta < 1.0):
        raise ValueError("delta must lie in (0, 1), got {!r}".format(delta))
    best = (math.inf, float("nan"))
    for r, a in zip(rdp, orders):
        if not math.isfinite(r) or a <= 1.0:
            continue
        eps = r - (math.log(delta) + math.log(a)) / (a - 1.0) + math.log((a - 1.0) / a)
        if eps < best[0]:
            best = (max(eps, 0.0), float(a))
    return best


class RDPAccountant:
    """Privacy spent by a sequence of DP-FedAvg rounds.  Every round records its sampling rate ``q`` = participants /
    population.  The engine and the manager draw a fixed-size sample; accounting for it as Poisson sampling at rate
    ``k / K`` is the usual approximation (exact when everyone participates, ``q = 1``)."""

    def __init__(self, noise_multiplier: float, orders: Iterable[float] = DEFAULT_ORDERS):
        self.noise_multiplier = float(noise_multiplier)
        self.orders = tuple(float(a) for a in orders)
        self.history: Dict[float, int] = {}          # q -> rounds

    @property
    def rounds(self) -> int:
        return sum(self.history.values())

    def step(self, q: float, rounds: int = 1) -> None:
        q = min(max(float(q), 0.0), 1.0)
        self.history[q] = self.history.get(q, 0) + int(rounds)

    def rdp(self) -> list:
        out = [0.0] * len(self.orders)
        for q, t in self.history.items():
            for i, a in enumerate(self.orders):
                out[i] += t * rdp_sampled_gaussian(q, self.noise_multiplier, a)
        return out

    def get_privacy_spent(self, delta: float) -> Tuple[float, float]:
        """``(epsilon, order)`` for ``delta``; ``(0, nan)`` before the first round, ``(inf, nan)`` without noise."""
        if not self.history:
            return 0.0, float("nan")
        if self.noise_multiplier <= 0.0:
            return math.inf, float("nan")
        return epsilon_from_rdp(self.rdp(), self.orders, delta)
