"""Secure aggregation (Bonawitz et al., CCS 2017, without dropout recovery): pairwise-masked fixed-point uploads.

Semantics, shared by the fused collective (``csrc/secagg.cuh``, ``Agg::secagg`` in ``csrc/fedavg.cu``), the standalone
encode kernel and :class:`~baton_b200.parallel.fedavg.NcclSession`:

* Participants are the live ranks with ``n_k > 0``.  ``N`` is the fp32 sum of the counts in live-rank order,
  ``inv = 1 / N`` and ``w_k = n_k * inv``, each operation rounded once (IEEE, fp32).
* Encode: ``y = clamp(x, -R, R)`` of every update element ``x = theta - global`` (NaN -> 0, +-inf -> +-R; a clamped or
  non-finite element counts as *saturated*), ``q = int32(rint_even(fp32(w_k * y) * 2^f))`` with
  ``f = 30 - ceil(log2 R)``: ``|sum_k q_k| <= 2^30 + P / 2`` never wraps.
* Mask: ``u_k = q_k + sum_{j > k} S_kj - sum_{j < k} S_jk  (mod 2^32)`` over the participants ``j != k``, ``S_ij`` the
  ChaCha20 keystream (RFC 8439) of pair ``(i, j)``: one 32-bit word per element, block counter ``e / 16``, nonce
  ``(epoch, 0, 0)``.  Pair keys come from an X25519 exchange at session start (:func:`agree_keys`).
* Decode: ``d = fp32(int32(sum_k u_k mod 2^32)) * 2^-f``, applied as ``global += d`` (or as the server optimizer's
  pseudo-gradient).  The masks cancel exactly, so ``d`` does not depend on the keys or the nonce.

Not masked: the counts ``n_k``, the per-epoch losses and the integer side arena.
"""
from __future__ import annotations

import hashlib
import hmac
import math
import secrets
import struct
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import numpy as np

MAX_ARENA = 1 << 36          # the 32-bit block counter e / 16 covers 2^36 elements
RANGE_MIN, RANGE_MAX = 2.0 ** -20, 2.0 ** 20


@dataclass(frozen=True)
class SecAggConfig:
    """``range``: the clamp ``R`` of every update element (fp32; 2^-20 <= R <= 2^20)."""
    range: float = 64.0

    def __post_init__(self):
        r = self.range
        if isinstance(r, bool) or not isinstance(r, (int, float)) or not math.isfinite(float(r)):
            raise ValueError("secagg_range must be a finite number, got {!r}".format(r))
        r32 = float(np.float32(r))
        if not (RANGE_MIN <= r32 <= RANGE_MAX):
            raise ValueError("secagg_range must be in [2^-20, 2^20], got {!r}".format(r))
        object.__setattr__(self, "range", r32)

    @property
    def frac_bits(self) -> int:
        """``f = 30 - ceil(log2 R)``."""
        return frac_bits(self.range)


def frac_bits(R: float) -> int:
    m, e = math.frexp(float(R))          # R = m 2^e, 0.5 <= m < 1
    return 30 - (e - 1 if m == 0.5 else e)


# ---------------------------------------------------------------- key agreement (RFC 7748 X25519, RFC 5869 HKDF)
_P = 2 ** 255 - 19
_A24 = 121665


def x25519(k: bytes, u: bytes) -> bytes:
    """X25519 (RFC 7748 section 5) with Python integers.  Not constant-time."""
    if len(k) != 32 or len(u) != 32:
        raise ValueError("X25519 takes 32-byte scalars and u-coordinates")
    kb = bytearray(k)
    kb[0] &= 248
    kb[31] &= 127
    kb[31] |= 64
    scalar = int.from_bytes(kb, "little")
    x1 = int.from_bytes(u, "little") & ((1 << 255) - 1)
    x2, z2, x3, z3, swap = 1, 0, x1, 1, 0
    for t in reversed(range(255)):
        bit = (scalar >> t) & 1
        swap ^= bit
        if swap:
            x2, x3, z2, z3 = x3, x2, z3, z2
        swap = bit
        a, b = (x2 + z2) % _P, (x2 - z2) % _P
        aa, bb = a * a % _P, b * b % _P
        e = (aa - bb) % _P
        c, d = (x3 + z3) % _P, (x3 - z3) % _P
        da, cb = d * a % _P, c * b % _P
        x3 = (da + cb) ** 2 % _P
        z3 = x1 * (da - cb) ** 2 % _P
        x2 = aa * bb % _P
        z2 = e * (aa + _A24 * e) % _P
    if swap:
        x2, z2 = x3, z3
    return (x2 * pow(z2, _P - 2, _P) % _P).to_bytes(32, "little")


X25519_BASE = (9).to_bytes(32, "little")


def hkdf_sha256(ikm: bytes, salt: bytes, info: bytes, length: int = 32) -> bytes:
    """HKDF-SHA256 (RFC 5869): extract, then expand to ``length`` bytes."""
    if not (0 < length <= 255 * 32):
        raise ValueError("HKDF output length out of range")
    prk = hmac.new(salt if salt else bytes(32), ikm, hashlib.sha256).digest()
    out, t, i = b"", b"", 1
    while len(out) < length:
        t = hmac.new(prk, t + info + bytes([i]), hashlib.sha256).digest()
        out += t
        i += 1
    return out[:length]


def pair_key(sk_i: bytes, pk_j: bytes, i: int, j: int, pks: Sequence[bytes]) -> bytes:
    """The 32-byte ChaCha20 key of the pair ``(min(i, j), max(i, j))`` as rank ``i`` derives it from its secret and
    peer ``j``'s public key; ``pks``: every rank's public key in rank order (the salt)."""
    shared = x25519(sk_i, pk_j)
    if shared == bytes(32):
        raise ValueError("X25519 gave the all-zero shared secret (RFC 7748 section 6.1): peer {}'s key is "
                         "invalid".format(j))
    lo, hi = min(i, j), max(i, j)
    salt = hashlib.sha256(b"".join(pks)).digest()
    return hkdf_sha256(shared, salt, b"baton secagg" + struct.pack("<II", lo, hi))


def agree_keys(group=None) -> Dict[int, bytes]:
    """``{peer rank: 32-byte pair key}`` for this rank: a fresh X25519 secret, the public keys exchanged with one
    ``all_gather_object`` over ``group`` (which the rendezvous authenticates, as it does the rest of the job).  Empty
    for a single rank."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return {}
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    sk = secrets.token_bytes(32)
    pk = x25519(sk, X25519_BASE)
    pks: List[bytes] = [b""] * world
    dist.all_gather_object(pks, pk, group=group)
    return {j: pair_key(sk, pks[j], rank, j, pks) for j in range(world) if j != rank}


def key_words(key: bytes) -> List[int]:
    """A 32-byte key as the eight little-endian uint32 words ChaCha20 reads."""
    return list(struct.unpack("<8I", key))


# ---------------------------------------------------------------- ChaCha20 (RFC 8439) keystream
_SIGMA = np.array([0x61707865, 0x3320646E, 0x79622D32, 0x6B206574], dtype=np.uint32)


def _rotl(x, n):
    return (x << np.uint32(n)) | (x >> np.uint32(32 - n))


def chacha20_blocks(key: Sequence[int], counters: np.ndarray, nonce: Sequence[int]) -> np.ndarray:
    """``[len(counters), 16]`` uint32 output words of the ChaCha20 block function."""
    nb = len(counters)
    init = np.empty((16, nb), dtype=np.uint32)
    init[0:4] = _SIGMA[:, None]
    init[4:12] = np.asarray(key, dtype=np.uint32)[:, None]
    init[12] = np.asarray(counters, dtype=np.uint32)
    init[13:16] = np.asarray(nonce, dtype=np.uint32)[:, None]
    x = [init[i].copy() for i in range(16)]

    def qr(a, b, c, d):
        x[a] += x[b]; x[d] = _rotl(x[d] ^ x[a], 16)
        x[c] += x[d]; x[b] = _rotl(x[b] ^ x[c], 12)
        x[a] += x[b]; x[d] = _rotl(x[d] ^ x[a], 8)
        x[c] += x[d]; x[b] = _rotl(x[b] ^ x[c], 7)

    with np.errstate(over="ignore"):
        for _ in range(10):
            qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
            qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
        out = np.stack(x) + init
    return out.T.copy()


def keystream(key: Sequence[int], nonce: Sequence[int], n: int, counter0: int = 0) -> np.ndarray:
    """``n`` uint32 keystream words: word ``e`` is word ``e % 16`` of block ``counter0 + e / 16``."""
    nb = -(-int(n) // 16)
    if counter0 + nb > 1 << 32:
        raise ValueError("the ChaCha20 block counter would wrap")
    ctr = (np.arange(nb, dtype=np.uint64) + np.uint64(counter0)).astype(np.uint32)
    return chacha20_blocks(key, ctr, nonce).reshape(-1)[:n]


# ---------------------------------------------------------------- encode / mask / decode
def weights(counts: Sequence[float]) -> Tuple[np.ndarray, float]:
    """``(w, N)``: the kernel's fp32 weights ``w_k = n_k * (1 / N)`` of the counts in live-rank order (0 where
    ``n_k == 0``), ``N`` their fp32 sum in that order."""
    c = np.asarray(counts, dtype=np.float32)
    total = np.float32(0.0)
    for x in c:
        total = np.float32(total + x)
    inv = np.float32(1.0) / total if total > 0 else np.float32(0.0)
    return (c * inv).astype(np.float32), float(total)


def encode(x: np.ndarray, w: float, R: float, f: int) -> Tuple[np.ndarray, int]:
    """``(q, saturated)``: the int32 fixed-point encoding of the fp32 update ``x`` at weight ``w``."""
    x = np.asarray(x, dtype=np.float32)
    R32 = np.float32(R)
    nan = np.isnan(x)
    sat = nan | (np.abs(x) > R32)
    y = np.where(nan, np.float32(0.0), np.clip(x, -R32, R32)).astype(np.float32)
    p = (np.float32(w) * y).astype(np.float32)
    s = (p * np.float32(2.0 ** f)).astype(np.float32)
    return np.rint(s).astype(np.int32), int(sat.sum())


def mask(q: np.ndarray, peers: Sequence[Tuple[Sequence[int], int]], nonce: Sequence[int],
         counter0: int = 0) -> np.ndarray:
    """``u = q + sum sign * S(key)  (mod 2^32)`` as uint32; ``peers``: ``(key words, sign +1 / -1)`` per peer."""
    u = np.asarray(q).astype(np.int32).view(np.uint32).copy()
    with np.errstate(over="ignore"):
        for key, sign in peers:
            s = keystream(key, nonce, u.size, counter0)
            u = u + s if sign > 0 else u - s
    return u


def decode(total: np.ndarray, f: int) -> np.ndarray:
    """``fp32(int32(total)) * 2^-f`` of the uint32 sum of the masked uploads."""
    t = np.asarray(total).astype(np.uint32).view(np.int32)
    return (t.astype(np.float32) * np.float32(2.0 ** -f)).astype(np.float32)


def peer_list(rank: int, participants: Sequence[int], keys: Dict[int, Sequence[int]]):
    """``(key words, sign)`` of every other participant: +1 for a higher rank, -1 for a lower one."""
    return [(keys[j], 1 if j > rank else -1) for j in participants if j != rank]


def reference_round(updates: Sequence[np.ndarray], counts: Sequence[float], R: float,
                    keys: Dict[Tuple[int, int], Sequence[int]], nonce: Sequence[int]) -> Tuple[np.ndarray, int]:
    """The whole secure round on the host over simulated parties (index = rank, all live): every participant's
    masked upload, their sum mod 2^32 and its decode ``d``; ``keys[(i, j)]``, ``i < j``: the pair keys.  Returns
    ``(d, saturated over all parties)``."""
    f = frac_bits(R)
    w, _ = weights(counts)
    parts = [k for k, c in enumerate(counts) if c > 0]
    total = np.zeros(np.asarray(updates[0]).size, dtype=np.uint32)
    sat = 0
    with np.errstate(over="ignore"):
        for k in parts:
            q, s = encode(updates[k], float(w[k]), R, f)
            sat += s
            mine = {j: keys[(min(j, k), max(j, k))] for j in parts if j != k}
            total = total + mask(q, peer_list(k, parts, mine), nonce)
    return decode(total, f), sat
