"""Synthetic federated shards.

Parity target: demo ``LinearTestWorker.get_data`` (reference demo.py:52-59):
every round draws ``n in [5, 20]``, ``X ~ N(0,1)`` of shape ``[32n, 10]`` and
``y = (p * X).sum(1)`` for a fixed ground-truth ``p`` (demo.py:55); the varying
``n_samples = 32n`` is what exercises the FedAvg weighting.

Added for the benchmark configurations: class-conditional image shards (32x32) and
token shards with three label partitions across K clients -- IID, label-skew
(each client sees ``classes_per_client`` classes) and Dirichlet(alpha) non-IID
(the standard FL benchmark partition; alpha=0.1 is highly skewed).

Held-out data for evaluating the global model: ``holdout_image_shard`` /
``holdout_token_shard`` draw IID, class-balanced samples of the same classes
(the same image class means, the same vocabulary bands) from a random stream
that no training client uses, so accuracy on them measures generalisation.

Personalized FL (FedBN / FedPer): ``image_shard(..., shift > 0)`` gives each client its own per-channel contrast and
brightness change (FedBN's feature-shift setting), and ``client_holdout_image_shard`` draws held-out samples from one
client's own label distribution and shift, for the per-client accuracy those methods report.
"""
from __future__ import annotations

import random
from dataclasses import dataclass
from typing import Sequence, List, Optional, Tuple

import torch

#: ground-truth weights of the reference regression task (demo.py:55)
LINEAR_TRUTH = (11.0, 5.0, 3.0, 2.0, 5.0, 6.0, 2.0, 7.0, 8.0, 1.0)


def linear_regression_shard(n: Optional[int] = None, rng: Optional[random.Random] = None,
                            generator: Optional[torch.Generator] = None,
                            device="cpu") -> Tuple[Tuple[torch.Tensor, torch.Tensor], int]:
    """Fresh regression shard; ``y`` has shape ``(N, 1)`` (fixes quirk 13)."""
    rng = rng or random
    if n is None:
        n = rng.randint(5, 20)
    p = torch.tensor(LINEAR_TRUTH)
    X = torch.randn(32 * n, len(LINEAR_TRUTH), generator=generator)
    y = (p * X).sum(1, keepdim=True)
    return (X.to(device), y.to(device)), 32 * n


@dataclass
class ShardSpec:
    """Label distribution of one client."""
    client: int
    class_probs: torch.Tensor  # [num_classes], sums to 1
    n_samples: int


def iid_label_shards(k: int, num_classes: int, n_samples: "int | Sequence[int]") -> List[ShardSpec]:
    ns = [n_samples] * k if isinstance(n_samples, int) else list(n_samples)
    p = torch.full((num_classes,), 1.0 / num_classes)
    return [ShardSpec(i, p.clone(), ns[i]) for i in range(k)]


def label_skew_shards(k: int, num_classes: int, n_samples: "int | Sequence[int]",
                      classes_per_client: int = 2) -> List[ShardSpec]:
    ns = [n_samples] * k if isinstance(n_samples, int) else list(n_samples)
    out = []
    for i in range(k):
        p = torch.zeros(num_classes)
        for j in range(classes_per_client):
            p[(i * classes_per_client + j) % num_classes] = 1.0 / classes_per_client
        out.append(ShardSpec(i, p, ns[i]))
    return out


def dirichlet_label_shards(k: int, num_classes: int, n_samples: "int | Sequence[int]",
                           alpha: float = 0.1, seed: int = 0) -> List[ShardSpec]:
    """Per-client class proportions ~ Dirichlet(alpha * 1)."""
    ns = [n_samples] * k if isinstance(n_samples, int) else list(n_samples)
    g = torch.Generator().manual_seed(seed)
    conc = torch.full((num_classes,), float(alpha))
    # torch.distributions has no generator argument; sample gammas directly
    gam = torch._standard_gamma(conc.expand(k, num_classes).contiguous(), generator=g).clamp_min(1e-30)
    probs = gam / gam.sum(1, keepdim=True)
    return [ShardSpec(i, probs[i], ns[i]) for i in range(k)]


def _labels_for(spec: ShardSpec, generator: Optional[torch.Generator]) -> torch.Tensor:
    return torch.multinomial(spec.class_probs, spec.n_samples, replacement=True, generator=generator)


# seed offset of the held-out stream: client k trains on seed * mult + 1000003 * (k + 1) and the class means use ``seed``
# itself; seed * mult + 500009 equals neither for any seed >= 0
_HOLDOUT_OFFSET = 500009


def _stream(seed: int, mult: int, client: int) -> torch.Generator:
    """Sample generator of training client ``client``."""
    return torch.Generator().manual_seed(seed * mult + 1000003 * (client + 1))


# seed offsets of a client's feature shift and of its own held-out samples, on top of its training stream's seed; neither
# equals another client's training stream, the global held-out stream or the other for any seed >= 0
_SHIFT_OFFSET = 250013
_CLIENT_HOLDOUT_OFFSET = 500009


def _client_shift(seed: int, client: int, channels: int, shift: float):
    """Client ``client``'s per-channel ``(contrast, brightness)``: ``exp(shift z1)`` and ``shift z2``, or None for
    ``shift == 0``."""
    if shift == 0.0:
        return None
    g = torch.Generator().manual_seed(seed * 7919 + 1000003 * (client + 1) + _SHIFT_OFFSET)
    z = torch.randn(2, channels, generator=g)
    return torch.exp(shift * z[0]), shift * z[1]


def _holdout_stream(seed: int, mult: int) -> torch.Generator:
    """Sample generator of the held-out data: a stream no training client and no class-mean draw uses."""
    return torch.Generator().manual_seed(seed * mult + _HOLDOUT_OFFSET)


def class_means(num_classes: int, *, channels: int = 3, size: int = 32, seed: int = 0) -> torch.Tensor:
    """The per-class mean images ``[num_classes, size, size, channels]`` behind :func:`image_shard`."""
    gm = torch.Generator().manual_seed(seed)
    return torch.randn(num_classes, size, size, channels, generator=gm) * 0.5


def _images(means, y, g, noise, dtype, channels_last, pin, affine=None):
    X = means[y] + noise * torch.randn(y.numel(), *means.shape[1:], generator=g)
    if affine is not None:
        X = X * affine[0] + affine[1]          # per channel (the last axis)
    if not channels_last:
        X = X.permute(0, 3, 1, 2).contiguous()
    X = X.to(dtype)
    if pin and torch.cuda.is_available():
        X, y = X.pin_memory(), y.pin_memory()
    return X, y


def _balanced_labels(num_classes: int, n: int, g: torch.Generator) -> torch.Tensor:
    """``n`` labels, every class ``n // num_classes`` or one more times, in random order."""
    return (torch.arange(n) % num_classes)[torch.randperm(n, generator=g)]


def image_shard(spec: ShardSpec, *, channels: int = 3, size: int = 32, seed: int = 0,
                dtype=torch.float32, channels_last: bool = True, pin: bool = False,
                noise: float = 1.0, shift: float = 0.0) -> Tuple[torch.Tensor, torch.Tensor]:
    """Class-conditional Gaussian images: each class has a fixed random mean
    pattern (shared across clients through ``seed``), samples are mean + noise.
    Returned as NHWC when ``channels_last`` (the layout the conv kernels use).
    ``shift > 0``: the client's images also get its own per-channel contrast ``exp(shift z1)`` and brightness
    ``shift z2`` (``z`` standard normal from a client-seeded stream); 0 returns the unshifted images."""
    means = class_means(spec.class_probs.numel(), channels=channels, size=size, seed=seed)
    g = _stream(seed, 7919, spec.client)
    y = _labels_for(spec, g)
    return _images(means, y, g, noise, dtype, channels_last, pin, _client_shift(seed, spec.client, channels, shift))


def client_holdout_image_shard(spec: ShardSpec, n: int, *, channels: int = 3, size: int = 32, seed: int = 0,
                               dtype=torch.float32, channels_last: bool = True, pin: bool = False,
                               noise: float = 1.0, shift: float = 0.0) -> Tuple[torch.Tensor, torch.Tensor]:
    """``n`` held-out images of client ``spec.client``: its label distribution and (``shift``) its feature shift, the
    class means of :func:`image_shard`, from a stream no training client and no global held-out set draws from."""
    means = class_means(spec.class_probs.numel(), channels=channels, size=size, seed=seed)
    g = torch.Generator().manual_seed(seed * 7919 + 1000003 * (spec.client + 1) + _CLIENT_HOLDOUT_OFFSET)
    y = torch.multinomial(spec.class_probs, n, replacement=True, generator=g)
    return _images(means, y, g, noise, dtype, channels_last, pin, _client_shift(seed, spec.client, channels, shift))


def holdout_image_shard(num_classes: int, n: int, *, channels: int = 3, size: int = 32, seed: int = 0,
                        dtype=torch.float32, channels_last: bool = True, pin: bool = False,
                        noise: float = 1.0) -> Tuple[torch.Tensor, torch.Tensor]:
    """Held-out images for evaluation: class-balanced labels, the class means of :func:`image_shard` with the same
    ``seed``, and noise from a random stream no training client draws from."""
    means = class_means(num_classes, channels=channels, size=size, seed=seed)
    g = _holdout_stream(seed, 7919)
    y = _balanced_labels(num_classes, n, g)
    return _images(means, y, g, noise, dtype, channels_last, pin)


def _tokens(y, seq_len, vocab, num_classes, g, pin):
    n = y.numel()
    base = torch.randint(0, vocab, (n, seq_len), generator=g)
    band = max(1, vocab // (num_classes * 4))
    hot = torch.randint(0, band, (n, seq_len), generator=g) + (y.view(-1, 1) * band)
    use_hot = torch.rand(n, seq_len, generator=g) < 0.3
    X = torch.where(use_hot, hot, base)
    if pin and torch.cuda.is_available():
        X, y = X.pin_memory(), y.pin_memory()
    return X, y


def token_shard(spec: ShardSpec, *, seq_len: int = 128, vocab: int = 30522, seed: int = 0,
                pin: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """Class-conditional token sequences for the BERT config: each class
    over-samples a class-specific slice of the vocabulary."""
    g = _stream(seed, 104729, spec.client)
    y = _labels_for(spec, g)
    return _tokens(y, seq_len, vocab, spec.class_probs.numel(), g, pin)


def holdout_token_shard(num_classes: int, n: int, *, seq_len: int = 128, vocab: int = 30522, seed: int = 0,
                        pin: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """Held-out token sequences for evaluation: class-balanced labels, the vocabulary bands of :func:`token_shard`,
    from a random stream no training client draws from."""
    g = _holdout_stream(seed, 104729)
    y = _balanced_labels(num_classes, n, g)
    return _tokens(y, seq_len, vocab, num_classes, g, pin)
