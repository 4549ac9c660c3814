"""Which federation features combine, in one place.

Every entry point that builds or runs a round passes the features it has to :func:`check_features` and leaves the
others at their defaults: :class:`~baton_b200.parallel.engine.FederatedEngine`, both sessions (at construction, and per
round with the round's effective ``dp`` / ``robust``), :class:`~baton_b200.config.FederationConfig`, the manager planes
and the local trainers.  The rules are checked in one fixed order, so a configuration that breaks two of them gets the
same reason from every entry point.  A new feature adds its rules here.  Checks of one feature's own values stay with
the feature (``check_dp``, ``check_robust``, ``TopKConfig``, ``ServerOptConfig``, ...).
"""
from __future__ import annotations

from typing import Optional, Tuple

OPTIMIZERS = ("sgd", "adamw")

SEATED_SERVER_OPT = ("a server optimizer needs the http plane: on the seated planes its state would be replicated on "
                     "the seats, an evicted seat would return with stale m and v, and the manager holds no copy to "
                     "resend")


def check_features(*, wire_dtype: str = "bf16", mode: str = "delta", dp=None, scaffold: bool = False, robust=None,
                   topk=None, server_opt=None, tile_flags: bool = False, plane: Optional[str] = None,
                   optimizer: str = "sgd", momentum: float = 0.0, nesterov: bool = False, prox_mu: float = 0.0,
                   local: bool = False, secure_agg: bool = False, frozen: bool = False, vit: bool = False) -> None:
    """``ValueError`` with the reason if the features cannot run together.  ``dp``, ``robust``, ``topk`` and
    ``server_opt`` are on unless they are None or False: the rules read only which features are on, so a caller may pass
    the features' configurations or bools.  Whoever takes a configuration from outside checks its type.  ``plane``:
    ``"http"`` or ``"seated"`` (the ``fused`` / ``nccl`` manager planes), None where no manager plane is involved.
    ``local``: client-local ``state_dict`` entries (FedBN / FedPer, ``parallel/personal.py``).  ``secure_agg``: secure
    aggregation (``parallel/secagg.py``).  ``frozen``: a model with frozen parameters (LoRA fine-tuning), whose
    arena range the collective skips.  ``vit``: a Vision Transformer (``models/vit.py``)."""
    if optimizer not in OPTIMIZERS:
        raise ValueError("optimizer must be one of {}, got {!r}".format(OPTIMIZERS, optimizer))
    adamw = optimizer == "adamw"
    dp, robust, topk, server_opt = (x is not None and x is not False for x in (dp, robust, topk, server_opt))
    rules = (
        (adamw and (momentum or nesterov), "momentum / nesterov are SGD options; AdamW keeps its own moments (betas)"),
        (adamw and prox_mu > 0, "AdamW with FedProx (prox_mu > 0) is not supported"),
        (adamw and scaffold, "AdamW with SCAFFOLD is not supported: option II's dc = (x - theta) / (K lr) - c assumes "
                             "SGD steps"),
        (scaffold and prox_mu > 0, "SCAFFOLD's correction and FedProx's proximal term are exclusive"),
        (topk and wire_dtype == "fp8", "top-k uploads with the fp8 wire are not supported: its block scales have no "
                                       "meaning on a sparse list"),
        (topk and dp, "top-k uploads with DP-FedAvg are not supported: the noise is calibrated to the dense clipped "
                      "mean"),
        (topk and robust, "top-k uploads with a robust aggregator are not supported: it needs every client's dense "
                          "update"),
        (topk and scaffold, "top-k uploads with SCAFFOLD are not supported: its control-variate segment is dense"),
        (topk and tile_flags, "top-k uploads with tile_flags are not supported"),
        (server_opt and plane == "seated", SEATED_SERVER_OPT),
        (scaffold and dp, "SCAFFOLD with DP-FedAvg is not supported: DP would also have to clip and noise dc"),
        (scaffold and tile_flags, "SCAFFOLD with tile_flags is not supported: the correction c - c_i reads c, which "
                                  "the previous round's collective writes, so it cannot run ahead of the join"),
        (robust and dp, "a robust aggregator with DP-FedAvg is not supported: DP's noise is calibrated to the clipped "
                        "mean"),
        (robust and scaffold, "a robust aggregator with SCAFFOLD is not supported: its control-variate update is a "
                              "mean"),
        (robust and tile_flags, "a robust aggregator with tile_flags is not supported"),
        (local and dp, "client-local entries with DP-FedAvg are not supported: the clip norm and the noise would have "
                       "to cover the shared entries only"),
        (local and scaffold, "client-local entries with SCAFFOLD are not supported: c and dc span the whole parameter "
                             "range"),
        (local and robust, "client-local entries with a robust aggregator or Krum are not supported: the client "
                           "segments span the whole arena"),
        (local and topk, "client-local entries with top-k uploads are not supported: the selection spans the whole "
                         "arena"),
        (local and tile_flags, "client-local entries with tile_flags are not supported: the flags index physical "
                               "granules, and the first layer may be local"),
        (local and plane is not None, "client-local entries need the SPMD engine: a manager plane's payload is a whole "
                                      "state_dict, and its seats would need per-client stores"),
        (secure_agg and wire_dtype != "fp32", "secure aggregation needs wire_dtype='fp32': its ring elements are 4 "
                                              "bytes, and the symmetric buffer is sized from the wire dtype"),
        (secure_agg and dp, "secure aggregation with DP-FedAvg is not supported: the reader-side clip factors and the "
                            "owner's noise sit outside the ring"),
        (secure_agg and robust, "secure aggregation with a robust aggregator or Krum is not supported: they need every "
                                "client's individual update"),
        (secure_agg and topk, "secure aggregation with top-k uploads is not supported: the sparse supports reveal "
                              "positions"),
        (secure_agg and scaffold, "secure aggregation with SCAFFOLD is not supported: its control-variate segment would "
                                  "need its own masks"),
        (secure_agg and local, "secure aggregation with client-local entries is not supported"),
        (secure_agg and tile_flags, "secure aggregation with tile_flags is not supported: the ring sum is decoded in "
                                    "the apply phase, not published tile by tile"),
        (secure_agg and plane is not None, "secure aggregation needs the SPMD engine: the manager planes have no key "
                                           "exchange, and their payload is a pickled state_dict"),
        (frozen and dp, "frozen parameters with DP-FedAvg are not supported: its round has no skipped range, so the "
                        "clip norm and the noise would cover the frozen weights"),
        (frozen and scaffold, "frozen parameters with SCAFFOLD are not supported: its round has no skipped range"),
        (frozen and robust, "frozen parameters with a robust aggregator or Krum are not supported: the client segments "
                            "span the whole arena"),
        (frozen and topk, "frozen parameters with top-k uploads are not supported: the selection spans the whole arena"),
        (frozen and secure_agg, "frozen parameters with secure aggregation are not supported: its ring has no skipped "
                                "range"),
        (frozen and tile_flags, "frozen parameters with tile_flags are not supported: the flags index physical "
                                "granules, and the skipped range has none"),
        (frozen and local, "frozen parameters with client-local entries are not supported: the collective skips one "
                           "range"),
        (frozen and plane is not None, "frozen parameters need the SPMD engine: a manager plane's payload is a whole "
                                       "state_dict"),
        (vit and tile_flags, "a Vision Transformer with tile_flags is not supported: its token kernel reads class_token "
                             "and pos_embedding, which the first GEMM's arrival flags do not cover"),
    )
    for broken, reason in rules:
        if broken:
            raise ValueError(reason)
    if mode != "delta":
        for on, name in ((topk, "top-k uploads"), (server_opt, "a server optimizer"), (dp, "DP-FedAvg"),
                         (scaffold, "SCAFFOLD"), (robust, "a robust aggregator"), (secure_agg, "secure aggregation")):
            if on:
                raise ValueError("{} needs mode='delta': it works on the update theta - global, which "
                                 "mode='weights' does not upload".format(name))


def peer_loads_only(*, wire_dtype: str, dp=None, scaffold: bool = False, robust=None, topk=None,
                    secure_agg: bool = False) -> bool:
    """True when a round cannot use NVLS: the switch adds raw wire values, so block-scaled fp8, DP's per-rank clip
    factors, SCAFFOLD's reader-side 1 / N, a selection (robust) and sparse lists (top-k) all need peer loads.  A secure
    round's ring sum would need ``multimem.ld_reduce.add.u32``, which sm_90a has in scalar form only (four times the
    switch operations of the float path, not measured)."""
    return wire_dtype == "fp8" or any(x is not None and x is not False for x in (dp, scaffold, robust, topk, secure_agg))


def round_plan(world: int, logical_clients: int = 0, sample_k: Optional[int] = None) -> Tuple[int, int]:
    """``(planned, max_clients)``: the participants a round plans for (what Krum's ``2f + 3`` and the robust
    aggregators' limit are checked against) and the client segments one rank may upload per round."""
    population = logical_clients if logical_clients and logical_clients > world else world
    planned = min(sample_k, population) if sample_k else population
    per_rank = -(-population // world) if population > world > 0 else 1
    return planned, min(per_rank, planned)
