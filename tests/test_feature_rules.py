"""Which combinations of federation features every entry point accepts.

``tests/golden/feature_rules.json`` holds, for each entry point that runs on the CPU, the outcome of every combination
of the features that entry point takes: one character per combination, in ``itertools.product`` order of its axes
(``.`` accepted, ``V`` ValueError, ``T`` TypeError, ``R`` RuntimeError).  The table was recorded before the cross-feature
rules were gathered in ``parallel/features.py``.  Every combination keeps its outcome, except those
:func:`newly_rejected` names: some entry points accepted them while others rejected them, and now all reject them.

``python tests/test_feature_rules.py --record`` rewrites the table (only for a rule that changes on purpose)."""
from __future__ import annotations

import itertools
import json
import pathlib
import sys

import pytest
import torch

GOLDEN = pathlib.Path(__file__).parent / "golden" / "feature_rules.json"
CODES = {"ok": ".", "ValueError": "V", "TypeError": "T", "RuntimeError": "R"}

WIRE = ["fp32", "bf16", "fp8"]
MODE = ["delta", "weights"]
ON = [False, True]
AGG = ["mean", "median", "trimmed_mean", "krum"]
PLANE = ["http", "fused", "nccl"]
SESSION = {"wire": WIRE, "mode": MODE, "dp": ON, "scaffold": ON, "aggregator": AGG, "topk": ON, "server_opt": ON,
           "tile_flags": ON}
LOCAL = {"prox_mu": [0.0, 0.01], "optimizer": ["sgd", "adamw"], "momentum": [0.0, 0.9]}
AXES = {
    "engine": dict(SESSION, **LOCAL),
    "nccl_session": SESSION,
    "fused_session": SESSION,
    # a world-1 NcclSession built without dp / robust, then one round with dp= / robust=
    "nccl_aggregate": {"wire": WIRE, "mode": MODE, "scaffold": ON, "topk": ON, "server_opt": ON, "tile_flags": ON,
                       "dp": ON, "aggregator": AGG},
    "config": dict({"wire": WIRE, "dp": ON, "aggregator": AGG, "server_opt": ON, "plane": PLANE}, **LOCAL),
    "manager_plane": {"plane": PLANE, "dp": ON, "aggregator": AGG, "server_opt": ON},
}


def _dp(r):
    from baton_b200.parallel.dp import DPConfig
    return DPConfig(1.0, 0.5, seed=1) if r["dp"] else None


def _robust(r):
    from baton_b200.parallel.robust import RobustConfig
    return RobustConfig(r["aggregator"]) if r["aggregator"] != "mean" else None


def _session_kw(r) -> dict:
    from baton_b200.parallel.compress import TopKConfig
    from baton_b200.parallel.server_opt import ServerOptConfig
    return dict(wire_dtype=r["wire"], mode=r["mode"], scaffold=r["scaffold"], tile_flags=r["tile_flags"],
                topk=TopKConfig(0.1) if r["topk"] else None,
                server_opt=ServerOptConfig("adam", 0.1) if r["server_opt"] else None)


def _arena():
    from baton_b200.models import LinearModel
    from baton_b200.parallel.arena import ParamArena
    return ParamArena(LinearModel(), torch.device("cpu"))


def _engine(r):
    from baton_b200.models import LinearModel
    from baton_b200.parallel.engine import FederatedEngine
    FederatedEngine(LinearModel(), "cpu", backend="nccl", loss="mse", logical_clients=4, wire_dtype=r["wire"],
                    mode=r["mode"], dp_clip=1.0 if r["dp"] else 0.0, dp_noise_multiplier=0.5 if r["dp"] else 0.0,
                    dp_seed=1, scaffold=r["scaffold"], aggregator=r["aggregator"],
                    compress="topk" if r["topk"] else None, topk_ratio=0.1,
                    server_opt="adam" if r["server_opt"] else None, server_lr=0.1, tile_flags=r["tile_flags"],
                    prox_mu=r["prox_mu"], optimizer=r["optimizer"], momentum=r["momentum"])


def _nccl_session(r):
    from baton_b200.parallel.fedavg import NcclSession
    NcclSession(_arena(), dp=_dp(r), robust=_robust(r), **_session_kw(r))


def _fused_session(r):
    from baton_b200.parallel.fedavg import FedAvgSession
    FedAvgSession(_arena(), dp=_dp(r), robust=_robust(r), **_session_kw(r))


def _nccl_aggregate(r):
    from baton_b200.parallel.fedavg import NcclSession
    a = _arena()
    s = NcclSession(a, **_session_kw(r))
    kw = {}
    if r["scaffold"]:
        kw["control"] = (torch.zeros(a.n_param), torch.zeros(a.n_param), 1)
    if r["topk"]:
        s.pack_topk(torch.zeros(a.n))
    s.aggregate(my_n=1.0, dp=_dp(r), robust=_robust(r), **kw)


def _config(r):
    from baton_b200.config import FederationConfig
    FederationConfig(wire_dtype=r["wire"], backend=r["plane"], clients=2, logical_clients=4,
                     dp_clip=1.0 if r["dp"] else 0.0, dp_noise_multiplier=0.5 if r["dp"] else 0.0,
                     aggregator=r["aggregator"], server_opt="adam" if r["server_opt"] else "none", server_lr=0.1,
                     prox_mu=r["prox_mu"], optimizer=r["optimizer"], momentum=r["momentum"])


def _manager_plane(r):
    from baton_b200.parallel.dataplane import make_manager_plane
    from baton_b200.parallel.server_opt import ServerOptConfig
    make_manager_plane(r["plane"], dp=_dp(r), robust=_robust(r),
                       server_opt=ServerOptConfig("adam", 0.1) if r["server_opt"] else None)


BUILD = {"engine": _engine, "nccl_session": _nccl_session, "fused_session": _fused_session,
         "nccl_aggregate": _nccl_aggregate, "config": _config, "manager_plane": _manager_plane}


def rows(entry):
    names = list(AXES[entry])
    for values in itertools.product(*AXES[entry].values()):
        yield dict(zip(names, values))


def outcome(entry, r) -> str:
    try:
        BUILD[entry](r)
    except Exception as e:      # noqa: BLE001 -- the class of whatever the entry point raises is the outcome
        return CODES.get(type(e).__name__, "?")
    return CODES["ok"]


def newly_rejected(entry, r) -> bool:
    """The combinations that were accepted at ``entry`` although another entry point rejected them."""
    if entry in ("nccl_session", "fused_session", "nccl_aggregate") and r["scaffold"] and r["tile_flags"]:
        return True         # SCAFFOLD with tile_flags: FederatedEngine rejected it, neither session did
    if entry == "nccl_aggregate":
        robust = r["aggregator"] != "mean"
        # a round's dp= / robust= on NcclSession: FedAvgSession.aggregate rejected these, NcclSession ran them
        return (robust and (r["dp"] or r["scaffold"] or r["mode"] == "weights" or r["tile_flags"])) or (
            r["dp"] and r["scaffold"])
    return False


def _needs_ext(entry):
    if entry == "fused_session":
        from baton_b200.ops._ext import load
        try:
            load()
        except Exception as e:      # noqa: BLE001
            pytest.skip("baton_b200._C is not built: {}".format(e))


@pytest.mark.parametrize("entry", list(AXES))
def test_every_combination_keeps_its_outcome(entry):
    _needs_ext(entry)
    want = json.loads(GOLDEN.read_text())[entry]
    assert want["axes"] == AXES[entry]
    bad = []
    for r, was in zip(rows(entry), want["outcomes"]):
        got = outcome(entry, r)
        expect = CODES["ValueError"] if newly_rejected(entry, r) else was
        if got != expect:
            bad.append((r, was, got))
    assert not bad, "{} combinations changed outcome, e.g. {}".format(len(bad), bad[:5])


WRONG_TYPES = [("robust", True), ("robust", 1), ("robust", "median"), ("topk", True), ("topk", 0.1),
               ("server_opt", True), ("server_opt", "adam")]


@pytest.mark.parametrize("name,value", WRONG_TYPES)
def test_a_feature_of_the_wrong_type_is_a_type_error(name, value):
    """The sessions (at construction, and a round's ``robust=``) and the http manager plane (``server_opt=``) reject
    anything but the feature's configuration with TypeError, even where the combination would be accepted."""
    from baton_b200.parallel.dataplane import HttpManagerPlane, make_manager_plane
    from baton_b200.parallel.fedavg import NcclSession
    kw = {name: value}
    calls = [lambda: NcclSession(_arena(), **kw)]
    if name == "server_opt":
        calls += [lambda: HttpManagerPlane(**kw), lambda: make_manager_plane("http", **kw)]
    if name == "robust":
        calls.append(lambda: NcclSession(_arena()).aggregate(my_n=1.0, **kw))
    try:
        from baton_b200.ops._ext import load
        load()
    except Exception:       # noqa: BLE001 -- without the extension only the host entry points run
        pass
    else:
        from baton_b200.parallel.fedavg import FedAvgSession
        calls.append(lambda: FedAvgSession(_arena(), **kw))
        if name == "robust":
            calls.append(lambda: FedAvgSession(_arena()).aggregate(my_n=1.0, **kw))
    for call in calls:
        with pytest.raises(TypeError):
            call()


if __name__ == "__main__" and "--record" in sys.argv:
    sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
    table = {e: {"axes": AXES[e], "outcomes": "".join(outcome(e, r) for r in rows(e))} for e in AXES}
    assert not any("?" in t["outcomes"] for t in table.values()), "an entry point raised an unexpected exception"
    GOLDEN.write_text(json.dumps(table, indent=1) + "\n")
