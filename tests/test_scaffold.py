"""SCAFFOLD, CPU tier: the constructor's rejections, the SPMD engine with logical clients against a hand-written SCAFFOLD,
and the same across two gloo ranks."""
import os
import subprocess
import sys

import pytest
import torch

from baton_b200.models import MLP2
from baton_b200.parallel.engine import FederatedEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from mp_scaffold_gloo import LR, EPOCHS, check_against_hand_written, shard  # noqa: E402


@pytest.mark.parametrize("kw", [{"dp_clip": 1.0}, {"prox_mu": 0.01}, {"mode": "weights"}, {"tile_flags": True}],
                         ids=["dp", "fedprox", "weights", "tile_flags"])
def test_scaffold_rejects_unsupported_combinations(kw):
    with pytest.raises(ValueError):
        FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse", scaffold=True, **kw)


def test_control_variates_need_scaffold():
    eng = FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse")
    with pytest.raises(RuntimeError):
        eng.control_variates()


def test_scaffold_engine_logical_clients_matches_hand_written():
    """4 logical clients, 2 sampled per round, 3 rounds, full-batch local steps: global model, c and every c_i."""
    torch.manual_seed(0)
    model = MLP2(10, 16, 1)
    init = [p.detach().clone() for p in model.parameters()]
    eng = FederatedEngine(model, "cpu", backend="nccl", loss="mse", lr=LR, batch_size=64, wire_dtype="fp32",
                          scaffold=True, logical_clients=4, sample_k=2, seed=3)
    rounds = []
    for _ in range(3):
        rounds.append(eng.run_round(lambda cid: shard(cid, 16 + 8 * cid), n_epoch=EPOCHS).participants)
    errs = check_against_hand_written(eng, init, rounds, lambda cid: shard(cid, 16 + 8 * cid), n_clients=4,
                                      hosted=lambda cid: True)
    assert max(errs.values()) < 2e-5, errs
    c, ci = eng.control_variates()
    assert sorted(ci) == sorted({cid for r in rounds for cid in r})
    assert float(c.abs().max()) > 0.0


def test_scaffold_two_gloo_ranks():
    port = 29400 + ((os.getpid() + 317) % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mp_scaffold_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT, env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
