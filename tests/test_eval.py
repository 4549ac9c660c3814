"""Evaluation of the global model on held-out data, CPU tier: the portable evaluator behind ``FederatedEngine.evaluate``,
the held-out generators, and the manager's ``GET /{name}/evaluate`` over fake GPU seats."""
import asyncio
import math
from types import SimpleNamespace

import torch
from torch import nn

from baton_b200.control.gpu_worker import EvaluatingSeat
from baton_b200.data import (ShardSpec, class_means, dirichlet_label_shards, holdout_image_shard, holdout_token_shard,
                             image_shard, token_shard)
from baton_b200.models import FederatedModule, LinearModel
from baton_b200.parallel.engine import FederatedEngine
from baton_b200.train import PortableLocalSGD
from conftest import run_async
from fedtest import Federation, ShardWorker
from test_seated_plane import FakeFabric, FakeSession


class TinyClassifier(FederatedModule):
    name = "tiny"
    loss_kind = "ce"

    def __init__(self):
        super().__init__()
        self.fc = nn.Linear(6, 4)
        self.bn = nn.BatchNorm1d(4)

    def forward(self, x):
        return self.bn(self.fc(x))


def test_portable_engine_evaluate_matches_hand_computation():
    torch.manual_seed(0)
    model = TinyClassifier()
    eng = FederatedEngine(model, "cpu", backend="nccl", lr=0.1, batch_size=8)
    X, y = torch.randn(40, 6), torch.randint(0, 4, (40,))
    eng.run_round((X, y), n_epoch=1)             # moves the weights and the BatchNorm running statistics
    Xe, ye = torch.randn(23, 6), torch.randint(0, 4, (23,))
    before = {k: v.clone() for k, v in model.state_dict().items()}
    model.train()
    res = eng.evaluate((Xe, ye), batch_size=5)   # ragged last batch
    assert model.training                        # the training flag is restored
    for k, v in model.state_dict().items():
        assert torch.equal(v, before[k]), k      # evaluation wrote no state (running statistics included)
    with torch.no_grad():
        model.eval()
        logits = model(Xe)
        model.train()
    want_loss = float(nn.functional.cross_entropy(logits, ye))
    want_acc = int((logits.argmax(-1) == ye).sum()) / 23
    assert res.n_samples == res.local_n_samples == 23
    assert math.isclose(res.loss, want_loss, rel_tol=1e-5) and math.isclose(res.local_loss, want_loss, rel_tol=1e-5)
    assert math.isclose(res.accuracy, want_acc, abs_tol=1e-9)
    empty = eng.evaluate(None)                   # a rank without held-out data contributes nothing
    assert empty.n_samples == 0 and math.isnan(empty.loss)


def test_portable_evaluate_regression_is_mean_squared_error():
    torch.manual_seed(1)
    model = LinearModel()
    tr = PortableLocalSGD(model, SimpleNamespace(device=torch.device("cpu")), loss="mse")
    X, y = torch.randn(17, 10), torch.randn(17, 1)
    loss_sum, correct, n = tr.evaluate(X, y, batch_size=4)
    with torch.no_grad():
        want = float(nn.functional.mse_loss(model(X), y))
    assert n == 17 and correct == 0 and math.isclose(loss_sum / n, want, rel_tol=1e-5)


def test_holdout_image_shard_is_balanced_shares_means_and_no_training_sample():
    seed, C = 3, 10
    X, y = holdout_image_shard(C, 1003, seed=seed, noise=0.5)
    assert X.shape == (1003, 32, 32, 3) and y.shape == (1003,)
    counts = torch.bincount(y, minlength=C)
    assert int(counts.max()) - int(counts.min()) <= 1
    means = class_means(C, seed=seed)
    # the same class structure as the training shards: the per-class sample mean sits on the training class mean
    for c in range(C):
        err = (X[y == c].mean(0) - means[c]).abs().mean()
        assert err < 0.05, (c, float(err))
    flat = X.reshape(X.shape[0], -1)
    for spec in dirichlet_label_shards(4, C, 300, alpha=0.5, seed=seed):
        Xt, _ = image_shard(spec, seed=seed, noise=0.5)
        d = torch.cdist(flat[:200], Xt.reshape(Xt.shape[0], -1))
        assert float(d.min()) > 1.0                # no held-out sample is a training sample
    X2, y2 = holdout_image_shard(C, 1003, seed=seed, noise=0.5)
    assert torch.equal(X, X2) and torch.equal(y, y2)      # deterministic in the seed


def test_holdout_stream_shares_no_draws_with_class_means_or_clients():
    from baton_b200.data import synthetic
    n = 40000
    for seed in (0, 1, 5):
        for mult in (7919, 104729):
            held = torch.randn(n, generator=synthetic._holdout_stream(seed, mult))
            others = [torch.randn(n, generator=torch.Generator().manual_seed(seed))]          # class means
            others += [torch.randn(n, generator=synthetic._stream(seed, mult, k)) for k in range(8)]
            pairs = set()
            for o in others:
                pairs.update(zip(o[:-1].tolist(), o[1:].tolist()))
            shared = sum(p in pairs for p in zip(held[:-1].tolist(), held[1:].tolist()))
            assert shared == 0, (seed, mult, shared)


def test_holdout_token_shard_is_balanced_and_uses_the_class_bands():
    C, vocab, n = 4, 1000, 400
    X, y = holdout_token_shard(C, n, seq_len=64, vocab=vocab, seed=2)
    counts = torch.bincount(y, minlength=C)
    assert int(counts.max()) - int(counts.min()) <= 1
    band = vocab // (C * 4)
    for c in range(C):
        in_band = ((X[y == c] >= c * band) & (X[y == c] < (c + 1) * band)).float().mean()
        assert in_band > 0.25                       # 30 % hot tokens plus the uniform share
    Xt, _ = token_shard(ShardSpec(0, torch.full((C,), 1.0 / C), n), seq_len=64, vocab=vocab, seed=2)
    assert not any(torch.equal(X[i], Xt[j]) for i in range(20) for j in range(n))


# ---------------------------------------------------------------- HTTP: GET /{name}/evaluate over fake seats
class FakeEvalSeat(EvaluatingSeat, ShardWorker):
    """A CPU stand-in for a GPU seat: the real route, the portable evaluator on the seat's replica."""

    def __init__(self, *a, eval_data=None, **kw):
        super().__init__(*a, **kw)
        self.eval_shard_fn = (lambda: eval_data) if eval_data is not None else None
        self.trainer = PortableLocalSGD(self.model, SimpleNamespace(device=torch.device("cpu")), loss="mse")


async def _seated_federation(eval_sizes):
    fed = Federation()
    exp = await fed.start_manager(dataplane="fused")
    fabric = FakeFabric()
    seats = []
    for r, k in enumerate(eval_sizes):
        m = LinearModel()
        m.load_state_dict(exp.model.state_dict())
        data = None if k is None else (torch.randn(k, 10, generator=torch.Generator().manual_seed(r)),
                                       torch.randn(k, 1, generator=torch.Generator().manual_seed(100 + r)))
        seats.append(await fed.add_worker(model=m, cls=FakeEvalSeat, n=5, seed=r, dataplane="fused",
                                          session=FakeSession(fabric, r, m), eval_data=data))
    return fed, exp, fabric, seats


def _hand_eval(seat, data):
    with torch.no_grad():
        return float(((seat.model(data[0]) - data[1]) ** 2).sum()), data[0].shape[0]


@run_async
async def test_manager_evaluate_returns_the_sample_weighted_aggregate_and_records_it():
    fed, exp, fabric, seats = await _seated_federation([7, 19, None])
    try:
        status, body = await fed.get("evaluate")
        assert status == 200 and body["n_samples"] == 0 and body["loss"] is None   # no seat holds the model yet
        orig = exp.plane.aggregate

        async def spy(experiment, responses):
            fabric.snapshot = {w.plane.rank: {k: v.clone() for k, v in w.model.state_dict().items()} for w in seats}
            return await orig(experiment, responses)
        exp.plane.aggregate = spy
        await fed.get("start_round?n_epoch=1")
        await fed.wait_round_closed()
        status, body = await fed.get("evaluate")
        assert status == 200
        parts = [_hand_eval(s, s.eval_shard_fn()) for s in seats[:2]]     # seat 2 has no held-out data: left out
        n = sum(k for _, k in parts)
        assert body["n_samples"] == n == 26 and body["n_seats"] == 2
        assert math.isclose(body["loss"], sum(l for l, _ in parts) / n, rel_tol=1e-5)
        assert body["accuracy"] == 0.0 and body["n_updates"] == 1
        status, metrics = await fed.get("metrics")
        assert status == 200 and [e["n_updates"] for e in metrics["evals"]] == [0, 1]
        assert math.isclose(metrics["evals"][-1]["loss"], body["loss"], rel_tol=1e-12)
        assert metrics["rounds"] == 1                                     # evaluations are not rounds
    finally:
        await fed.close()


@run_async
async def test_manager_evaluate_answers_423_during_a_round():
    fed, exp, fabric, seats = await _seated_federation([5])
    try:
        await exp.update_manager.start_update(n_epoch=1)
        status, _ = await fed.get("evaluate")
        assert status == 423
        exp.update_manager.end_update()
        status, _ = await fed.get("evaluate")
        assert status == 200
    finally:
        await fed.close()


@run_async
async def test_manager_evaluate_discards_a_fan_out_during_which_a_round_opened():
    fed, exp, fabric, seats = await _seated_federation([5, 9])
    try:
        for w in seats:
            exp.client_manager.clients[w.client_id]["model_synced"] = True
        orig = exp._evaluate_seat
        opened = []

        async def seat_then_round_opens(cid):
            out = await orig(cid)
            if not opened:
                opened.append(cid)
                await exp.update_manager.start_update(n_epoch=1)     # a round opens mid fan-out
            return out
        exp._evaluate_seat = seat_then_round_opens
        status, _ = await fed.get("evaluate")
        assert status == 423 and opened and exp.metrics.evals == []  # seats may have seen different models
        exp.update_manager.end_update()
        exp._evaluate_seat = orig
        status, body = await fed.get("evaluate")
        assert status == 200 and body["n_seats"] == 2 and len(exp.metrics.evals) == 1
    finally:
        await fed.close()


@run_async
async def test_manager_evaluate_answers_501_on_the_http_plane():
    fed = Federation()
    await fed.start_manager(dataplane="http")
    try:
        await fed.add_worker(n=5, seed=0)
        status, _ = await fed.get("evaluate")
        assert status == 501
    finally:
        await fed.close()


@run_async
async def test_seat_without_held_out_data_answers_501():
    fed, exp, fabric, seats = await _seated_federation([None])
    try:
        s = seats[0]
        async with fed.client.session.post("http://127.0.0.1:{}/lineartest/evaluate?client_id={}&key={}".format(
                s.port, s.client_id, s.key)) as resp:
            assert resp.status == 501
        async with fed.client.session.post("http://127.0.0.1:{}/lineartest/evaluate?client_id=x&key=y".format(
                s.port)) as resp:
            assert resp.status == 404
        await asyncio.sleep(0)
    finally:
        await fed.close()


def test_two_gloo_ranks_global_result_is_the_sample_weighted_mean_of_the_local_results():
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29900 + (os.getpid() % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "mp_eval_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=root, env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
