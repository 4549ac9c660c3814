"""Epoch-graph capture and the cyclic garbage collector.  A model and its graphed trainer reference each other, so the
CUDA graphs of a dropped engine are destroyed by the collector, which runs at arbitrary allocations.  Destroying a
graph while a stream is capturing is not permitted and invalidates the capture in progress, so the trainer keeps the
collector switched off while it captures (training and evaluation graphs) and restores it afterwards."""
import gc

import pytest
import torch

DEV = "cuda:0"


@pytest.mark.gpu
def test_collector_is_off_while_graphs_are_captured():
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    eng = FederatedEngine(MLP2(16, 64, 1), DEV, backend="fused", loss="mse", lr=0.002, batch_size=64,
                          aggregator="median")
    seen = []
    step, eval_pass = eng.trainer._step, eng.trainer._eval_pass

    def spy(fn):
        def wrapped(*a, **kw):
            seen.append((torch.cuda.is_current_stream_capturing(), gc.isenabled()))
            return fn(*a, **kw)
        return wrapped
    eng.trainer._step, eng.trainer._eval_pass = spy(step), spy(eval_pass)
    gen = torch.Generator().manual_seed(1)
    X = torch.randn(256, 16, generator=gen)
    X, y = X.to(DEV), (X @ torch.arange(1.0, 17.0)).unsqueeze(1).to(DEV)
    assert gc.isenabled()
    for _ in range(2):
        eng.run_round((X, y), n_epoch=1)
    eng.evaluate((X, y), batch_size=128)
    eng.sync()
    torch.cuda.synchronize()
    eng.session.check()
    captured = [enabled for capturing, enabled in seen if capturing]
    assert captured and not any(captured)           # the epoch and the evaluation pass were captured, collector off
    assert any(enabled for capturing, enabled in seen if not capturing)    # warm-up steps ran with it on
    assert gc.isenabled()                           # and it is back on
