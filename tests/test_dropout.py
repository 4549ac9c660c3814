"""Dropout of BERT training, CPU tier: the host mask against the counter formula, its statistics and edges, the
configuration checks, the CPU model in train and eval mode, and the reproducibility of trainer and engine runs."""
import json

import numpy as np
import pytest
import torch

from baton_b200.config import FederationConfig
from baton_b200.data.augment import augment_key
from baton_b200.data.dropout import (DropoutRun, check_dropout, check_run, counter_word, dropout_keep,
                                     dropout_reference, scale, threshold)
from baton_b200.demo import build_model
from baton_b200.models.bert import BertConfig, BertForSequenceClassification
from baton_b200.parallel.dp import philox4x32_10
from baton_b200.parallel.engine import FederatedEngine
from baton_b200.train import PortableLocalSGD, run_local_sgd


def _tiny(p_hidden=0.1, p_attn=0.1, classifier=None):
    torch.manual_seed(0)
    return BertForSequenceClassification(BertConfig(
        vocab_size=1024, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=512,
        max_position_embeddings=128, hidden_dropout_prob=p_hidden, attention_probs_dropout_prob=p_attn,
        classifier_dropout=classifier), name="bert_tiny")


def _tokens(n=24, S=16, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 1024, (n, S), generator=g), torch.randint(0, 2, (n,), generator=g)


def test_mask_follows_the_counter_word_by_word():
    key, stream, site, t, p = 0x0123456789ABCDEF, (5 << 32) | 3, 7, 1234, 0.3
    n = 37
    keep = dropout_keep(key, stream, site, t, n, p)
    T = threshold(p)
    for i in range(n):
        ctr = np.array([[i >> 2, 0x80000000 | site << 22 | t, stream & 0xFFFFFFFF, stream >> 32]], dtype=np.uint32)
        x = philox4x32_10(ctr, (key & 0xFFFFFFFF, key >> 32))[0]
        assert keep[i] == (int(x[i & 3]) >= T), i


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_fraction_within_binomial_bounds(p):
    n = 200_000
    k = int(dropout_keep(augment_key(1), 9, 3, 5, n, p).sum())
    sd = (n * p * (1 - p)) ** 0.5
    assert abs(k - n * (1 - p)) < 5 * sd


def test_sites_steps_streams_and_keys_give_different_masks():
    base = dict(key=11, stream=2, site=3, t=4)
    ref = dropout_keep(n=4096, p=0.5, **base)
    for field, other in (("key", 12), ("stream", 3), ("site", 4), ("t", 5), ("stream", (2 << 32) | 2)):
        kw = dict(base, **{field: other})
        assert not np.array_equal(ref, dropout_keep(n=4096, p=0.5, **kw)), field
    assert np.array_equal(ref, dropout_keep(n=4096, p=0.5, **base))


def test_threshold_and_scale_at_the_edges():
    assert threshold(0.0) == 0 and dropout_keep(1, 2, 3, 4, 100, 0.0).all()
    assert threshold(0.5) == 1 << 31 and scale(0.5) == 2.0
    assert threshold(0.1) == 429496729 and scale(0.1) == float(np.float32(1 / 0.9))
    assert threshold(np.nextafter(1.0, 0.0)) == (1 << 32) - 1
    assert threshold(2.0 ** -32) == 1 and threshold(np.nextafter(2.0 ** -32, 0.0)) == 0


def test_reference_scales_kept_values_and_zeroes_the_rest():
    x = torch.arange(1, 65, dtype=torch.float32).view(8, 8)
    y = dropout_reference(x, 5, 6, 1, 2, 0.25)
    keep = torch.from_numpy(dropout_keep(5, 6, 1, 2, 64, 0.25)).view(8, 8)
    assert torch.equal(y[keep], x[keep] * np.float32(scale(0.25))) and bool((y[~keep] == 0).all())


@pytest.mark.parametrize("bad", [-0.1, 1.0, 1.5, float("nan"), "x", None, True])
def test_validation_errors(bad):
    with pytest.raises(ValueError):
        check_dropout(bad)
    with pytest.raises(ValueError):
        BertConfig(hidden_dropout_prob=bad)
    with pytest.raises(ValueError):
        BertConfig(attention_probs_dropout_prob=bad)
    if bad is not None:                                          # classifier_dropout=None follows the hidden one
        with pytest.raises(ValueError):
            BertConfig(classifier_dropout=bad)


def test_counter_limits():
    assert counter_word(511, (1 << 22) - 1) == 0xFFFFFFFF
    for site, t in ((512, 0), (0, 1 << 22), (-1, 0)):
        with pytest.raises(ValueError):
            counter_word(site, t)
    check_run(74, 1 << 22)                                       # BERT-large's sites, the last step
    with pytest.raises(ValueError):
        check_run(513, 1)
    with pytest.raises(ValueError):
        check_run(2, (1 << 22) + 1)
    m = _tiny()
    with pytest.raises(ValueError):
        run_local_sgd(m, *_tokens(8), n_epoch=(1 << 22) + 1, batch_size=8, loss="ce")


def test_config_defaults_and_classifier_follows_hidden():
    c = BertConfig()
    assert (c.hidden_dropout_prob, c.attention_probs_dropout_prob, c.classifier_dropout) == (0.0, 0.0, None)
    assert BertConfig(hidden_dropout_prob=0.2).classifier_p == 0.2
    assert BertConfig(hidden_dropout_prob=0.2, classifier_dropout=0.0).classifier_p == 0.0
    assert _tiny(0.0, 0.0).has_dropout is False and _tiny(0.0, 0.1).has_dropout and _tiny(0.0, 0.0, 0.3).has_dropout
    assert _tiny().n_dropout_sites == 8


def test_cpu_model_train_differs_from_eval_and_eval_ignores_p():
    ids, _ = _tokens(6)
    m, m0 = _tiny(), _tiny(0.0, 0.0)
    m0.load_state_dict(m.state_dict())
    run = m.dropout_run
    run.begin(augment_key(3), 7, 1, 1, m.n_dropout_sites)
    run.at(0, 0)
    m.train()
    with torch.no_grad():
        a = m(ids)
        b = m(ids)
        m.eval()
        e = m(ids)
        m0.eval()
        e0 = m0(ids)
        m0.train()
        t0 = m0(ids)
    run.end()
    assert torch.equal(a, b)                                     # the masks are a function of the run state
    assert not torch.allclose(a, e)
    assert torch.equal(e, e0) and torch.equal(t0, e0)
    m.train()
    with torch.no_grad():
        assert torch.equal(m(ids), e)                            # outside a run nothing is dropped


def test_cpu_sites_match_a_hand_written_forward():
    """Every site of the CPU model applies the reference mask of its site id to the tensor the contract names."""
    m = _tiny(0.2, 0.3, 0.4)
    ids, _ = _tokens(3, 8)
    key, stream, t = augment_key(9), 4, 2
    run = m.dropout_run
    run.begin(key, stream, 3, 1, m.n_dropout_sites)
    run.at(0, t)
    m.train()
    with torch.no_grad():
        got = m(ids)
    run.end()
    import math
    import torch.nn.functional as TF
    B, S = ids.shape
    c = m.config
    D, H = c.hidden_size, c.num_attention_heads
    dh = D // H

    def drop(x, site, p):
        return dropout_reference(x.contiguous(), key, stream, site, t, p)

    def ln(mod, x):
        return TF.layer_norm(x, (D,), mod.weight, mod.bias, c.layer_norm_eps)
    with torch.no_grad():
        e = m.embeddings
        x = ln(e.LayerNorm, e.word_embeddings.weight[ids.reshape(-1)] + e.position_embeddings.weight[
            torch.arange(S).repeat(B)] + e.token_type_embeddings.weight[torch.zeros(B * S, dtype=torch.long)])
        x = drop(x, 0, 0.2)
        for l, L in enumerate(m.layers):
            qkv = x @ L.qkv.weight.T + L.qkv.bias
            q, k, v = (u.reshape(B, S, H, dh).transpose(1, 2) for u in qkv.split(D, dim=-1))
            p = drop(torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh), dim=-1), 1 + 3 * l, 0.3)
            a = (p @ v).transpose(1, 2).reshape(B * S, D)
            x = ln(L.attn_ln, drop(a @ L.attn_out.weight.T + L.attn_out.bias, 2 + 3 * l, 0.2) + x)
            f = TF.gelu(x @ L.ffn_in.weight.T + L.ffn_in.bias, approximate="tanh")
            x = ln(L.ffn_ln, drop(f @ L.ffn_out.weight.T + L.ffn_out.bias, 3 + 3 * l, 0.2) + x)
        pooled = torch.tanh(x.view(B, S, D)[:, 0] @ m.pooler.weight.T + m.pooler.bias)
        want = drop(pooled, 7, 0.4) @ m.classifier.weight.T + m.classifier.bias
    assert torch.allclose(got, want, atol=1e-5, rtol=1e-5)


def test_run_local_sgd_is_reproducible_from_seed_and_stream():
    X, y = _tokens(20)
    outs = []
    for _ in range(2):
        m = _tiny()
        losses = run_local_sgd(m, X, y, n_epoch=2, lr=0.01, batch_size=8, loss="ce", augment_seed=4, augment_stream=9,
                               generator=torch.Generator().manual_seed(0))
        outs.append((losses, [p.detach().clone() for p in m.parameters()]))
    assert outs[0][0] == outs[1][0]
    assert all(torch.equal(a, b) for a, b in zip(outs[0][1], outs[1][1]))
    m = _tiny()
    other = run_local_sgd(m, X, y, n_epoch=2, lr=0.01, batch_size=8, loss="ce", augment_seed=4, augment_stream=10,
                          generator=torch.Generator().manual_seed(0))
    assert other != outs[0][0]
    assert not m.dropout_run.active


def test_config_round_trip_and_non_bert_models_rejected():
    cfg = FederationConfig(model="bert_base", dropout=0.1)
    assert FederationConfig.from_json(cfg.to_json()).dropout == 0.1
    assert json.loads(cfg.to_json())["dropout"] == 0.1
    for model in ("lineartest", "mlp2", "resnet18", "resnet50_gn"):
        with pytest.raises(ValueError):
            FederationConfig(model=model, dropout=0.1)
        with pytest.raises(ValueError):
            build_model(model, 0.1)
    for bad in (-0.5, 1.0):
        with pytest.raises(ValueError):
            FederationConfig(model="bert_base", dropout=bad)
    m = build_model("bert_base", 0.1)
    assert (m.config.hidden_dropout_prob, m.config.attention_probs_dropout_prob, m.config.classifier_p) == (0.1, 0.1, 0.1)
    assert build_model("bert_base").has_dropout is False


def _engine_round(seed):
    m = _tiny()
    eng = FederatedEngine(m, "cpu", backend="nccl", loss="ce", lr=0.01, batch_size=8, logical_clients=2, seed=seed)
    data = {c: _tokens(16, seed=c) for c in range(2)}
    for _ in range(2):
        eng.run_round(lambda cid: data[cid], n_epoch=1)
    return [p.detach().clone() for p in m.parameters()]


def test_portable_engine_round_is_reproducible_from_its_seed():
    a, b, c = _engine_round(5), _engine_round(5), _engine_round(6)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    assert not all(torch.equal(u, v) for u, v in zip(a, c))


def test_portable_trainer_draws_the_contract_masks():
    """PortableLocalSGD sets the run state per step: a one-step run equals the hand-set run state."""
    X, y = _tokens(8)
    m1, m2 = _tiny(), _tiny()
    from baton_b200.parallel.arena import ParamArena
    arena = ParamArena(m1, torch.device("cpu"))
    tr = PortableLocalSGD(m1, arena, loss="ce")
    seen = []
    orig = m1.dropout_run.at

    def spy(epoch, step, words=None):
        seen.append((m1.dropout_run.key, m1.dropout_run.stream, epoch, step))
        return orig(epoch, step, words)
    m1.dropout_run.at = spy
    tr.run(X, y, n_epoch=2, lr=0.01, batch_size=4, augment_seed=3, augment_stream=8)
    assert seen == [(augment_key(3), 8, e, s) for e in range(2) for s in range(2)]
    assert not m1.dropout_run.active
