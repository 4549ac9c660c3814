"""Gradient-norm clipping on the GPU: the norm kernel (fp64 accuracy, determinism, torch's coefficient, non-finite
gradients), the clipped forms of the arena optimizer kernels against their unclipped forms fed the clipped gradient,
the graphed trainers and the engine rounds."""
import pytest
import torch

from test_gpu_fedprox import _bits, _image_data, _rel, _resnet_trainer

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def F():
    from baton_b200.ops import functional
    return functional


def _norm(F, g, C):
    """(norm, coef, fp64 sum of squares) of the norm kernel on ``g`` with threshold ``C``."""
    work = torch.zeros(F.load().GRAD_NORM_WORK_WORDS, dtype=torch.int64, device=DEV)
    out = torch.zeros(2, dtype=torch.float32, device=DEV)
    F.grad_norm_clip(g, torch.tensor([C], dtype=torch.float32, device=DEV), work, out[0:1], out[1:2])
    return out[0:1].clone(), out[1:2].clone(), float(work[-1:].view(torch.float64))


@pytest.mark.parametrize("n", [11_177_538, 4096 * 3 + 2, 7])
def test_norm_kernel_is_fp64_accurate_deterministic_and_gives_torch_coefficient(F, n):
    gen = torch.Generator(device=DEV).manual_seed(n)
    g = torch.randn(n, device=DEV, generator=gen) * torch.rand(n, device=DEV, generator=gen) ** 4 * 1e-2
    want = torch.linalg.vector_norm(g.double())
    C = float(want) * 0.3
    norm, coef, sq = _norm(F, g, C)
    assert abs(sq ** 0.5 - float(want)) <= 1e-12 * float(want), (sq ** 0.5, float(want))
    assert torch.equal(norm, want.float().reshape(1))
    for _ in range(3):
        n2, c2, _ = _norm(F, g, C)
        assert torch.equal(_bits(n2), _bits(norm)) and torch.equal(_bits(c2), _bits(coef))
    for c in (C, float(want) * 5.0, 1e-3):
        _, coef, _ = _norm(F, g, c)
        ref = torch.clamp((norm + 1e-6).reciprocal() * torch.tensor(c, dtype=torch.float32), max=1.0)
        assert torch.equal(_bits(coef), _bits(ref)), (c, float(coef), float(ref))


@pytest.mark.parametrize("bad", [float("inf"), float("nan")])
def test_non_finite_gradients_follow_torch(F, bad):
    g = torch.randn(4096, device=DEV)
    g[17] = bad
    norm, coef, _ = _norm(F, g, 1.0)
    p = torch.zeros(4096, device=DEV, requires_grad=True)
    p.grad = g.clone()
    torch.nn.utils.clip_grad_norm_([p], 1.0)                   # torch on the same device
    ref = p.grad
    want_coef = torch.clamp((norm + 1e-6).reciprocal() * 1.0, max=1.0)
    assert torch.equal(coef.isnan(), want_coef.isnan()) and (coef.isnan().all() or torch.equal(coef, want_coef))
    w = torch.zeros(4096, device=DEV)
    hyper = torch.tensor([1.0, 0.0, 0.0, 0.0, 0.0, 0.0], device=DEV)
    F.grad_norm_clip(g, torch.tensor([1.0], device=DEV), torch.zeros(F.load().GRAD_NORM_WORK_WORDS,
                     dtype=torch.int64, device=DEV), norm, hyper[5:6])
    F.fused_sgd(w, g.clone(), hyper, zero_grad=True, clip=True)
    # w = -1 * g' : the same NaN / zero pattern as torch's clipped gradient
    assert torch.equal(w.isnan(), ref.isnan()) and torch.equal(-w[~w.isnan()], ref[~ref.isnan()])


def _state(n, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    r = lambda s=1.0: torch.randn(n, device=DEV, generator=gen) * s      # noqa: E731
    return r(), r(0.1), r(0.01), r(0.5), r(0.01), r(0.01).abs()          # w, g, m, anchor, corr, v


FORMS = ["plain", "momentum", "nesterov", "prox", "scaf", "adam"]


def _sgd_args(F, form, st, coef, wd=1e-3):
    """(hyper, kwargs of fused_sgd / fused_sgd_segments) of one optimizer form, clip coefficient `coef` in place."""
    w, g, m, a, c, v = st
    if form == "adam":
        row = F.adamw_rows(0.01, (0.9, 0.99), 1e-8, wd, 3, 1)[0].to(DEV)
        row[F.ADAMW_ROW_CLIP] = coef
        return row, dict(momentum_buf=m, adam_v=v)
    hyper = torch.tensor([0.05, 0.9, wd, 0.0, 0.1 if form == "prox" else 0.0, coef], device=DEV)
    kw = dict(momentum_buf=m if form in ("momentum", "nesterov", "prox", "scaf") else None,
              nesterov=form == "nesterov")
    if form == "prox":
        kw["prox_anchor"] = a
    if form == "scaf":
        kw["corr"] = c
    return hyper, kw


def _clone(st):
    return tuple(t.clone() for t in st)


@pytest.mark.parametrize("form", FORMS)
def test_clipped_arena_pass_is_unclipped_pass_on_the_clipped_gradient(F, form):
    """Whole-arena form: clipped(g) == unclipped(fl32(g * coef)) bit for bit, with the device-written coefficient."""
    n = 1 << 20
    base = _state(n, 1)
    _, coef, _ = _norm(F, base[1], float(torch.linalg.vector_norm(base[1])) * 0.25)
    assert 0.2 < float(coef) < 0.3

    def run(clip):
        st = _clone(base)
        if not clip:
            st = (st[0], torch.mul(st[1], coef), *st[2:])
        hyper, kw = _sgd_args(F, form, st, float(coef))
        wb = torch.zeros(n, dtype=BF16, device=DEV)
        F.fused_sgd(st[0], st[1], hyper, w_bf16=wb, clip=clip, **kw)
        torch.cuda.synchronize()
        return st, wb

    (sa, wa), (sb, wb) = run(True), run(False)
    assert torch.equal(_bits(wa), _bits(wb))
    for i in (0, 1, 2, 5):
        assert torch.equal(_bits(sa[i]), _bits(sb[i])), i
    assert (sa[1] == 0).all()                # the gradient is zeroed


@pytest.mark.parametrize("form", FORMS)
def test_clipped_segment_pass_is_unclipped_pass_on_the_clipped_gradient(F, form):
    n = 4 * 8192 + 1000
    base = _state(n, 2)
    segs = torch.tensor(F.sgd_segments(n, [], [(8192, 8192), (3 * 8192 + 3, 500)]), dtype=torch.int64).to(DEV)
    assert segs[:, 2].sum() >= 2
    coef = torch.tensor([0.37], device=DEV)

    def run(clip):
        st = _clone(base)
        if not clip:
            st = (st[0], torch.mul(st[1], coef), *st[2:])
        hyper, kw = _sgd_args(F, form, st, float(coef), wd=0.0 if form == "plain" else 1e-3)
        wb = torch.zeros(n, dtype=BF16, device=DEV)
        F.fused_sgd_segments(st[0], st[1], hyper, segs, w_bf16=wb, clip=clip, **kw)
        torch.cuda.synchronize()
        return st, wb

    (sa, wa), (sb, wb) = run(True), run(False)
    assert torch.equal(_bits(wa), _bits(wb))
    for i in (0, 2, 5):
        assert torch.equal(_bits(sa[i]), _bits(sb[i])), i


def test_clipped_emitted_upload_equals_collective_pack(F):
    """The clipped arena pass emitting the upload copy gives the round of the unclipped pass fed fl32(g * coef) with
    the collective's own pack, bit for bit, over several rounds."""
    from baton_b200.models import resnet18
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.fedavg import FedAvgSession

    def run(clip, prepack):
        torch.manual_seed(0)
        arena = ParamArena(resnet18(10), DEV, momentum=True)
        sess = FedAvgSession(arena, wire_dtype="bf16", mode="delta", n_ctas=32)
        gen = torch.Generator(device=DEV).manual_seed(7)
        hyper = torch.tensor([0.1, 0.9, 0.0, 0.0, 0.0, 0.0], device=DEV)
        work = torch.zeros(F.load().GRAD_NORM_WORK_WORDS, dtype=torch.int64, device=DEV)
        norm = torch.zeros(1, device=DEV)
        for rnd in range(3):
            arena.grad.copy_(torch.randn(arena.n_param, device=DEV, generator=gen) * 0.01)
            arena.theta[arena.n_param:].add_(0.001 * (rnd + 1))
            F.grad_norm_clip(arena.grad[: arena.n_param], torch.tensor([1.0], device=DEV), work, norm, hyper[5:6])
            if not clip:
                arena.grad.mul_(hyper[5])
            if prepack:
                sess.arm_prepack(64.0)
            F.fused_sgd(arena.theta[: arena.n_param], arena.grad, hyper, arena.momentum,
                        arena.theta_bf16[: arena.n_param], pack=sess.pack_spec() if prepack else None, clip=clip)
            sess.aggregate(my_n=64.0, prepacked=prepack)
            assert sess.last_prepacked == prepack
        torch.cuda.synchronize()
        sess.check()
        assert float(hyper[5]) < 0.5
        return arena.theta.clone(), arena.global_w.clone(), arena.theta_bf16.clone(), arena.momentum.clone()

    want = run(False, False)
    for got in (run(False, True), run(True, True)):
        for a, b in zip(got, want):
            assert torch.equal(_bits(a), _bits(b)), int((_bits(a) != _bits(b)).nonzero()[0])


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_mlp_captured_clipped_run_follows_portable_torch_reference(optimizer):
    from baton_b200.models import MLP2
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.train import GraphedLocalSGD, PortableLocalSGD
    X = torch.randn(256, 16, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    y = X @ torch.arange(1.0, 17.0, device=DEV).unsqueeze(1)
    kw = dict(n_epoch=4, lr=0.01 if optimizer == "sgd" else 1e-3, batch_size=256, optimizer=optimizer,
              weight_decay=1e-3)

    def run(trainer, C):
        torch.manual_seed(0)
        m = MLP2(16, 64, 1)
        arena = ParamArena(m, DEV)
        tr = trainer(m, arena, loss="mse")
        p0 = arena.theta[: arena.n_param].clone()
        tr.run(X, y, max_grad_norm=C, **kw)                  # one full batch per epoch: the shuffle does not matter
        torch.cuda.synchronize()
        return arena.theta[: arena.n_param] - p0, tr.last_grad_norms()

    (got, gn), (want, wn), (plain, _) = run(GraphedLocalSGD, 5.0), run(PortableLocalSGD, 5.0), run(GraphedLocalSGD, 0.0)
    print("mlp {}: norms {} / {}; update rel diff {:.2e}, clipped/unclipped {:.2e}".format(
        optimizer, gn, wn, _rel(got, want), _rel(plain, want)))
    assert all(w > 5.0 for r in wn for w in r), wn               # every step clips
    assert gn[0][0] == pytest.approx(wn[0][0], rel=1e-3)          # the same first gradient
    # AdamW is nearly invariant to a gradient scale, so clipping moves its update less than SGD's
    assert _rel(got, want) < 1e-5 and _rel(plain, want) > 100 * _rel(got, want), (_rel(got, want), _rel(plain, want))


def test_resnet18_captured_clipped_run_matches_eager_differs_from_unclipped_and_reuses_its_graph():
    X, y = _image_data(DEV, 600)             # 4 full batches of 128 + a ragged one of 88
    kw = dict(n_epoch=2, lr=0.05, batch_size=128, momentum=0.9)
    C = 0.5

    def run(use_graph, C, trainer=None):
        m, arena, tr = trainer or _resnet_trainer(DEV, use_graph)
        n = arena.n_param
        g0 = arena.theta[:n].clone()
        torch.manual_seed(9)
        m.train(X, y, max_grad_norm=C, **kw)
        torch.cuda.synchronize()
        assert torch.equal(arena.theta_bf16[:n], arena.theta[:n].to(BF16))
        return arena.theta[:n] - g0, tr

    (a, tra), (b, _), (c, trc) = run(True, C), run(True, C), run(False, C)
    norms = tra.last_grad_norms()
    flat = [v for r in norms for v in r]
    assert len(norms) == 2 and all(len(r) == 5 for r in norms)
    assert all(v == v and 0 < v < float("inf") for v in flat)
    assert sum(v > C for v in flat) > len(flat) // 2, flat            # most steps clip
    noise, diff = _rel(b, a), _rel(c, a)
    (p1, _), (p2, _) = run(True, 0.0), run(True, 0.0)
    big, _ = run(True, 1e30)
    plain_noise, off, big_diff = _rel(p2, p1), _rel(a, p1), _rel(big, p1)
    print("clipped update rel diff: graphed/graphed {:.2e}, graphed/eager {:.2e}; unclipped graphed/graphed {:.2e}; "
          "clipped/unclipped {:.2e}; C=1e30/unclipped {:.2e}; norms {:.3g}..{:.3g}".format(
              noise, diff, plain_noise, off, big_diff, min(flat), max(flat)))
    assert diff <= 3.0 * noise + 2e-3, (diff, noise)
    assert off > 10.0 * max(noise, plain_noise) and off > 0.05, (off, noise)
    assert big_diff <= 3.0 * plain_noise + 2e-3, (big_diff, plain_noise)
    # a new threshold replays the same graph; only switching clipping on or off captures another
    n0 = len(tra._graphs)
    run(True, 0.25, (tra.model, tra.arena, tra))
    assert len(tra._graphs) == n0
    run(True, 0.0, (tra.model, tra.arena, tra))
    assert len(tra._graphs) == n0 + 1
    assert tra.last_grad_norms() is None


@pytest.mark.parametrize("form", ["tile_flags", "logical"])
def test_engine_rounds_with_clipping_report_norms(form):
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    X, y = _image_data(DEV, 512)
    torch.manual_seed(0)
    kw = dict(tile_flags=True) if form == "tile_flags" else dict(logical_clients=3)
    eng = FederatedEngine(resnet18(10), DEV, backend="fused", lr=0.05, batch_size=128, n_ctas=64, max_grad_norm=1.0,
                          **kw)
    hist = []
    for _ in range(3):
        hist += eng.run_round((lambda cid: (X, y)) if form == "logical" else (X, y), n_epoch=1).loss_history
    eng.sync()
    torch.cuda.synchronize()
    eng.session.check()
    norms = eng.last_grad_norms()
    assert sorted(norms) == ([0, 1, 2] if form == "logical" else [0]), norms
    for rows in norms.values():
        assert len(rows) == 1 and len(rows[0]) == 4
        assert all(v == v and 0 < v < float("inf") for v in rows[0]), rows
    assert all(h == h for h in hist) and hist[-1] < hist[0], hist
