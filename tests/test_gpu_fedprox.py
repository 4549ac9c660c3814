"""FedProx on the GPU: the proximal form of the SGD kernels (arena pass, optimizer epilogue of the weight-gradient GEMMs,
leftover segment pass), the graphed trainer and the engine rounds."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
HYPER = [(0.0, False, 0.0), (0.0, False, 5e-4), (0.9, False, 0.0), (0.9, False, 5e-4), (0.9, True, 0.0),
         (0.9, True, 5e-4)]
SHAPES = {
    "igemm_layer3": ((128, 4, 4, 128), 3, 2, 1, 256),
    "shortcut_layer4": ((128, 2, 2, 256), 1, 2, 0, 512),
    "centre_layer4": ((128, 1, 1, 512), 3, 1, 1, 512),
}
LR = 0.05


@pytest.fixture(scope="module")
def F():
    from baton_b200.ops import functional
    return functional


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32)


def _formula64(w, g, a, m, lr, mom, wd, prox, nesterov):
    """fp64 FedProx + SGD (torch.optim.SGD with dampening 0); returns (w, m)."""
    w, g, a = w.double(), g.double(), a.double()
    gp = g + wd * w + prox * (w - a)
    if m is None:
        return w - lr * gp, None
    m = mom * m.double() + gp
    step = gp + mom * m if nesterov else m
    return w - lr * step, m


@pytest.mark.parametrize("prox", [1e-3, 0.1])
@pytest.mark.parametrize("mu,nesterov,wd", HYPER)
def test_fused_sgd_with_anchor_matches_fp64_formula(F, mu, nesterov, wd, prox):
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(1)
    n = 8192 + 24
    w0 = torch.randn(n, device=dev, generator=gen)
    anchor = w0 + 0.5 * torch.randn(n, device=dev, generator=gen)
    g0 = torch.randn(n, device=dev, generator=gen)
    m0 = torch.randn(n, device=dev, generator=gen) * 0.1 if mu else None
    hyper = torch.tensor([LR, mu, wd, 0.0, prox], device=dev)
    want_w, want_m = _formula64(w0, g0, anchor, m0, LR, mu, wd, prox, nesterov)
    for wire_fp32 in (None, False, True):
        w, g, wb = w0.clone(), g0.clone(), w0.to(BF16)
        m = m0.clone() if m0 is not None else None
        pack, wire = None, None
        if wire_fp32 is not None:
            wire = torch.zeros(n, dtype=torch.float32 if wire_fp32 else BF16, device=dev)
            slot = torch.tensor([wire.data_ptr()], dtype=torch.int64, device=dev)
            pack = {"wire_slot": slot, "global_w": anchor, "scale": torch.tensor([3.0], device=dev), "n_pack": n,
                    "wire_fp32": wire_fp32}
        F.fused_sgd(w, g, hyper, m, wb, zero_grad=True, nesterov=nesterov, pack=pack, prox_anchor=anchor)
        torch.cuda.synchronize()
        assert torch.allclose(w.double(), want_w, rtol=1e-6, atol=1e-6), float((w.double() - want_w).abs().max())
        if m is not None:
            assert torch.allclose(m.double(), want_m, rtol=1e-6, atol=1e-6)
        assert (g == 0).all()
        assert torch.equal(wb, w.to(BF16))
        if wire is not None:
            d = (w - anchor) * 3.0
            assert torch.equal(_bits(wire), _bits(d if wire_fp32 else d.to(BF16)))


@pytest.mark.parametrize("mu,nesterov,wd", HYPER)
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_epilogue_with_anchor_matches_accumulate_then_fused_sgd(F, shape, mu, nesterov, wd):
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    xs, k, stride, pad, cout = SHAPES[shape]
    n_img, h, _, c = xs
    ho = F.conv_out_size(h, k, stride, pad)
    x = torch.randn(xs, device=dev).to(BF16)
    dy = torch.randn(n_img * ho * ho, cout, device=dev).to(BF16)
    centre = shape.startswith("centre")
    numel = cout * k * k * c
    off = 1024
    n = off + numel + 1032
    theta0 = torch.randn(n, device=dev) * 0.05
    anchor = theta0 + torch.randn(n, device=dev) * 0.02          # theta != anchor everywhere
    mom0 = torch.randn(n, device=dev) * 0.01 if mu else None
    hyper = torch.tensor([0.05, mu, wd, 0.0, 0.1], device=dev)

    def state():
        grad = torch.zeros(n, device=dev)
        grad[:off] = torch.linspace(-1.0, 1.0, off, device=dev)
        grad[off + numel:] = torch.linspace(-0.5, 0.5, n - off - numel, device=dev)
        theta = theta0.clone()
        return theta, grad, theta.to(BF16), mom0.clone() if mom0 is not None else None

    def out_view(grad):
        w2d = grad[off: off + numel].view(cout, k * k * c)
        return w2d.view(cout, k * k, c)[:, (k * k) // 2, :] if centre else w2d

    def wgrad(out2d, sgd=None):
        if centre:
            return F.gemm(dy, x.view(n_img, c), a_mn=True, b_mn=True, out=out2d, accumulate=True, sgd=sgd) is not None
        return F.conv_igemm_wgrad_(dy, x, out2d, k, k, stride, pad, sgd=sgd)

    theta_r, grad_r, wb_r, mom_r = state()
    assert wgrad(out_view(grad_r))
    F.fused_sgd(theta_r, grad_r, hyper, mom_r, wb_r, zero_grad=True, nesterov=nesterov, prox_anchor=anchor)

    theta, grad, wb, mom = state()
    out2d = out_view(grad)
    assert wgrad(out2d, F.sgd_epilogue_args(theta, grad, out2d, hyper, mom, wb, nesterov, anchor)), "epilogue declined"
    assert (grad[off: off + numel] == 0).all()
    fused = [(off + (4 * c if centre else 0), out2d.shape[0], out2d.shape[1], out2d.stride(0))]
    segs = F.sgd_segments(n, fused, [(off, numel)] if centre else [])
    F.fused_sgd_segments(theta, grad, hyper, torch.tensor(segs, dtype=torch.int64, device=dev), mom, wb,
                         nesterov=nesterov, prox_anchor=anchor)
    torch.cuda.synchronize()
    assert torch.equal(_bits(theta), _bits(theta_r))
    assert torch.equal(_bits(wb), _bits(wb_r))
    if mom is not None:
        assert torch.equal(_bits(mom), _bits(mom_r))
    assert (grad == 0).all() and (grad_r == 0).all()


def test_nograd_segment_with_anchor_moves_only_what_differs_from_the_anchor(F):
    """Kind-1 chunks with prox > 0, wd = 0, no momentum: w == a stays bit-exact (and is not rewritten), w != a gets the
    proximal step exactly as the arena kernel computes it with a zero gradient; the gradient is never touched."""
    dev = torch.device("cuda:0")
    n = 3 * 8192 + 42                                    # the last chunk has a scalar tail
    gen = torch.Generator(device=dev).manual_seed(4)
    theta0 = torch.randn(n, device=dev, generator=gen)
    anchor = theta0.clone()
    # whole float4 groups move (a vector store covers four elements), so each group is either all equal or all different
    moved = (torch.rand((n + 3) // 4, device=dev, generator=gen) < 0.3).repeat_interleave(4)[:n]
    anchor[moved] += torch.randn(int(moved.sum()), device=dev, generator=gen)
    hyper = torch.tensor([0.1, 0.0, 0.0, 0.0, 0.25], device=dev)
    segs = torch.tensor([[0, 8192, 1], [8192, 8192, 0], [16384, n - 16384, 1]], dtype=torch.int64, device=dev)
    ng = torch.cat([torch.arange(0, 8192), torch.arange(16384, n)]).to(dev)
    stale = theta0.to(BF16)
    stale[ng[~moved[ng]]] = 0                            # a rewritten shadow element would be refreshed; these must not be
    theta, grad, wb = theta0.clone(), torch.full((n,), float("nan"), device=dev), stale.clone()
    grad[8192:16384] = 1.0
    F.fused_sgd_segments(theta, grad, hyper, segs, None, wb, prox_anchor=anchor)
    ref = theta0.clone()
    F.fused_sgd(ref, torch.zeros(n, device=dev), hyper, None, None, prox_anchor=anchor)
    torch.cuda.synchronize()
    same, diff = ng[~moved[ng]], ng[moved[ng]]
    assert torch.equal(_bits(theta[same]), _bits(theta0[same]))
    assert (wb[same] == 0).all(), "an element equal to its anchor must not be written"
    assert torch.equal(_bits(theta[diff]), _bits(ref[diff]))
    assert torch.equal(wb[diff], theta[diff].to(BF16))
    want = theta0[diff].double() - 0.1 * 0.25 * (theta0[diff].double() - anchor[diff].double())
    assert torch.allclose(theta[diff].double(), want, rtol=0, atol=1e-6)
    assert torch.isnan(grad[ng]).all(), "a no-grad segment must not read or write the gradient"
    assert (grad[8192:16384] == 0).all()


def _resnet_trainer(dev, use_graph=True, seed=0):
    from baton_b200.models import resnet18
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.train import GraphedLocalSGD
    torch.manual_seed(seed)
    m = resnet18(10)
    arena = ParamArena(m, dev)
    m.build_workspace(dev)
    tr = GraphedLocalSGD(m, arena, loss="ce", use_graph=use_graph)
    m._graphed_trainer = tr
    return m, arena, tr


def _image_data(dev, n=512):
    from baton_b200.data import ShardSpec, image_shard
    X, y = image_shard(ShardSpec(0, torch.full((10,), 0.1), n), noise=0.3)
    return X.to(dev).to(BF16), y.to(dev)


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def test_graphed_resnet18_fedprox_matches_eager_pulls_toward_global_and_reuses_graphs():
    dev = torch.device("cuda:0")
    X, y = _image_data(dev)
    kw = dict(n_epoch=2, lr=0.05, batch_size=128)

    def run(use_graph, mu):
        m, arena, tr = _resnet_trainer(dev, use_graph)
        torch.manual_seed(9)
        m.train(X, y, prox_mu=mu, **kw)
        torch.cuda.synchronize()
        n = arena.n_param
        return arena.theta[:n].clone(), arena.global_w[:n].clone()

    # graphed vs eager, calibrated by graphed vs graphed (the BatchNorm statistics use fp32 atomics)
    (a, g0), (b, _), (c, _) = run(True, 0.1), run(True, 0.1), run(False, 0.1)
    noise, diff = _rel(b - g0, a - g0), _rel(c - g0, a - g0)
    print("update rel diff: graphed/graphed {:.2e}, graphed/eager {:.2e}".format(noise, diff))
    assert diff <= 3.0 * noise + 2e-3, (diff, noise)
    # the proximal term shortens the round's step
    dist = [float((run(True, mu)[0] - g0).norm()) for mu in (0.0, 0.1, 1.0)]
    assert dist[0] > dist[1] > dist[2] > 0, dist
    # the coefficient lives in device memory: only switching the term on adds a graph
    m, arena, tr = _resnet_trainer(dev)
    m.train(X, y, prox_mu=0.0, **kw)
    n0 = len(tr._graphs)
    m.train(X, y, prox_mu=0.01, **kw)
    assert len(tr._graphs) == n0 + 1
    m.train(X, y, prox_mu=0.1, **kw)
    assert len(tr._graphs) == n0 + 1
    assert torch.equal(arena.theta_bf16[: arena.n_param], arena.theta[: arena.n_param].to(BF16))


def test_mlp_autograd_path_fedprox_matches_torch_oracle():
    from baton_b200.models import MLP2
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.train import GraphedLocalSGD
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    m = MLP2(16, 64, 1)                     # 64-byte fp32 rows: the on-device batch gather moves 16-byte vectors
    oracle = MLP2(16, 64, 1).to(dev)
    oracle.load_state_dict(m.state_dict())
    arena = ParamArena(m, dev)
    arena.global_w.add_(torch.randn_like(arena.global_w) * 0.05)        # the round's global model != the weights
    anchors = [arena._view(arena.global_w, arena.slots[k]).clone() for k, _ in m.named_parameters()]
    tr = GraphedLocalSGD(m, arena, loss="mse")
    m._graphed_trainer = tr
    X = torch.randn(256, 16, device=dev)
    y = X @ torch.arange(1.0, 17.0, device=dev).unsqueeze(1)
    lr, mu = 0.01, 0.5
    m.train(X, y, n_epoch=3, lr=lr, batch_size=256, prox_mu=mu)        # one full batch per epoch
    for _ in range(3):
        oracle.zero_grad(set_to_none=True)
        torch.nn.functional.mse_loss(oracle(X), y).backward()
        with torch.no_grad():
            for p, a in zip(oracle.parameters(), anchors):
                p.sub_(lr * (p.grad + mu * (p - a)))
    torch.cuda.synchronize()
    for (k, p), q in zip(m.named_parameters(), oracle.parameters()):
        assert torch.allclose(p, q, rtol=1e-4, atol=1e-5), (k, float((p - q).abs().max()))


@pytest.mark.parametrize("wire,mode", [("bf16", "delta"), ("fp32", "delta"), ("bf16", "weights")])
def test_fedprox_upload_copy_emitted_by_the_optimizer_matches_in_kernel_pack(wire, mode):
    """The last FedProx step writes the wire copy itself, reading the anchor once where it is also the delta base;
    the round result must equal that of the collective's own pack."""
    from baton_b200.models import resnet18
    from baton_b200.ops import functional as F
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.fedavg import FedAvgSession
    dev = torch.device("cuda:0")
    results = []
    for prepack in (False, True):
        torch.manual_seed(0)
        m = resnet18(10)
        arena = ParamArena(m, dev)
        sess = FedAvgSession(arena, wire_dtype=wire, mode=mode, n_ctas=32)
        hyper = torch.tensor([0.1, 0.0, 0.0, 0.0, 0.1], device=dev)
        gen = torch.Generator(device=dev).manual_seed(7)
        for rnd in range(3):
            arena.theta[: arena.n_param].add_(torch.randn(arena.n_param, device=dev, generator=gen) * 0.01)
            arena.grad.copy_(torch.randn(arena.n_param, device=dev, generator=gen) * 0.01)
            arena.theta[arena.n_param:].add_(0.001 * (rnd + 1))
            if prepack:
                sess.arm_prepack(64.0)
            F.fused_sgd(arena.theta[: arena.n_param], arena.grad, hyper, None, arena.theta_bf16[: arena.n_param],
                        pack=sess.pack_spec() if prepack else None, prox_anchor=arena.global_w[: arena.n_param])
            sess.aggregate(my_n=64.0, prepacked=prepack)
            assert sess.last_prepacked == prepack
        torch.cuda.synchronize()
        sess.check()
        results.append((arena.theta.clone(), arena.global_w.clone(), arena.theta_bf16.clone()))
    for a, b in zip(*results):
        assert torch.equal(a, b)


def test_fedprox_engine_rounds_with_tile_flags_match_plain_engine():
    """K3 gates the head of the next round's epoch on the collective's arrival flags; every SGD kernel that reads the
    anchor runs after the join, so tile_flags=True gives the global model of tile_flags=False within the atomics'
    run-to-run spread (calibrated by two plain runs)."""
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    dev = torch.device("cuda:0")
    X, y = _image_data(dev, 1024)

    def run(k3):
        torch.manual_seed(0)
        eng = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, tile_flags=k3, n_ctas=64,
                              prox_mu=0.1)
        assert eng.k3 == k3 and eng.hp["prox_mu"] == 0.1
        g0 = eng.arena.global_w.clone()
        hist = []
        for _ in range(4):
            hist += eng.run_round((X, y), n_epoch=1).loss_history
        eng.sync()
        torch.cuda.synchronize()
        eng.session.check()
        if k3:
            assert next(iter(eng.trainer._graphs.values()))["graph2"] is not None
            assert eng.session.last_prepacked
        assert torch.equal(eng.arena.theta, eng.arena.global_w)
        return eng.arena.global_w[: eng.arena.n_param] - g0[: eng.arena.n_param], hist

    (a, ha), (b, _), (c, hc) = run(False), run(False), run(True)
    noise, diff = _rel(b, a), _rel(c, a)
    print("global update rel diff: plain/plain {:.2e}, plain/k3 {:.2e}".format(noise, diff))
    assert diff <= 3.0 * noise + 2e-3, (diff, noise)
    assert hc[-1] < hc[0], hc
