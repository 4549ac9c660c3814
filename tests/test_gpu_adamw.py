"""Local AdamW on the GPU: the AdamW step of the three optimizer sites (arena pass, leftover segment pass, optimizer
epilogue of the weight-gradient GEMMs), the upload copy it emits, graphed ResNet-18 epochs, BERT and engine rounds."""
import math

import pytest
import torch

from test_gpu_fedprox import SHAPES, _bits, _image_data, _rel, _resnet_trainer

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
DEV = torch.device("cuda:0")
LR, BETAS, EPS = 0.01, (0.9, 0.999), 1e-8


@pytest.fixture(scope="module")
def F():
    from baton_b200.ops import functional
    return functional


def _row(F, t, wd, lr=LR):
    """Device AdamW row of step t."""
    return F.adamw_rows(lr, BETAS, EPS, wd, t, 1)[0].to(DEV)


def _formula64(w, g, m, v, t, wd, lr=LR):
    """fp64 AdamW step t (torch.optim.AdamW's update); m and v are ignored at t == 1.  Returns (w, m, v)."""
    b1, b2 = BETAS
    w, g = w.double(), g.double()
    m0 = torch.zeros_like(w) if t == 1 else m.double()
    v0 = torch.zeros_like(w) if t == 1 else v.double()
    m = b1 * m0 + (1 - b1) * g
    v = b2 * v0 + (1 - b2) * g * g
    w = w * (1 - lr * wd) - lr / (1 - b1 ** t) * m / (v.sqrt() / math.sqrt(1 - b2 ** t) + EPS)
    return w, m, v


def _state(n, seed, garbage):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    w = torch.randn(n, device=DEV, generator=gen)
    g = torch.randn(n, device=DEV, generator=gen)
    if garbage:       # what t == 1 must ignore: huge, negative and non-finite moments
        m = torch.full((n,), float("nan"), device=DEV)
        v = torch.full((n,), -1e30, device=DEV)
    else:
        m = 0.1 * torch.randn(n, device=DEV, generator=gen)
        v = torch.rand(n, device=DEV, generator=gen)
    return w, g, m, v


@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("t", [1, 7])
def test_fused_sgd_adamw_matches_fp64_formula(F, t, wd):
    n = 8192 + 24
    w0, g0, m0, v0 = _state(n, 1, garbage=(t == 1))
    want_w, want_m, want_v = _formula64(w0, g0, m0, v0, t, wd)
    glob = w0 + 0.5
    for wire_fp32 in (None, False, True):
        w, g, m, v, wb = w0.clone(), g0.clone(), m0.clone(), v0.clone(), w0.to(BF16)
        pack, wire = None, None
        if wire_fp32 is not None:
            wire = torch.zeros(n, dtype=torch.float32 if wire_fp32 else BF16, device=DEV)
            slot = torch.tensor([wire.data_ptr()], dtype=torch.int64, device=DEV)
            pack = {"wire_slot": slot, "global_w": glob, "scale": torch.tensor([3.0], device=DEV), "n_pack": n,
                    "wire_fp32": wire_fp32}
        F.fused_sgd(w, g, _row(F, t, wd), m, wb, zero_grad=True, pack=pack, adam_v=v)
        torch.cuda.synchronize()
        assert torch.allclose(w.double(), want_w, rtol=1e-6, atol=1e-6), float((w.double() - want_w).abs().max())
        assert torch.allclose(m.double(), want_m, rtol=1e-6, atol=1e-7)
        assert torch.allclose(v.double(), want_v, rtol=1e-6, atol=1e-9)
        assert (g == 0).all()
        assert torch.equal(wb, w.to(BF16))
        if wire is not None:
            d = (w - glob) * 3.0
            assert torch.equal(_bits(wire), _bits(d if wire_fp32 else d.to(BF16)))


@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("t", [1, 3])
def test_segments_adamw_kinds(F, t, wd):
    """Kind 0 is the arena kernel's step bit for bit.  Kind 1 is the step with g = 0: with wd == 0 after the first
    step it is skipped (nothing is read or written); at the first step it runs and leaves m = v = 0."""
    n = 3 * 8192 + 42
    w0, g0, m0, v0 = _state(n, 4, garbage=(t == 1))
    if t > 1:                 # a kind-1 element's moments are 0 after the first step of a run
        m0[:8192] = 0
        v0[:8192] = 0
        m0[16384:] = 0
        v0[16384:] = 0
    segs = torch.tensor([[0, 8192, 1], [8192, 8192, 0], [16384, n - 16384, 1]], dtype=torch.int64, device=DEV)
    ng = torch.cat([torch.arange(0, 8192), torch.arange(16384, n)]).to(DEV)
    row = _row(F, t, wd)
    w, g, m, v = w0.clone(), g0.clone(), m0.clone(), v0.clone()
    g[ng] = float("nan")                     # never read
    wb = torch.zeros(n, dtype=BF16, device=DEV)
    F.fused_sgd_segments(w, g, row, segs, m, wb, adam_v=v)
    # reference: the arena kernel with the true gradient (zero on kind-1 elements)
    wr, gr, mr, vr = w0.clone(), g0.clone(), m0.clone(), v0.clone()
    gr[ng] = 0
    F.fused_sgd(wr, gr, row, mr, None, adam_v=vr)
    torch.cuda.synchronize()
    k0 = torch.arange(8192, 16384, device=DEV)
    for got, ref in ((w, wr), (m, mr), (v, vr)):
        assert torch.equal(_bits(got[k0]), _bits(ref[k0]))
    assert (g[k0] == 0).all() and torch.isnan(g[ng]).all()
    assert torch.equal(wb[k0], w[k0].to(BF16))
    skipped = wd == 0.0 and t > 1
    if skipped or wd == 0.0:
        assert torch.equal(_bits(w[ng]), _bits(w0[ng])) and (wb[ng] == 0).all()
    else:
        assert torch.equal(_bits(w[ng]), _bits(wr[ng])) and torch.equal(wb[ng], w[ng].to(BF16))
        assert torch.equal(w[ng], w0[ng] * (1 - LR * wd))
    if skipped:
        assert torch.equal(_bits(m[ng]), _bits(m0[ng])) and torch.equal(_bits(v[ng]), _bits(v0[ng]))
    else:
        assert (m[ng] == 0).all() and (v[ng] == 0).all()


@pytest.mark.parametrize("t,wd", [(1, 0.0), (5, 0.1)])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_epilogue_adamw_matches_accumulate_then_fused_sgd(F, shape, t, wd):
    torch.manual_seed(0)
    xs, k, stride, pad, cout = SHAPES[shape]
    n_img, h, _, c = xs
    ho = F.conv_out_size(h, k, stride, pad)
    x = torch.randn(xs, device=DEV).to(BF16)
    dy = torch.randn(n_img * ho * ho, cout, device=DEV).to(BF16)
    centre = shape.startswith("centre")
    numel = cout * k * k * c
    off = 1024
    n = off + numel + 1032
    theta0 = torch.randn(n, device=DEV) * 0.05
    m0 = torch.randn(n, device=DEV) * 0.01
    v0 = torch.rand(n, device=DEV) * 1e-4
    if centre:                # the off-centre taps never had a gradient: their moments are 0
        tap = torch.zeros(cout, k * k, c, dtype=torch.bool, device=DEV)
        tap[:, (k * k) // 2, :] = True
        sl = slice(off, off + numel)
        m0[sl] = torch.where(tap.flatten(), m0[sl], torch.zeros_like(m0[sl]))
        v0[sl] = torch.where(tap.flatten(), v0[sl], torch.zeros_like(v0[sl]))
    row = _row(F, t, wd)

    def state():
        grad = torch.zeros(n, device=DEV)
        grad[:off] = torch.linspace(-1.0, 1.0, off, device=DEV)
        grad[off + numel:] = torch.linspace(-0.5, 0.5, n - off - numel, device=DEV)
        theta = theta0.clone()
        return theta, grad, theta.to(BF16), m0.clone(), v0.clone()

    def out_view(grad):
        w2d = grad[off: off + numel].view(cout, k * k * c)
        return w2d.view(cout, k * k, c)[:, (k * k) // 2, :] if centre else w2d

    def wgrad(out2d, sgd=None):
        if centre:
            return F.gemm(dy, x.view(n_img, c), a_mn=True, b_mn=True, out=out2d, accumulate=True, sgd=sgd) is not None
        return F.conv_igemm_wgrad_(dy, x, out2d, k, k, stride, pad, sgd=sgd)

    theta_r, grad_r, wb_r, m_r, v_r = state()
    assert wgrad(out_view(grad_r))
    F.fused_sgd(theta_r, grad_r, row, m_r, wb_r, zero_grad=True, adam_v=v_r)

    theta, grad, wb, m, v = state()
    out2d = out_view(grad)
    assert wgrad(out2d, F.sgd_epilogue_args(theta, grad, out2d, row, m, wb, adam_v=v)), "declined"
    assert (grad[off: off + numel] == 0).all()
    fused = [(off + (4 * c if centre else 0), out2d.shape[0], out2d.shape[1], out2d.stride(0))]
    segs = F.sgd_segments(n, fused, [(off, numel)] if centre else [])
    F.fused_sgd_segments(theta, grad, row, torch.tensor(segs, dtype=torch.int64, device=DEV), m, wb, adam_v=v)
    torch.cuda.synchronize()
    for got, ref in ((theta, theta_r), (wb, wb_r), (m, m_r), (v, v_r)):
        assert torch.equal(_bits(got), _bits(ref))


@pytest.mark.parametrize("wire", ["fp32", "bf16"])
def test_adamw_emitted_upload_equals_collective_pack(F, wire):
    from baton_b200.models import resnet18
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.fedavg import FedAvgSession

    def run(prepack):
        torch.manual_seed(0)
        arena = ParamArena(resnet18(10), DEV, momentum=True)
        v = torch.zeros(arena.n_param, device=DEV)
        sess = FedAvgSession(arena, wire_dtype=wire, mode="delta", n_ctas=32, nvls=False)
        gen = torch.Generator(device=DEV).manual_seed(7)
        for t in (1, 2, 3):
            arena.grad.copy_(torch.randn(arena.n_param, device=DEV, generator=gen) * 0.01)
            if prepack:
                sess.arm_prepack(64.0)
            F.fused_sgd(arena.theta[: arena.n_param], arena.grad, _row(F, t, 0.05), arena.momentum,
                        arena.theta_bf16[: arena.n_param], pack=sess.pack_spec() if prepack else None, adam_v=v)
            sess.aggregate(my_n=64.0, prepacked=prepack)
            assert sess.last_prepacked == prepack
        torch.cuda.synchronize()
        sess.check()
        return arena.global_w.clone(), arena.theta_bf16.clone()

    (g, b), (gp, bp) = run(False), run(True)
    assert torch.equal(_bits(gp), _bits(g)) and torch.equal(_bits(bp), _bits(b))


def test_graphed_resnet18_adamw_matches_eager_across_epochs(monkeypatch):
    """Two epochs with a ragged last batch: graphed == eager within the run-to-run spread of the BatchNorm statistics'
    fp32 atomics.  A bias correction that restarted every epoch (the captured step index reused as t) misses by far."""
    from baton_b200.train import GraphedLocalSGD
    X, y = _image_data(DEV, 600)                      # 4 full batches of 128 + a ragged one of 88
    # with a tiny eps, AdamW moves every element by about lr whatever its gradient, so elements whose gradient is at the
    # level of the atomics' rounding move in random directions; eps = 1e-4 keeps them still and the comparison sharp
    kw = dict(n_epoch=2, lr=1e-3, batch_size=128, weight_decay=0.01, optimizer="adamw", eps=1e-4)

    def run(use_graph):
        m, arena, tr = _resnet_trainer(DEV, use_graph)
        n = arena.n_param
        g0 = arena.theta[:n].clone()
        torch.manual_seed(9)
        m.train(X, y, **kw)
        torch.cuda.synchronize()
        assert torch.equal(arena.theta_bf16[:n], arena.theta[:n].to(BF16))
        return arena.theta[:n] - g0

    a, b, c = run(True), run(True), run(False)
    noise, diff = _rel(b, a), _rel(c, a)
    orig = GraphedLocalSGD._adam_rows

    def restart_each_epoch(self, lr, betas, eps, wd, n_epoch, steps):
        one = orig(self, lr, betas, eps, wd, 1, steps)
        return one.repeat(n_epoch, 1)
    monkeypatch.setattr(GraphedLocalSGD, "_adam_rows", restart_each_epoch)
    wrong = run(True)
    bad = _rel(wrong, a)
    print("2-epoch update rel diff: graphed/graphed {:.2e}, graphed/eager {:.2e}, per-epoch restart {:.2e}".format(
        noise, diff, bad))
    assert diff <= 3.0 * noise + 2e-2, (diff, noise)
    assert bad > 5.0 * max(diff, noise) and bad > 0.05, (bad, diff, noise)


def test_bert_tiny_adamw_matches_fp32_torch_adamw_and_trains():
    from baton_b200.models import bert_tiny
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.train import GraphedLocalSGD
    torch.manual_seed(2)
    m = bert_tiny(3)
    ref = bert_tiny(3)
    ref.load_state_dict(m.state_dict())
    arena = ParamArena(m, DEV)
    tr = GraphedLocalSGD(m, arena, loss="ce")
    m._graphed_trainer = tr
    X = torch.randint(0, 1024, (64, 64))
    yy = X[:, :8].sum(1) % 3
    lr, wd, steps = 1e-3, 0.01, 3
    before = {k: p.detach().float().cpu().clone() for k, p in m.named_parameters()}
    m.train(X.to(DEV), yy.to(DEV), n_epoch=steps, lr=lr, batch_size=64, weight_decay=wd, optimizer="adamw")
    opt = torch.optim.AdamW(ref.parameters(), lr=lr, weight_decay=wd)
    for _ in range(steps):                            # full batch: the sample order does not matter
        opt.zero_grad()
        torch.nn.functional.cross_entropy(ref(X), yy).backward()
        opt.step()
    refp = dict(ref.named_parameters())
    got = torch.cat([(p.detach().float().cpu() - before[k]).flatten() for k, p in m.named_parameters()])
    want = torch.cat([(refp[k].detach() - before[k]).flatten() for k, _ in m.named_parameters()])
    cos = float(torch.nn.functional.cosine_similarity(got, want, dim=0))
    print("bert_tiny 3-step AdamW update: cosine {:.4f}, rel diff {:.3e}".format(cos, _rel(got, want)))
    assert cos > 0.9 and _rel(got, want) < 0.5, (cos, _rel(got, want))
    X2 = torch.randint(0, 1024, (256, 64), device=DEV)
    y2 = X2[:, :8].sum(1) % 3
    hist = m.train(X2, y2, n_epoch=8, lr=1e-3, batch_size=32, optimizer="adamw")
    assert hist[-1] < hist[0], hist


def test_world1_engine_adamw_logical_clients_with_dp():
    """3 logical clients and DP clipping (noise 0 so the two sessions can be compared) on one GPU: the fused collective
    and the NCCL session agree, and each client's AdamW run starts fresh (a second engine replaying the same rounds
    gives the same bits)."""
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
    gen = torch.Generator().manual_seed(1)
    shards = {}
    for cid in range(3):
        Xc = torch.randn(128 + 64 * cid, 16, generator=gen)
        shards[cid] = (Xc.to(DEV), (Xc @ (torch.arange(1.0, 17.0) * (1 + 0.5 * cid))).unsqueeze(1).to(DEV))
    out = {}
    for backend in ("fused", "nccl", "fused2"):
        torch.manual_seed(0)
        eng = FederatedEngine(MLP2(16, 64, 1), DEV, backend=backend.rstrip("2"), loss="mse", lr=0.01, batch_size=64,
                              wire_dtype="fp32", optimizer="adamw", weight_decay=0.01, logical_clients=3, seed=11,
                              dp_clip=5.0, dp_noise_multiplier=0.0, dp_seed=3)
        g0 = eng.arena.global_w.clone()
        for _ in range(3):
            eng.run_round(lambda cid: shards[cid], n_epoch=2)
        eng.sync()
        torch.cuda.synchronize()
        assert eng.arena.adam_v is not None and torch.isfinite(eng.arena.global_w).all()
        out[backend] = eng.arena.global_w.clone()
        assert float((out[backend] - g0).abs().max()) > 0
    assert _rel(out["fused"], out["nccl"]) < 1e-5, _rel(out["fused"], out["nccl"])
    assert _rel(out["fused2"], out["fused"]) < 1e-6
