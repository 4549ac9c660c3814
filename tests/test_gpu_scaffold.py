"""SCAFFOLD on the GPU: the correction term in the SGD kernels (arena pass, leftover segment pass, optimizer epilogue of
the weight-gradient GEMMs), the control-variate kernels, the SCAFFOLD collective and engine rounds."""
import os
import subprocess
import sys

import pytest
import torch

from test_gpu_fedprox import HYPER, LR, SHAPES, _bits, _image_data, _rel

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def F():
    from baton_b200.ops import functional
    return functional


def _formula64(w, g, corr, m, lr, mom, wd, nesterov):
    """fp64 SCAFFOLD step (torch.optim.SGD with dampening 0 on g + wd*w + corr); returns (w, m)."""
    w, g, corr = w.double(), g.double(), corr.double()
    gp = g + wd * w + corr
    if m is None:
        return w - lr * gp, None
    m = mom * m.double() + gp
    step = gp + mom * m if nesterov else m
    return w - lr * step, m


@pytest.mark.parametrize("mu,nesterov,wd", HYPER)
def test_fused_sgd_with_corr_matches_fp64_formula(F, mu, nesterov, wd):
    gen = torch.Generator(device=DEV).manual_seed(1)
    n = 8192 + 24
    w0 = torch.randn(n, device=DEV, generator=gen)
    glob = w0 + 0.5 * torch.randn(n, device=DEV, generator=gen)
    g0 = torch.randn(n, device=DEV, generator=gen)
    corr = 0.3 * torch.randn(n, device=DEV, generator=gen)
    m0 = torch.randn(n, device=DEV, generator=gen) * 0.1 if mu else None
    hyper = torch.tensor([LR, mu, wd, 0.0], device=DEV)
    want_w, want_m = _formula64(w0, g0, corr, m0, LR, mu, wd, nesterov)
    for wire_fp32 in (None, False, True):
        w, g, wb = w0.clone(), g0.clone(), w0.to(BF16)
        m = m0.clone() if m0 is not None else None
        pack, wire = None, None
        if wire_fp32 is not None:
            wire = torch.zeros(n, dtype=torch.float32 if wire_fp32 else BF16, device=DEV)
            slot = torch.tensor([wire.data_ptr()], dtype=torch.int64, device=DEV)
            pack = {"wire_slot": slot, "global_w": glob, "scale": torch.tensor([3.0], device=DEV), "n_pack": n,
                    "wire_fp32": wire_fp32}
        F.fused_sgd(w, g, hyper, m, wb, zero_grad=True, nesterov=nesterov, pack=pack, corr=corr)
        torch.cuda.synchronize()
        assert torch.allclose(w.double(), want_w, rtol=1e-6, atol=1e-6), float((w.double() - want_w).abs().max())
        if m is not None:
            assert torch.allclose(m.double(), want_m, rtol=1e-6, atol=1e-6)
        assert (g == 0).all()
        assert torch.equal(wb, w.to(BF16))
        if wire is not None:          # the upload is the new weights' delta, whatever term moved them
            d = (w - glob) * 3.0
            assert torch.equal(_bits(wire), _bits(d if wire_fp32 else d.to(BF16)))
    # a zero correction is the plain step, bit for bit
    w, wp = w0.clone(), w0.clone()
    F.fused_sgd(w, g0.clone(), hyper, m0.clone() if m0 is not None else None, corr=torch.zeros_like(corr),
                nesterov=nesterov)
    F.fused_sgd(wp, g0.clone(), hyper, m0.clone() if m0 is not None else None, nesterov=nesterov)
    torch.cuda.synchronize()
    assert torch.equal(_bits(w), _bits(wp))


def test_nograd_segment_with_corr_moves_by_minus_lr_corr(F):
    """Kind-1 chunks are not skipped with a correction: they move by -lr * corr (bit-equal to the arena kernel with a
    zero gradient), elements with a zero correction are not rewritten, the gradient is never touched."""
    n = 3 * 8192 + 42
    gen = torch.Generator(device=DEV).manual_seed(4)
    theta0 = torch.randn(n, device=DEV, generator=gen)
    moved = (torch.rand((n + 3) // 4, device=DEV, generator=gen) < 0.3).repeat_interleave(4)[:n]
    corr = torch.zeros(n, device=DEV)
    corr[moved] = torch.randn(int(moved.sum()), device=DEV, generator=gen)
    hyper = torch.tensor([0.1, 0.0, 0.0, 0.0], device=DEV)
    segs = torch.tensor([[0, 8192, 1], [8192, 8192, 0], [16384, n - 16384, 1]], dtype=torch.int64, device=DEV)
    ng = torch.cat([torch.arange(0, 8192), torch.arange(16384, n)]).to(DEV)
    stale = theta0.to(BF16)
    stale[ng[~moved[ng]]] = 0
    theta, grad, wb = theta0.clone(), torch.full((n,), float("nan"), device=DEV), stale.clone()
    grad[8192:16384] = 1.0
    F.fused_sgd_segments(theta, grad, hyper, segs, None, wb, corr=corr)
    ref = theta0.clone()
    F.fused_sgd(ref, torch.zeros(n, device=DEV), hyper, None, None, corr=corr)
    torch.cuda.synchronize()
    same, diff = ng[~moved[ng]], ng[moved[ng]]
    assert torch.equal(_bits(theta[same]), _bits(theta0[same]))
    assert (wb[same] == 0).all(), "an element with a zero correction must not be written"
    assert torch.equal(_bits(theta[diff]), _bits(ref[diff]))
    assert torch.equal(wb[diff], theta[diff].to(BF16))
    want = theta0[diff].double() - 0.1 * corr[diff].double()
    assert torch.allclose(theta[diff].double(), want, rtol=0, atol=1e-6)
    assert torch.isnan(grad[ng]).all()
    assert (grad[8192:16384] == 0).all()


@pytest.mark.parametrize("mu,nesterov,wd", HYPER)
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_epilogue_with_corr_matches_accumulate_then_fused_sgd(F, shape, mu, nesterov, wd):
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
    corr = torch.randn(n, device=DEV) * 0.02
    mom0 = torch.randn(n, device=DEV) * 0.01 if mu else None
    hyper = torch.tensor([0.05, mu, wd, 0.0], device=DEV)

    def state():
        grad = torch.zeros(n, device=DEV)
        grad[:off] = torch.linspace(-1.0, 1.0, off, device=DEV)
        grad[off + numel:] = torch.linspace(-0.5, 0.5, n - off - numel, device=DEV)
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
    F.fused_sgd(theta_r, grad_r, hyper, mom_r, wb_r, zero_grad=True, nesterov=nesterov, corr=corr)

    theta, grad, wb, mom = state()
    out2d = out_view(grad)
    assert wgrad(out2d, F.sgd_epilogue_args(theta, grad, out2d, hyper, mom, wb, nesterov, corr=corr)), "declined"
    assert (grad[off: off + numel] == 0).all()
    fused = [(off + (4 * c if centre else 0), out2d.shape[0], out2d.shape[1], out2d.stride(0))]
    segs = F.sgd_segments(n, fused, [(off, numel)] if centre else [])
    F.fused_sgd_segments(theta, grad, hyper, torch.tensor(segs, dtype=torch.int64, device=DEV), mom, wb,
                         nesterov=nesterov, corr=corr)
    torch.cuda.synchronize()
    assert torch.equal(_bits(theta), _bits(theta_r))
    assert torch.equal(_bits(wb), _bits(wb_r))
    if mom is not None:
        assert torch.equal(_bits(mom), _bits(mom_r))


def test_control_variate_kernels_match_their_formulas(F):
    n = 4096 + 8
    gen = torch.Generator(device=DEV).manual_seed(2)
    c, ci, g, t, up0 = (torch.randn(n, device=DEV, generator=gen) for _ in range(5))
    corr = torch.empty(n, device=DEV)
    F.scaffold_corr(corr, c, ci)
    inv = 1.0 / (12 * 0.05)
    want_dc = (g.double() - t.double()) * inv - c.double()
    for first in (True, False):
        cv, up = ci.clone(), up0.clone()
        F.scaffold_dc(up, cv, c, g, t, inv, first=first)
        torch.cuda.synchronize()
        assert torch.allclose(cv.double(), ci.double() + want_dc, rtol=1e-6, atol=1e-5)
        want_up = want_dc if first else up0.double() + want_dc
        assert torch.allclose(up.double(), want_up, rtol=1e-6, atol=1e-5)
    assert torch.equal(corr, c - ci)


@pytest.mark.parametrize("wire", ["fp32", "bf16", "fp8"])
def test_world1_scaffold_collective(wire):
    """Segment 0 == the plain collective bit for bit, c == c + cast(dc) / N, prepacked == in-kernel pack, and the
    result does not depend on the CTA count or the tile size."""
    from baton_b200.models import resnet18
    from baton_b200.ops import functional as F
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.fedavg import FedAvgSession
    n_clients = 4

    def run(scaffold, prepack=False, n_ctas=32, tile=0):
        torch.manual_seed(0)
        arena = ParamArena(resnet18(10), DEV)
        sess = FedAvgSession(arena, wire_dtype=wire, mode="delta", n_ctas=n_ctas, tile_elems=tile, nvls=False,
                             scaffold=scaffold)
        c = torch.zeros(arena.n_param, device=DEV)
        gen = torch.Generator(device=DEV).manual_seed(7)
        hyper = torch.tensor([0.1, 0.0, 0.0, 0.0], device=DEV)
        dcs = []
        for _ in range(3):
            arena.grad.copy_(torch.randn(arena.n_param, device=DEV, generator=gen) * 0.01)
            dc = torch.randn(arena.n_param, device=DEV, generator=gen)
            dcs.append(dc)
            if prepack:
                sess.arm_prepack(64.0)
            F.fused_sgd(arena.theta[: arena.n_param], arena.grad, hyper, None, arena.theta_bf16[: arena.n_param],
                        pack=sess.pack_spec() if prepack else None)
            sess.aggregate(my_n=64.0, prepacked=prepack, control=(c, dc, n_clients) if scaffold else None)
            assert sess.last_prepacked == (prepack and wire != "fp8")
        torch.cuda.synchronize()
        sess.check()
        return arena.global_w.clone(), arena.theta_bf16.clone(), c, dcs

    g_plain, b_plain, _, _ = run(False)
    g, b, c, dcs = run(True)
    assert torch.equal(_bits(g), _bits(g_plain)) and torch.equal(_bits(b), _bits(b_plain))
    if wire == "fp8":                         # e4m3 with a shared power-of-two scale per 32 elements
        ref = sum(dcs) / n_clients
        assert float((c - ref).abs().max()) <= 0.2 * float(ref.abs().max())
    else:                                     # 1 / N = 1 / 4 scales exactly: c = sum of cast(dc) / N, bit for bit
        want = torch.zeros_like(c)
        for dc in dcs:
            want = want + (dc if wire == "fp32" else dc.to(BF16).float()) / n_clients
        assert torch.equal(_bits(c), _bits(want))
    for kw in ({"prepack": True}, {"n_ctas": 7, "tile": 4096}, {"n_ctas": 132, "tile": 1024}):
        g2, b2, c2, _ = run(True, **kw)
        assert torch.equal(_bits(g2), _bits(g)) and torch.equal(_bits(c2), _bits(c)), kw


def test_resnet18_first_scaffold_round_equals_plain_round():
    """From c = c_i = 0 the correction is zero, so the first round's global model is the plain engine's -- within the
    run-to-run spread of the BatchNorm statistics' fp32 atomics (calibrated by two plain runs)."""
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    X, y = _image_data(DEV, 1024)

    def run(scaffold):
        torch.manual_seed(0)
        eng = FederatedEngine(resnet18(10), DEV, backend="fused", lr=0.05, batch_size=128, n_ctas=64,
                              scaffold=scaffold)
        g0 = eng.arena.global_w.clone()
        eng.run_round((X, y), n_epoch=1)
        eng.sync()
        torch.cuda.synchronize()
        eng.session.check()
        if scaffold:
            c, ci = eng.control_variates()
            assert sorted(ci) == [0] and float(c.abs().max()) > 0.0
            assert torch.equal(c, ci[0].to(BF16).float())     # N = 1: c = cast(dc_0) on the bf16 wire, c_0 = dc_0
        return eng.arena.global_w - g0

    a, b, s = run(False), run(False), run(True)
    noise, diff = _rel(b, a), _rel(s, a)
    print("first-round update rel diff: plain/plain {:.2e}, plain/scaffold {:.2e}".format(noise, diff))
    assert diff <= 3.0 * noise + 1e-6, (diff, noise)


def test_scaffold_engine_fused_matches_nccl_logical_clients():
    """4 logical clients, 2 sampled per round, 3 rounds, fp32 wire: the fused collective and the NCCL session give the
    same global model, c and c_i; c is the mean of all N client variates."""
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
    gen = torch.Generator().manual_seed(1)
    shards = {}
    for cid in range(4):
        X = torch.randn(128 + 64 * cid, 16, generator=gen)
        shards[cid] = (X.to(DEV), (X @ (torch.arange(1.0, 17.0) * (1 + 0.5 * cid))).unsqueeze(1).to(DEV))
    out = {}
    for backend in ("fused", "nccl"):
        torch.manual_seed(0)
        eng = FederatedEngine(MLP2(16, 64, 1), DEV, backend=backend, loss="mse", lr=0.002, batch_size=64,
                              wire_dtype="fp32", scaffold=True, logical_clients=4, sample_k=2, seed=11)
        for _ in range(3):
            eng.run_round(lambda cid: shards[cid], n_epoch=2)
        eng.sync()
        torch.cuda.synchronize()
        c, ci = eng.control_variates()
        out[backend] = (eng.arena.global_w.clone(), c.clone(), {k: v.clone() for k, v in ci.items()})
    (gf, cf, cif), (gn, cn, cin) = out["fused"], out["nccl"]
    assert _rel(gf, gn) < 1e-5 and _rel(cf, cn) < 1e-4, (_rel(gf, gn), _rel(cf, cn))
    assert sorted(cif) == sorted(cin)
    for k in cif:
        assert _rel(cif[k], cin[k]) < 1e-4, k
    mean = sum(cif.values()) / 4.0
    assert _rel(cf, mean) < 1e-5, _rel(cf, mean)


@pytest.mark.multigpu
def test_fused_scaffold_collective_multi_gpu_matches_nccl_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    n = min(torch.cuda.device_count(), 8)
    port = 29500 + ((os.getpid() + 613) % 1000)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n),
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "mp_scaffold_check.py")]
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=root)
    tail = "\n".join(proc.stdout.splitlines()[-60:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
