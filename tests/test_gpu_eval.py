"""Evaluation of the global model on the GPU: the eval-mode BatchNorm epilogue of the convolution GEMMs, the fold
kernel, the forward-only classifier head, and ``FederatedEngine.evaluate`` on ResNet-18 / ResNet-50 against an fp32
CPU oracle."""
import math
import struct

import pytest
import torch
import torch.nn.functional as TF

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


@pytest.fixture(scope="module")
def F():
    from baton_b200.ops import functional as F
    F.load()
    return F


def _eps_bits(eps):
    return struct.unpack("<i", struct.pack("<f", eps))[0]


def _fold(F, gamma, beta, mean, var, eps=1e-5):
    """scale / shift of one BatchNorm through the fold kernel -> ([2C] table, scale, shift)"""
    c = gamma.numel()
    arena = torch.cat([gamma, beta, mean, var]).contiguous()
    desc = torch.tensor([[0, c, 2 * c, 3 * c, 0, c, _eps_bits(eps)]], dtype=torch.int64, device=gamma.device)
    out = torch.full((2 * c,), float("nan"), device=gamma.device)
    F.bn_fold_eval(arena, desc, out)
    return out, out[:c], out[c:]


# (cin, cout, k, stride, pad, h): the forward convolutions of ResNet-18 on 32x32 inputs, shortcuts included
RESNET18_CONVS = [(3, 64, 7, 2, 3, 32), (64, 64, 3, 1, 1, 8), (64, 128, 3, 2, 1, 8), (64, 128, 1, 2, 0, 8),
                  (128, 128, 3, 1, 1, 4), (128, 256, 3, 2, 1, 4), (128, 256, 1, 2, 0, 4), (256, 256, 3, 1, 1, 2),
                  (256, 512, 3, 2, 1, 2), (256, 512, 1, 2, 0, 2), (512, 512, 3, 1, 1, 1)]
# (force_bn, cluster): fixed-depth kernel at both tile widths, cluster split-K (the launcher shrinks the cluster where
# K is too short for it)
FAMILIES = [(64, 1), (128, 1), (64, 2), (128, 4)]


def _conv(F, x, wt, k, s, p, family, affine=None, out=None):
    """The GEMM ``_conv_bn_eval`` runs for this shape, with a forced kernel family."""
    n, h, w, c = x.shape
    cout = wt.shape[0]
    bn, ck = family
    sk = -ck if ck > 1 else 1
    if h == 1 and w == 1 and k % 2 == 1 and p == k // 2 and k > 1:
        return F.gemm(x.view(n, c), wt.view(cout, k * k, c)[:, (k // 2) * k + k // 2, :], affine=affine, out=out,
                      force_bn=bn, split_k=sk)
    if c % 64 == 0:
        return F.conv_igemm_fwd(x, wt, k, k, s, p, affine=affine, cluster_k=ck, force_bn=bn, out=out)
    return F.gemm(F.im2col(x, k, k, s, p)[0], wt, affine=affine, out=out, force_bn=bn, split_k=sk)


@pytest.mark.parametrize("n", [128, 37])
@pytest.mark.parametrize("cin,cout,k,stride,pad,h", RESNET18_CONVS)
def test_affine_epilogue_matches_gemm_then_bn_apply_and_fp32(F, cin, cout, k, stride, pad, h, n):
    dev = torch.device("cuda:0")
    torch.manual_seed(cin * 7 + cout + k + n)
    x = torch.randn(n, h, h, cin, device=dev).to(BF16)
    kt = k * k * cin
    w = (torch.randn(cout, kt, device=dev) * (2.0 / kt) ** 0.5).to(BF16)
    wt = F.pad_rows(w, F.round_up(kt, 8)) if kt % 8 else w
    gamma = torch.rand(cout, device=dev) + 0.5
    beta = torch.randn(cout, device=dev) * 0.2
    mean = torch.randn(cout, device=dev) * 0.3
    var = torch.rand(cout, device=dev) + 0.2
    table, scale, shift = _fold(F, gamma, beta, mean, var)
    ho = F.conv_out_size(h, k, stride, pad)
    M = n * ho * ho
    # fp32 reference of the convolution itself (bf16 operands, fp32 everything else)
    w4 = w.float().view(cout, k, k, cin).permute(0, 3, 1, 2)
    z32 = TF.conv2d(x.float().permute(0, 3, 1, 2), w4, stride=stride, padding=pad).permute(0, 2, 3, 1).reshape(M, cout)
    C = F.load()
    for relu, with_res in ((False, False), (True, False), (True, True), (False, True)):
        res = (torch.randn(M, cout, device=dev) * 0.5).to(BF16) if with_res else None
        af = F.affine_epilogue_args(table, 0, cout, relu, res)
        want32 = z32 * scale + shift + (res.float() if with_res else 0.0)
        want32 = want32.clamp_min(0.0) if relu else want32
        for family in FAMILIES:
            y = torch.full((M, cout), float("nan"), device=dev, dtype=BF16)
            got = _conv(F, x, wt, k, stride, pad, family, affine=af, out=y)
            assert got is not None, ("declined", family)
            # reference: the same GEMM without the epilogue, rounded to bf16, then bn_apply in eval mode
            z = _conv(F, x, wt, k, stride, pad, family)
            ref = torch.empty_like(z)
            sm = torch.empty(cout, device=dev)
            C.bn_apply(z, res, ref, torch.zeros(2 * cout, device=dev), gamma, beta, mean, var, sm, sm.clone(), None, M,
                       cout, 1e-5, 0.1, relu, False)
            torch.cuda.synchronize()
            assert not torch.isnan(y.float()).any(), ("unwritten output", family, relu, with_res)
            assert _rel(y, ref) < 1e-2, (family, relu, with_res, _rel(y, ref))
            assert _rel(y, want32) < 1e-2, (family, relu, with_res, _rel(y, want32))


def test_affine_epilogue_declines_what_it_cannot_do(F):
    dev = torch.device("cuda:0")
    a = torch.randn(256, 64, device=dev).to(BF16)
    b = torch.randn(64, 64, device=dev).to(BF16)
    table = torch.ones(128, device=dev)
    af = F.affine_epilogue_args(table, 0, 64, True)
    assert F.gemm(a, b, out_dtype=torch.float32, affine=af) is None                  # fp32 output
    assert F.gemm(a, b, bias=torch.zeros(64, device=dev), affine=af) is None         # bias
    assert F.gemm(a, b[:60], affine=F.affine_epilogue_args(table, 0, 60, True)) is None   # N % 8 != 0
    assert F.gemm(a, b, affine=af) is not None


def test_fold_kernel_matches_norm_formula_within_one_ulp(F):
    from baton_b200.models import resnet18
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.ops import nn as bnn
    from baton_b200.train import bn_fold_table
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    m = resnet18(10)
    arena = ParamArena(m, dev)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, bnn.BatchNorm2d):
                mod.weight.uniform_(-1.5, 1.5)
                mod.bias.normal_(0, 0.3)
                mod.running_mean.normal_(0, 0.5)
                mod.running_var.uniform_(0.01, 3.0)
    table, size = bn_fold_table(m, arena)
    out = torch.full((size,), float("nan"), device=dev)
    F.bn_fold_eval(arena.theta, table, out)
    torch.cuda.synchronize()
    for mod in m.modules():
        if not isinstance(mod, bnn.BatchNorm2d):
            continue
        c, o = mod.num_features, mod.eval_off
        rstd = torch.rsqrt(mod.running_var + mod.eps)
        g = mod.weight.detach()
        want_scale = g * rstd
        prod = mod.running_mean * g * rstd
        want_shift = mod.bias.detach() - prod
        got_scale, got_shift = out[o: o + c], out[o + c: o + 2 * c]
        ulps = (got_scale.view(torch.int32).long() - want_scale.view(torch.int32).long()).abs()
        assert int(ulps.max()) <= 1
        # shift: an FMA may fuse the product into the subtraction, which skips one rounding of the product and moves
        # the final one: at most two ulps of the larger term apart
        bound = torch.maximum(mod.bias.detach().abs(), prod.abs()) * 2.0 ** -21
        assert bool(((got_shift - want_shift).abs() <= bound).all())


@pytest.mark.parametrize("classes", [10, 32])
@pytest.mark.parametrize("rows", [128, 37])
def test_forward_only_head_matches_fp32(F, classes, rows):
    dev = torch.device("cuda:0")
    torch.manual_seed(classes + rows)
    x = torch.randn(rows, 512, device=dev).to(BF16)
    w = (torch.randn(classes, 512, device=dev) * 0.05).to(BF16)
    b = torch.randn(classes, device=dev) * 0.1
    t = torch.randint(0, classes, (rows,), device=dev)
    acc = torch.tensor([1.5, 2.0], device=dev)               # the kernel adds into it
    _, logits = F.linear_xent_eval(x, w, b, t, acc, want_logits=True)
    torch.cuda.synchronize()
    z = x.float() @ w.float().t() + b
    assert _rel(logits, z) < 1e-4
    want_loss = float(TF.cross_entropy(z, t, reduction="sum"))
    assert abs(float(acc[0]) - 1.5 - want_loss) <= 1e-4 * abs(want_loss) + 1e-4
    top2 = z.topk(2, dim=1).values
    close = int(((top2[:, 0] - top2[:, 1]) < 1e-3).sum())    # near-ties may go either way
    assert abs(float(acc[1]) - 2.0 - int((z.argmax(1) == t).sum())) <= close


# ------------------------------------------------------------------ whole model
def _engine(model_fn, batch, n_train, rounds, seed=0):
    from baton_b200.data import ShardSpec, image_shard
    from baton_b200.parallel.engine import FederatedEngine
    dev = torch.device("cuda:0")
    torch.manual_seed(seed)
    eng = FederatedEngine(model_fn(10), dev, backend="fused", lr=0.05, batch_size=batch)
    X, y = image_shard(ShardSpec(0, torch.full((10,), 0.1), n_train), noise=0.3, seed=seed, dtype=BF16)
    X, y = X.to(dev), y.to(dev)
    for _ in range(rounds):
        eng.run_round((X, y), n_epoch=2)
    return eng, (X, y)


def _holdout(n, seed=0, noise=0.3):
    from baton_b200.data import holdout_image_shard
    X, y = holdout_image_shard(10, n, noise=noise, seed=seed, dtype=BF16)
    return X.cuda(), y.cuda()


def _oracle(model_fn, model, X):
    """``model`` in fp32 on the CPU (TF.conv2d / TF.batch_norm in eval mode) -> logits"""
    ref = model_fn(10)
    ref.load_state_dict({k: v.detach().float().cpu() for k, v in model.state_dict().items()})
    ref.eval()
    with torch.no_grad():
        return ref(X.float().cpu())


def _fused_logits(eng, X, y, batch):
    """logits of the fused evaluation pass (head of the pass: fold + weights, then explicit_eval per batch)"""
    m, tr = eng.model, eng.trainer
    tr._eval_head()
    acc = torch.zeros(2, device=X.device)
    torch.nn.Module.train(m, False)
    parts = [m.explicit_eval(X[s: s + batch], y[s: s + batch], acc, want_logits=True) for s in range(0, X.shape[0], batch)]
    torch.nn.Module.train(m, True)
    return torch.cat(parts).cpu(), acc


def _check_against(z, ref, tol, what):
    rel_l2 = float((z - ref).norm() / ref.norm())
    agree = float((z.argmax(1) == ref.argmax(1)).float().mean())
    print("{}: logits rel. L2 {:.2e}, argmax agreement {:.4f}".format(what, rel_l2, agree))
    assert rel_l2 < tol, (what, rel_l2)
    assert agree >= 0.99, (what, agree)


# The held-out noise (0.8, against 0.3 in training) keeps the held-out loss away from zero, where a relative loss error
# says nothing and run-to-run differences of the (atomic, non-deterministic) training would dominate it, while most
# predictions stay clear of the near-ties a bf16 forward may break the other way.
@pytest.mark.parametrize("arch,batch,n_train,n_eval", [("resnet18", 128, 1024, 1000), ("resnet50", 16, 256, 400)])
def test_evaluate_matches_fp32_cpu_oracle_and_eager_path(arch, batch, n_train, n_eval):
    from baton_b200 import models
    model_fn = getattr(models, arch)
    eng, _ = _engine(model_fn, batch, n_train, rounds=2)
    Xe, ye = _holdout(n_eval, noise=0.8)
    res = eng.evaluate((Xe, ye), batch_size=batch)
    print("{}: held-out loss {:.4f} accuracy {:.4f}".format(arch, res.loss, res.accuracy))
    assert res.n_samples == n_eval and res.loss > 0.2, res
    ref = _oracle(model_fn, eng.model, Xe)
    ref_loss = float(TF.cross_entropy(ref, ye.cpu()))
    assert abs(res.loss - ref_loss) <= 1e-2 * abs(ref_loss), (res.loss, ref_loss)
    z, _ = _fused_logits(eng, Xe, ye, batch)
    _check_against(z, ref, 3e-2, arch + " fused vs fp32 CPU")
    # the eager CUDA eval path (GEMM, then bn_apply in eval mode)
    m = eng.model
    torch.nn.Module.train(m, False)
    with torch.no_grad():
        eager = torch.cat([m(Xe[s: s + batch]).float() for s in range(0, n_eval, batch)]).cpu()
    torch.nn.Module.train(m, True)
    _check_against(z, eager, 2e-2, arch + " fused vs eager CUDA")


def test_declined_epilogue_falls_back_to_gemm_then_bn_apply(monkeypatch):
    """Every GEMM declines the epilogue: ``_conv_bn_eval`` runs the plain GEMM and ``bn_apply`` in eval mode, and the
    pass computes what the fused one does."""
    from baton_b200.models import resnet18
    from baton_b200.ops import _ext
    from baton_b200.ops import functional as F
    eng, _ = _engine(resnet18, 128, 1024, rounds=2)
    Xe, ye = _holdout(1000, noise=0.8)                              # as in the oracle test: few near-ties
    eng.evaluate((Xe, ye), batch_size=128)                         # builds the fold table
    fused, acc_f = _fused_logits(eng, Xe, ye, 128)
    gemm, conv = F.gemm, F.conv_igemm_fwd

    def declining(fn):
        return lambda *a, **k: None if k.get("affine") is not None else fn(*a, **k)
    monkeypatch.setattr(F, "gemm", declining(gemm))
    monkeypatch.setattr(F, "conv_igemm_fwd", declining(conv))
    c0 = _ext.launch_counts()
    fallback, acc_b = _fused_logits(eng, Xe, ye, 128)
    counts = _ext.launch_counts() - c0
    assert counts["bn_apply"] == 20 * 8, counts                     # 20 BatchNorms, 8 batches
    _check_against(fallback, fused, 2e-2, "fallback vs fused")
    assert abs(float(acc_b[0]) - float(acc_f[0])) <= 1e-2 * abs(float(acc_f[0]))


def test_evaluate_changes_no_state_reuses_its_graph_and_folds_every_batchnorm():
    from baton_b200.models import resnet18
    eng, (X, y) = _engine(resnet18, 128, 512, rounds=2)
    eng.sync()
    a, tr = eng.arena, eng.trainer
    tr.loss_acc.fill_(0.25)
    snap = {"theta": a.theta.clone(), "grad": a.grad.clone(), "theta_bf16": a.theta_bf16.clone(),
            "int_arena": a.int_arena.clone(), "loss_acc": tr.loss_acc.clone()}
    if a.momentum is not None:
        snap["momentum"] = a.momentum.clone()
    Xe, ye = _holdout(700)                                     # 5 full batches + a ragged one of 60
    r1 = eng.evaluate((Xe, ye), batch_size=128)
    torch.cuda.synchronize()
    now = {"theta": a.theta, "grad": a.grad, "theta_bf16": a.theta_bf16, "int_arena": a.int_arena,
           "loss_acc": tr.loss_acc, "momentum": a.momentum}
    for k, v in snap.items():
        assert torch.equal(now[k], v), k
    # every BatchNorm ran in a GEMM epilogue: the captured pass has the fold and no BatchNorm kernel
    counts = tr.eval_launches
    assert counts["bn_fold_eval"] == 1 and counts["bn_apply"] == 0 and counts["bn_stats"] == 0, counts
    assert counts["linear_xent_eval"] == 6, counts
    assert counts["pad_rows"] == 1, counts                      # the stem's padded weights: once per pass
    captures = tr.eval_captures
    r2 = eng.evaluate((Xe, ye), batch_size=128)
    assert tr.eval_captures == captures                        # replayed, not captured again
    assert abs(r2.loss - r1.loss) <= 1e-5 * abs(r1.loss) and r2.accuracy == r1.accuracy   # loss: fp32 atomics
    # training goes on normally, and the replayed graph folds the NEW running statistics at its head
    tr.loss_acc.zero_()
    out = eng.run_round((X, y), n_epoch=1)
    assert len(out.loss_history) == 1 and math.isfinite(out.loss_history[0])
    r3 = eng.evaluate((Xe, ye), batch_size=128)
    assert tr.eval_captures == captures
    ref = _oracle(resnet18, eng.model, Xe)
    ref_loss = float(TF.cross_entropy(ref, ye.cpu()))
    assert abs(r3.loss - ref_loss) <= 1e-2 * abs(ref_loss), (r3.loss, ref_loss, r1.loss)
    # host shards are staged into evaluation buffers of their own
    staged = dict(eng._stage)
    r4 = eng.evaluate((Xe.cpu().pin_memory(), ye.cpu().pin_memory()), batch_size=128)
    assert set(eng._stage) == set(staged) and all(eng._stage[k] is staged[k] for k in staged)
    assert len(eng._eval_stage) == 1
    # the graph cache is bounded: fresh device tensors every call do not pile up captured passes
    fresh = [(Xe[:64].clone(), ye[:64].clone()) for _ in range(tr.EVAL_GRAPHS_MAX + 2)]   # live: distinct addresses
    for pair in fresh:
        eng.evaluate(pair, batch_size=32)
    assert len(tr._eval_graphs) == tr.EVAL_GRAPHS_MAX
    assert abs(r4.loss - r3.loss) <= 1e-5 * abs(r3.loss) and r4.accuracy == r3.accuracy


def test_held_out_accuracy_shows_learning():
    from baton_b200.models import resnet18
    eng, _ = _engine(resnet18, 128, 1024, rounds=3)
    res = eng.evaluate(_holdout(1000), batch_size=512)
    assert res.accuracy > 0.5, res                             # chance is 0.1
    assert res.local_accuracy == res.accuracy and res.n_samples == 1000
