"""Model tier on the GPU: ResNet-18 on the sm_90a layers against the stock fp32
PyTorch model with the same weights; CUDA-graphed local SGD trains."""
import pytest
import torch

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


def _randomize_bn(m):
    with torch.no_grad():
        for mod in m.modules():
            if hasattr(mod, "running_mean") and hasattr(mod, "weight"):
                mod.weight.uniform_(0.5, 1.5)
                mod.bias.uniform_(-0.2, 0.2)


def test_resnet18_forward_backward_matches_stock_model():
    import torchvision
    from baton_b200.models import resnet18
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    m = resnet18(10)
    _randomize_bn(m)
    tv = torchvision.models.resnet18(num_classes=10)
    tv.load_state_dict(m.state_dict())
    tv = tv.to(dev).train()
    arena = ParamArena(m, dev)
    m.build_workspace(dev)
    m.train()
    x = torch.randn(64, 32, 32, 3, device=dev)
    y = torch.randint(0, 10, (64,), device=dev)
    logits = m(x.to(BF16))
    ref = tv(x.to(BF16).float().permute(0, 3, 1, 2))
    assert logits.dtype == torch.float32
    assert _rel(logits, ref) < 6e-2, _rel(logits, ref)
    from baton_b200.ops import nn as bnn
    loss, _ = bnn.cross_entropy(logits, y)
    loss.backward()
    torch.nn.functional.cross_entropy(ref, y).backward()
    sd_ref = dict(tv.named_parameters())
    fp32_grads = {n: p.grad.clone() for n, p in sd_ref.items()}
    # calibration: the SAME stock model under bf16 autocast vs its own fp32 gradients tells how much
    # of the deviation is just bf16 arithmetic through 18 layers (batch 64, 1x1 final feature maps)
    tv.zero_grad()
    with torch.autocast("cuda", dtype=BF16):
        torch.nn.functional.cross_entropy(tv(x.to(BF16).float().permute(0, 3, 1, 2)).float(), y).backward()
    cos = torch.nn.functional.cosine_similarity
    mine, stock = {}, {}
    for name, p in m.named_parameters():
        mine[name] = float(cos(p.grad.float().flatten(), fp32_grads[name].flatten(), dim=0))
        stock[name] = float(cos(sd_ref[name].grad.float().flatten(), fp32_grads[name].flatten(), dim=0))
    worst = min(mine, key=mine.get)
    mean_mine = sum(mine.values()) / len(mine)
    mean_stock = sum(stock.values()) / len(stock)
    print("grad cosine vs fp32: ours mean {:.4f} min {:.4f} ({}), stock-autocast mean {:.4f} min {:.4f}".format(
        mean_mine, mine[worst], worst, mean_stock, min(stock.values())))
    # the hand-written bf16 path must be as close to fp32 as stock bf16 autocast is
    assert mean_mine > 0.93 and mean_mine > mean_stock - 0.02, (mean_mine, mean_stock)
    assert mine[worst] > min(stock.values()) - 0.06, (worst, mine[worst], stock[worst])
    # state_dict stays loadable by the stock model after adoption + a step
    tv.load_state_dict(m.state_dict())


def test_graphed_local_sgd_learns_and_matches_eager():
    from baton_b200.data import ShardSpec, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.train import GraphedLocalSGD
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    spec = ShardSpec(0, torch.full((10,), 0.1), 1024)
    X, y = image_shard(spec, noise=0.3)
    X, y = X.to(dev).to(BF16), y.to(dev)
    m = resnet18(10)
    arena = ParamArena(m, dev, momentum=True)
    m.build_workspace(dev)
    tr = GraphedLocalSGD(m, arena, loss="ce")
    m._graphed_trainer = tr
    hist = m.train(X, y, n_epoch=6, lr=0.05, batch_size=128, momentum=0.9)
    assert len(hist) == 6 and hist[-1] < hist[0] * 0.7, hist
    assert tr.last_stats["accuracy"][-1] > 0.5
    # second call reuses the captured graph
    n_graphs = len(tr._graphs)
    m.train(X, y, n_epoch=1, lr=0.05, batch_size=128, momentum=0.9)
    assert len(tr._graphs) == n_graphs
    assert int(m.bn1.num_batches_tracked) == 7 * 8
    # bf16 shadow is in sync with the fp32 master after training
    assert torch.equal(arena.theta_bf16[: arena.n_param], arena.theta[: arena.n_param].to(BF16))


@pytest.mark.parametrize("arch,randomize", [("resnet18", False), ("resnet18", True), ("resnet50", True)])
def test_explicit_step_matches_autograd_path(arch, randomize):
    """The hand-scheduled step (``ResNet.explicit_step``: no autograd engine, two-piece block gradients summed inside
    the BatchNorm-backward kernel, shortcut branch on a side stream) must produce the gradients ``loss.backward()``
    produces on the same weights and batch.  The BatchNorm statistics are accumulated with fp32 atomics, so two
    identical runs of the SAME path already differ once the bf16 roundings flip; the comparison is therefore
    calibrated against autograd-vs-autograd.  With the default init (last BatchNorm gamma of every block = 0) the main
    branch is silent and the match is tight; with randomised BatchNorm parameters every branch matters."""
    from baton_b200 import models
    from baton_b200.ops import nn as bnn
    from baton_b200.parallel.arena import ParamArena
    dev = torch.device("cuda:0")
    torch.manual_seed(11)
    x = torch.randn(128, 32, 32, 3, device=dev).to(BF16)
    y = torch.randint(0, 10, (128,), device=dev)

    def run(explicit):
        torch.manual_seed(3)
        m = getattr(models, arch)(10)
        if randomize:
            _randomize_bn(m)
        arena = ParamArena(m, dev)
        m.build_workspace(dev)
        m.train()
        if explicit:
            stats = m.explicit_step(x, y)
        else:
            logits = m(x)
            loss, stats = bnn.cross_entropy(logits, y)
            loss.backward()
            bnn.WGRAD.join()
        torch.cuda.synchronize()
        return stats.clone(), arena.grad.clone(), torch.cat([b.float().flatten() for b in m.buffers()])

    a, b, c = run(False), run(False), run(True)
    cos = torch.nn.functional.cosine_similarity
    noise = 1.0 - float(cos(a[1], b[1], dim=0))              # autograd vs autograd
    diff = 1.0 - float(cos(a[1], c[1], dim=0))               # autograd vs hand-scheduled
    print("grad 1-cos: autograd/autograd {:.2e}, autograd/explicit {:.2e}".format(noise, diff))
    assert diff <= 2.0 * noise + 1e-4, (diff, noise)
    dl_noise, dl = float((a[0][0] - b[0][0]).abs()), float((a[0][0] - c[0][0]).abs())
    assert dl <= 3.0 * dl_noise + 2e-3 * float(a[0][0].abs()), (dl, dl_noise)
    db_noise, db = _rel(b[2], a[2]), _rel(c[2], a[2])
    assert db <= 3.0 * db_noise + 1e-3, (db, db_noise)       # running statistics / step counters advanced alike
