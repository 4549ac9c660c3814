"""CPU / gloo worker for tests/test_lora.py (torchrun --nproc-per-node 2 tests/mp_lora_gloo.py).

Drives :class:`FederatedEngine` on a LoRA ``bert_tiny`` through the ``torch.distributed`` session on gloo, each rank
with a shard of its own size, and checks one round against each rank's trained adapters (captured at the end of its
local training):

* the frozen range is bit-for-bit what it was before the round, on both ranks;
* the trainable entries equal the host's sample-weighted mean of the trained values on both ranks;
* with ``freeze_a`` (FFA-LoRA) the merged product ``B A`` equals the mean of the clients' merged products;
* ranks whose frozen weights differ fail at construction, on every rank."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models.bert import LoraConfig, bert_tiny  # noqa: E402
from baton_b200.parallel.engine import FederatedEngine  # noqa: E402


def shard(rank):
    n = 16 + 16 * rank
    g = torch.Generator().manual_seed(100 + rank)
    X = torch.randint(0, 1024, (n, 32), generator=g)
    return X, X[:, 0] % 2


def main():
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    fails = []

    def expect(cond, msg):
        ok = torch.tensor([1 if cond else 0])
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if not int(ok):
            fails.append(msg)

    for freeze_a in (False, True):
        torch.manual_seed(7)
        eng = FederatedEngine(bert_tiny(2, lora=LoraConfig(8, 16, targets=("query", "value", "ffn_in"),
                                                           freeze_a=freeze_a)),
                              "cpu", backend="nccl", lr=0.05, batch_size=8, wire_dtype="fp32", optimizer="adamw")
        a = eng.arena
        lo, hi = a.frozen_range
        frozen0 = a.theta[lo:hi].clone()
        trained = {}
        run = eng.trainer.run

        def capture(*args, **kw):
            out = run(*args, **kw)
            trained["theta"] = a.theta[:lo].clone()
            trained["ab"] = {k: v.double() for k, v in eng.model.lora_state_dict().items()}
            return out
        eng.trainer.run = capture
        X, y = shard(rank)
        eng.run_round((X, y), n_epoch=2)
        n = torch.tensor([float(X.shape[0])])
        mine = trained["theta"] * n
        tot = n.clone()
        dist.all_reduce(mine)
        dist.all_reduce(tot)
        mean = mine / tot
        expect(torch.equal(a.theta[lo:hi], frozen0), "frozen range changed (freeze_a={})".format(freeze_a))
        expect(torch.allclose(a.theta[:lo], mean, rtol=1e-5, atol=1e-6),
               "trainable entries are not the sample-weighted mean (freeze_a={})".format(freeze_a))
        if freeze_a:
            sd = eng.model.lora_state_dict()
            for k in sd:
                if not k.endswith("lora_B.weight"):
                    continue
                ka = k.replace("lora_B", "lora_A")
                prod = trained["ab"][k] @ trained["ab"][ka] * float(n)
                dist.all_reduce(prod)
                merged = sd[k].double() @ sd[ka].double()
                expect(torch.allclose(merged, prod / float(tot), rtol=1e-5, atol=1e-7),
                       "FFA-LoRA: merged B A is not the mean of the clients' products ({})".format(k))
    # ranks that start from different base weights fail loudly, all of them
    torch.manual_seed(7)
    m = bert_tiny(2, lora=LoraConfig(8, 16))
    if rank == 1:
        with torch.no_grad():
            m.layers[0].ffn_out.weight[0, 0] += 1.0
    try:
        FederatedEngine(m, "cpu", backend="nccl", lr=0.05, batch_size=8)
        raised = False
    except ValueError as e:
        raised = "frozen parameters differ" in str(e)
    expect(raised, "differing frozen weights were not rejected")
    if rank == 0:
        print("RESULT", "PASS" if not fails else "FAIL " + "; ".join(fails))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
