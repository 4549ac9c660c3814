"""Secure aggregation on the CPU (``parallel/secagg.py``): the RFC vectors of X25519, HKDF and ChaCha20, the encode rules,
mask cancellation over simulated parties, the uniformity of masked uploads, the ``NcclSession`` secure round against
the host reference and the plain mean, the feature rules at every entry point, and a 2..4-process gloo run
(``tests/mp_secagg_gloo.py``)."""
import os
import struct

import numpy as np
import pytest
import torch

from baton_b200.parallel import secagg as sa
from baton_b200.parallel.features import check_features, peer_loads_only
from baton_b200.parallel.secagg import SecAggConfig

H = bytes.fromhex
RFC_KEY = list(struct.unpack("<8I", bytes(range(32))))


# ---------------------------------------------------------------- RFC vectors
def test_x25519_rfc7748_5_2():
    k = H("a546e36bf0527c9d3b16154b82465edd62144c0ac1fc5a18506a2244ba449ac4")
    u = H("e6db6867583030db3594c1a424b15f7c726624ec26b3353b10a903a6d0ab1c4c")
    assert sa.x25519(k, u) == H("c3da55379de9c6908e94ea4df28d084f32eccf03491c71f754b4075577a28552")


def test_x25519_rfc7748_6_1():
    a = H("77076d0a7318a57d3c16c17251b26645df4c2f87ebc0992ab177fba51db92c2a")
    b = H("5dab087e624a8a4b79e17f8b83800ee66f3bb1292618b6fd1c2f8b27ff88e0eb")
    pa, pb = sa.x25519(a, sa.X25519_BASE), sa.x25519(b, sa.X25519_BASE)
    assert pa == H("8520f0098930a754748b7ddcb43ef75a0dbf3a0d26381af4eba4a98eaa9b4e6a")
    assert pb == H("de9edb7d7b7dc1b4d35b61c2ece435373f8343c85b78674dadfc7e146f882b4f")
    shared = H("4a5d9d5ba4ce2de1728e3bf480350f25e07e21c947d19e3376f09b3c1e161742")
    assert sa.x25519(a, pb) == shared and sa.x25519(b, pa) == shared


def test_hkdf_rfc5869_case1():
    okm = sa.hkdf_sha256(bytes([0x0B]) * 22, bytes(range(13)), bytes(range(0xF0, 0xFA)), 42)
    assert okm == H("3cb25f25faacd57a90434f64d0362f2a2d2d0a90cf1a5a4c5db02d56ecc4c5bf34007208d5b887185865")


def test_chacha20_rfc8439_2_3_2():
    ks = sa.keystream(RFC_KEY, [0x09000000, 0x4A000000, 0], 16, counter0=1)
    assert ks.tobytes() == H("10f1e7e4d13b5915500fdd1fa32071c4c7d1f4c733c068030422aa9ac3d46c4e"
                             "d2826446079faa0914c2d705d98b02a2b5129cd1de164eb9cbd083e8a2503c4e")


SUNSCREEN = (b"Ladies and Gentlemen of the class of '99: If I could offer you only one tip for the future, "
             b"sunscreen would be it.")
SUNSCREEN_CT = H("6e2e359a2568f98041ba0728dd0d6981e97e7aec1d4360c20a27afccfd9fae0bf91b65c5524733ab8f593dabcd62b357"
                 "1639d624e65152ab8f530c359f0861d807ca0dbf500d6a6156a38e088a22b65e52bc514d16ccf806818ce91ab7793736"
                 "5af90bbf74a35be6b40b8eedf2785e42874d")


def test_chacha20_rfc8439_2_4_2():
    ks = sa.keystream(RFC_KEY, [0, 0x4A000000, 0], 30, counter0=1).tobytes()
    assert bytes(p ^ k for p, k in zip(SUNSCREEN, ks)) == SUNSCREEN_CT


def test_all_zero_shared_secret_rejected():
    sk = bytes(range(32))
    with pytest.raises(ValueError, match="all-zero"):
        sa.pair_key(sk, bytes(32), 0, 1, [bytes(32), bytes(32)])     # the u = 0 point of small order


def test_pair_key_symmetric():
    sk = [bytes([i + 1]) * 32 for i in range(3)]
    pk = [sa.x25519(s, sa.X25519_BASE) for s in sk]
    for i in range(3):
        for j in range(3):
            if i != j:
                assert sa.pair_key(sk[i], pk[j], i, j, pk) == sa.pair_key(sk[j], pk[i], j, i, pk)
    assert sa.pair_key(sk[0], pk[1], 0, 1, pk) != sa.pair_key(sk[0], pk[2], 0, 2, pk)


# ---------------------------------------------------------------- encode rules
def test_frac_bits_from_range():
    assert SecAggConfig().frac_bits == 24
    for R, f in ((1.0, 30), (1.5, 29), (2.0, 29), (64.0, 24), (65.0, 23), (2.0 ** -20, 50), (2.0 ** 20, 10)):
        assert sa.frac_bits(R) == f, R
        assert R * 2.0 ** f <= 2.0 ** 30 < 2 * R * 2.0 ** f


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -1.0, 0.0, 2.0 ** 21, 1e-9, "64", True])
def test_range_rejected(bad):
    with pytest.raises(ValueError):
        SecAggConfig(bad)


def test_encode_clamp_nonfinite_saturation():
    R, f = 2.0, sa.frac_bits(2.0)
    x = np.array([0.5, -3.0, 3.0, np.nan, np.inf, -np.inf, 2.0, -2.0], dtype=np.float32)
    q, sat = sa.encode(x, 1.0, R, f)
    scale = 2.0 ** f
    assert q.tolist() == [int(0.5 * scale), int(-2 * scale), int(2 * scale), 0, int(2 * scale), int(-2 * scale),
                          int(2 * scale), int(-2 * scale)]
    assert sat == 5          # -3, 3, nan, +inf, -inf; exactly +-R is not clamped


def test_encode_round_half_even():
    f = 24
    ulp = np.float32(2.0 ** -f)
    x = np.array([0.5, 1.5, 2.5, -0.5, -1.5, 3.5], dtype=np.float32) * ulp
    q, _ = sa.encode(x, 1.0, 64.0, f)
    assert q.tolist() == [0, 2, 2, 0, -2, 4]


def test_encode_weight_rounded_once():
    rng = np.random.default_rng(0)
    x = rng.standard_normal(4096).astype(np.float32)
    w = np.float32(3.0) * (np.float32(1.0) / np.float32(7.0))
    q, _ = sa.encode(x, float(w), 64.0, 24)
    p = (w * x).astype(np.float32)
    assert np.array_equal(q, np.rint(p.astype(np.float64) * 2.0 ** 24).astype(np.int32))


def test_weights_fp32_in_order():
    w, N = sa.weights([3.0, 0.0, 5.0, 7.0])
    assert N == 15.0
    inv = np.float32(1.0) / np.float32(15.0)
    assert w.tolist() == [float(np.float32(3.0) * inv), 0.0, float(np.float32(5.0) * inv), float(np.float32(7.0) * inv)]
    assert sa.weights([0.0, 0.0])[0].tolist() == [0.0, 0.0]


# ---------------------------------------------------------------- masks
def _pair_keys(P, seed):
    rng = np.random.default_rng(seed)
    return {(i, j): [int(x) for x in rng.integers(0, 2 ** 32, 8, dtype=np.uint64)]
            for i in range(P) for j in range(i + 1, P)}


@pytest.mark.parametrize("P", range(2, 9))
def test_masks_cancel(P):
    rng = np.random.default_rng(P)
    n = 1000 + 7 * P
    counts = [float(rng.integers(1, 50)) if k % 3 != 1 else 0.0 for k in range(P)]   # some non-participants
    counts[0] = 11.0
    keys = _pair_keys(P, 100 + P)
    xs = [rng.standard_normal(n).astype(np.float32) * 0.1 for _ in range(P)]
    w, _ = sa.weights(counts)
    parts = [k for k in range(P) if counts[k] > 0]
    f = 24
    plain = np.zeros(n, dtype=np.int64)
    masked = np.zeros(n, dtype=np.uint32)
    for k in parts:
        q, _ = sa.encode(xs[k], float(w[k]), 64.0, f)
        plain += q
        mine = {j: keys[(min(j, k), max(j, k))] for j in parts if j != k}
        u = sa.mask(q, sa.peer_list(k, parts, mine), [77, 0, 0])
        assert not np.array_equal(u, q.view(np.uint32)) or len(parts) == 1
        masked = masked + u
    assert np.array_equal(masked.view(np.int32).astype(np.int64), plain)
    d, _ = sa.reference_round(xs, counts, 64.0, keys, [77, 0, 0])
    assert np.array_equal(d, (plain.astype(np.int32).astype(np.float32) * np.float32(2.0 ** -f)))


def _chi2_bytes(u):
    counts = np.bincount(np.asarray(u).view(np.uint8), minlength=256)
    exp = counts.sum() / 256.0
    return float(((counts - exp) ** 2 / exp).sum())


@pytest.mark.parametrize("scale", [0.0, 30.0])
def test_masked_upload_is_byte_uniform(scale):
    from scipy.stats import chi2
    n = 1 << 16
    x = (np.random.default_rng(5).standard_normal(n) * scale).astype(np.float32)
    q, _ = sa.encode(x, 1.0, 64.0, 24)
    raw = _chi2_bytes(q)
    u = sa.mask(q, [(_pair_keys(2, 9)[(0, 1)], 1)], [3, 0, 0])
    stat = _chi2_bytes(u)
    assert stat < chi2.ppf(0.999, 255), stat
    assert raw > chi2.ppf(0.999, 255)        # the unmasked encoding is far from uniform


# ---------------------------------------------------------------- NcclSession (world 1, gloo-free)
def _arena(seed=0):
    from baton_b200.models import MLP2
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(seed)
    return ParamArena(MLP2(10, 16, 3), torch.device("cpu"))


def test_nccl_session_secure_round_matches_reference_and_mean():
    from baton_b200.parallel.fedavg import NcclSession
    arena = _arena()
    cfg = SecAggConfig(8.0)
    sess = NcclSession(arena, wire_dtype="fp32", secagg=cfg)
    x0 = arena.global_w.clone()
    delta = torch.randn(arena.n, generator=torch.Generator().manual_seed(1)) * 0.05
    delta[3] = 100.0
    arena.theta.copy_(x0 + delta)
    sess.aggregate(my_n=7.0)
    src = ((x0 + delta) - x0).numpy()
    d, sat = sa.reference_round([src], [7.0], cfg.range, {}, [0, 0, 0])
    expect = (x0.numpy() + d).astype(np.float32)
    assert np.array_equal(arena.global_w.numpy().view(np.int32), expect.view(np.int32))
    assert torch.equal(arena.theta, arena.global_w)
    assert sess.last_secagg_saturation() == sat == 1
    f = cfg.frac_bits
    ok = np.abs(d - np.clip(src, -8, 8)) <= 2.0 ** -(f + 1) + 1e-7 * np.abs(src)
    assert ok.all()


def test_nccl_session_secure_round_server_opt():
    from baton_b200.parallel.fedavg import NcclSession
    from baton_b200.parallel.server_opt import ServerOptConfig, apply_update_
    arena = _arena(1)
    so = ServerOptConfig("adam", lr=0.01)
    sess = NcclSession(arena, wire_dtype="fp32", secagg=SecAggConfig(), server_opt=so)
    x = arena.global_w.clone()
    m, v = so.init_state(arena.n_param, "cpu")
    for rnd in range(2):
        delta = torch.randn(arena.n, generator=torch.Generator().manual_seed(10 + rnd)) * 0.01
        arena.theta.copy_(arena.global_w + delta)
        src = (arena.theta - arena.global_w).numpy()
        d, _ = sa.reference_round([src], [4.0], 64.0, {}, [0, 0, 0])
        sess.aggregate(my_n=4.0)
        apply_update_(x, torch.from_numpy(d), arena.n_param, m, v, so)
        assert torch.equal(arena.global_w.view(torch.int32), x.view(torch.int32)), rnd
        sm, sv = sess.server_state()
        assert torch.equal(sm, m) and torch.equal(sv, v)


def test_engine_secure_round_cpu_logical_clients_and_sampling():
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    model = MLP2(12, 16, 3)
    eng = FederatedEngine(model, "cpu", backend="nccl", wire_dtype="fp32", secure_agg=True, logical_clients=4,
                          sample_k=3, lr=0.1, batch_size=16, server_opt="avgm", server_lr=1.0)
    shards = {c: (torch.randn(32, 12, generator=torch.Generator().manual_seed(c)),
                  torch.randint(0, 3, (32,), generator=torch.Generator().manual_seed(50 + c))) for c in range(4)}
    before = eng.arena.global_w.clone()
    res = eng.run_round(lambda c: shards[c], n_epoch=1)
    assert len(res.participants) == 3
    assert not torch.equal(before, eng.arena.global_w)
    assert eng.last_secagg_saturation() == 0


# ---------------------------------------------------------------- feature rules
RULES = [
    (dict(wire_dtype="bf16"), "wire_dtype='fp32'"),
    (dict(wire_dtype="fp8"), "wire_dtype='fp32'"),
    (dict(wire_dtype="fp32", mode="weights"), "mode='delta'"),
    (dict(wire_dtype="fp32", dp=True), "DP-FedAvg"),
    (dict(wire_dtype="fp32", robust=True), "robust aggregator or Krum"),
    (dict(wire_dtype="fp32", topk=True), "top-k"),
    (dict(wire_dtype="fp32", scaffold=True), "SCAFFOLD"),
    (dict(wire_dtype="fp32", local=True), "client-local"),
    (dict(wire_dtype="fp32", tile_flags=True), "tile_flags"),
    (dict(wire_dtype="fp32", plane="http"), "SPMD engine"),
    (dict(wire_dtype="fp32", plane="seated"), "SPMD engine"),
]


@pytest.mark.parametrize("kw,reason", RULES)
def test_rules_check_features(kw, reason):
    with pytest.raises(ValueError, match=reason.replace("(", r"\(").replace(")", r"\)")):
        check_features(secure_agg=True, **kw)


@pytest.mark.parametrize("kw", [dict(server_opt=True), dict(prox_mu=0.1), dict(optimizer="adamw"),
                                dict(momentum=0.9)])
def test_rules_combine(kw):
    check_features(secure_agg=True, wire_dtype="fp32", **kw)


def test_peer_loads_only():
    assert peer_loads_only(wire_dtype="fp32", secure_agg=True)
    assert not peer_loads_only(wire_dtype="fp32")


ENGINE_RULES = [
    (dict(wire_dtype="bf16"), "wire_dtype='fp32'"),
    (dict(mode="weights"), "mode='delta'"),
    (dict(dp_clip=1.0), "DP-FedAvg"),
    (dict(aggregator="median"), "robust aggregator"),
    (dict(compress="topk"), "top-k"),
    (dict(scaffold=True), "SCAFFOLD"),
    (dict(local_keys="head"), "client-local"),
    (dict(tile_flags=True), "tile_flags"),
]


@pytest.mark.parametrize("kw,reason", ENGINE_RULES)
def test_rules_engine(kw, reason):
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
    args = dict(wire_dtype="fp32", backend="nccl")
    args.update(kw)
    with pytest.raises(ValueError, match=reason.replace("(", r"\(").replace(")", r"\)")):
        FederatedEngine(MLP2(8, 8, 3), "cpu", secure_agg=True, **args)


def test_rules_engine_range_and_type():
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
    with pytest.raises(ValueError):
        FederatedEngine(MLP2(8, 8, 3), "cpu", backend="nccl", wire_dtype="fp32", secure_agg=True,
                        secagg_range=float("inf"))
    with pytest.raises(TypeError):
        FederatedEngine(MLP2(8, 8, 3), "cpu", backend="nccl", wire_dtype="fp32", secure_agg=1)


@pytest.mark.parametrize("kw,reason", [(dict(wire_dtype="bf16"), "wire_dtype='fp32'"),
                                       (dict(wire_dtype="fp32", mode="weights"), "mode='delta'"),
                                       (dict(wire_dtype="fp32", scaffold=True), "SCAFFOLD")])
def test_rules_session(kw, reason):
    from baton_b200.parallel.fedavg import NcclSession
    with pytest.raises(ValueError, match=reason.replace("(", r"\(").replace(")", r"\)")):
        NcclSession(_arena(), secagg=SecAggConfig(), **kw)


def test_rules_session_round_override():
    from baton_b200.parallel.dp import DPConfig
    from baton_b200.parallel.fedavg import NcclSession
    from baton_b200.parallel.robust import RobustConfig
    sess = NcclSession(_arena(), wire_dtype="fp32", secagg=SecAggConfig())
    with pytest.raises(ValueError, match="DP-FedAvg"):
        sess.aggregate(my_n=1.0, dp=DPConfig(1.0, 0.0, seed=1))
    with pytest.raises(ValueError, match="robust"):
        sess.aggregate(my_n=1.0, robust=RobustConfig("median"))
    with pytest.raises(TypeError):
        NcclSession(_arena(), wire_dtype="fp32", secagg=64.0)


# ---------------------------------------------------------------- multi-process (gloo)
@pytest.mark.slow
@pytest.mark.parametrize("nproc", [2, 3, 4])
def test_gloo_secure_rounds(nproc):
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29400 + ((os.getpid() + 977 + 13 * nproc) % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "mp_secagg_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=root,
                          env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
