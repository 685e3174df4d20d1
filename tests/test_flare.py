"""FLARE aggregation (``--aggr flare``) on CPU: options and the banner, the MMD statement (identical sets, symmetry, permutations, a
two-Gaussian closed form, non-finite features, the sigma^2 <= 0 fallback, |F| in {0, 1, 2}), ``flare_weights`` against brute force, the
feature tap of every zoo model, the in-process step against a loop over the statement and the avg oracle, engine runs (log fields,
resume) and 2-rank gloo runs on both transports against one process."""
import json
import math
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.aggregation import Aggregation
from rlr_b200.engine import FLEngine
from rlr_b200.options import MODELS, make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- options ------------------------------------------------------------------------------------------------------------
def test_defaults():
    a = make_args(aggr="flare")
    assert a.root_size == 100 and a.flare_k is None and a.flare_tau == 1.0
    b = make_args(aggr="flare", root_size=7, flare_k=3, flare_tau=0.5)
    assert (b.root_size, b.flare_k, b.flare_tau) == (7, 3, 0.5)
    assert make_args().flare_k is None and make_args().flare_tau is None
    assert make_args(aggr="flare", server_clip=True, clip=1.0, noise=0.1).server_clip     # composes with server clipping and noise


@pytest.mark.parametrize("kw", [
    dict(aggr="avg", flare_k=2),
    dict(aggr="fltrust", flare_tau=1.0),
    dict(aggr="flare", flare_k=0),
    dict(aggr="flare", flare_k=-1),
    dict(aggr="flare", flare_k=1.5),
    dict(aggr="flare", flare_tau=0.0),
    dict(aggr="flare", flare_tau=-1.0),
    dict(aggr="flare", flare_tau=float("inf")),
    dict(aggr="flare", flare_tau=float("nan")),
    dict(aggr="flare", root_size=0),
    dict(aggr="rfa", root_size=10),
])
def test_flare_options_rejected(kw):
    with pytest.raises(ValueError):
        make_args(**kw)


def test_banner_line(capsys):
    from rlr_b200.options import print_exp_details
    print_exp_details(make_args())
    assert "FLARE" not in capsys.readouterr().out
    print_exp_details(make_args(aggr="flare", root_size=64, flare_k=3, flare_tau=2.0))
    out = capsys.readouterr().out
    assert "FLARE (root / k / tau): 64 / 3 / 2.0" in out and "Aggregation Function: flare" in out
    print_exp_details(make_args(aggr="flare"))
    assert "FLARE (root / k / tau): 100 / floor(|F|/2) / 1.0" in capsys.readouterr().out


# ---- the statement ------------------------------------------------------------------------------------------------------
def _brute_S(Z, s2):
    """S_ij by explicit loops over sample pairs, fp64 numpy."""
    Z = np.asarray(Z, dtype=np.float64)
    K = Z.shape[0]
    S = np.zeros((K, K))
    for i in range(K):
        for j in range(K):
            S[i, j] = sum(math.exp(-float(((a - b) ** 2).sum()) / s2) for a in Z[i] for b in Z[j])
    return S


def _brute_s2(Z):
    X = np.asarray(Z, dtype=np.float64).reshape(-1, Z.shape[-1])
    N = X.shape[0]
    return sum(float(((X[a] - X[b]) ** 2).sum()) for a in range(N) for b in range(N) if a != b) / (N * (N - 1))


def test_sigma2_and_sums_match_brute_force():
    gen = torch.Generator().manual_seed(1)
    Z = torch.randn(3, 5, 4, generator=gen)
    s2 = ops.flare_sigma2(Z, [0, 1, 2])
    assert abs(s2 - _brute_s2(Z.numpy())) < 1e-12 * s2
    np.testing.assert_allclose(ops.flare_sums_statement(Z, [True] * 3, s2), _brute_S(Z.numpy(), s2), rtol=1e-12)


def test_mmd_zero_for_identical_sets_symmetric_and_permutation_invariant():
    gen = torch.Generator().manual_seed(2)
    Z = torch.randn(5, 6, 8, generator=gen)
    Z[3] = Z[1]
    res = ops.flare_statement(Z)
    M = res.M
    assert M[1, 3] == 0.0 and M[3, 1] == 0.0
    assert np.array_equal(M, M.T) and np.array_equal(np.diag(M), np.zeros(5)) and (M >= 0).all()
    perm = [4, 2, 0, 3, 1]
    Mp = ops.flare_statement(Z[perm]).M
    np.testing.assert_allclose(Mp, M[np.ix_(perm, perm)], rtol=1e-12, atol=1e-15)
    # the samples' order within a set does not matter either
    Z2 = Z.clone()
    Z2[0] = Z[0][torch.randperm(6, generator=gen)]
    np.testing.assert_allclose(ops.flare_statement(Z2).M, M, rtol=1e-12, atol=1e-15)


def test_two_gaussian_closed_form():
    """Two sets of n samples with the Gaussian kernel and sigma^2 fixed: for point sets {a} and {b} (n copies each) the biased MMD is
    2 - 2 exp(-||a - b||^2 / sigma^2); for sets of two points each it is the closed form of the three kernel averages."""
    a, b = np.array([0.0, 1.0]), np.array([2.0, -1.0])
    Z = torch.tensor(np.stack([np.tile(a, (3, 1)), np.tile(b, (3, 1))]), dtype=torch.float32)
    s2 = 2.5
    M = ops.flare_mmd_matrix(ops.flare_sums_statement(Z, [True, True], s2), [0, 1], 3)
    assert abs(M[0, 1] - (2.0 - 2.0 * math.exp(-8.0 / s2))) < 1e-14
    x, y = np.array([[0.0], [1.0]]), np.array([[3.0], [5.0]])
    k = lambda u, v: math.exp(-(u - v) ** 2 / s2)
    kxx = sum(k(p, q) for p in x[:, 0] for q in x[:, 0]) / 4
    kyy = sum(k(p, q) for p in y[:, 0] for q in y[:, 0]) / 4
    kxy = sum(k(p, q) for p in x[:, 0] for q in y[:, 0]) / 4
    Z = torch.tensor(np.stack([x, y]), dtype=torch.float32)
    M = ops.flare_mmd_matrix(ops.flare_sums_statement(Z, [True, True], s2), [0, 1], 2)
    assert abs(M[0, 1] - (kxx + kyy - 2 * kxy)) < 1e-14


def test_non_finite_candidates_are_excluded():
    gen = torch.Generator().manual_seed(3)
    Z = torch.randn(6, 4, 8, generator=gen)
    Z[2, 1, 3] = float("nan")
    Z[4, 0, 0] = float("inf")
    res = ops.flare_statement(Z)
    assert res.members == [0, 1, 3, 5] and res.weights[2] == 0 and res.weights[4] == 0
    assert abs(res.weights.sum() - 1.0) < 1e-15
    clean = ops.flare_statement(Z[[0, 1, 3, 5]])
    assert np.array_equal(clean.M, res.M) and np.array_equal(clean.weights, res.weights[[0, 1, 3, 5]])
    assert clean.sigma2 == res.sigma2                                  # the bandwidth pools F only


def test_special_cases():
    gen = torch.Generator().manual_seed(4)
    Z = torch.randn(3, 4, 8, generator=gen)
    nan = torch.full_like(Z[0], float("nan"))
    none = ops.flare_statement(torch.stack([nan, nan]))               # |F| = 0
    assert none.members == [] and np.array_equal(none.weights, np.zeros(2))
    one = ops.flare_statement(torch.stack([nan, Z[0], nan]))           # |F| = 1: weight 1, no MMD pass
    assert one.members == [1] and one.weights.tolist() == [0.0, 1.0, 0.0] and one.M is None
    flat = ops.flare_statement(torch.ones(4, 3, 8))                    # every pooled feature equal: sigma^2 = 0
    assert flat.sigma2 == 0.0 and flat.M is None and flat.weights.tolist() == [0.25] * 4
    two = ops.flare_statement(Z[:2])                                   # |F| = 2: k = 1, each the other's neighbour
    assert two.counts.tolist() == [1, 1] and two.weights.tolist() == [0.5, 0.5]
    called = []
    ops.flare(torch.stack([Z[0], nan]), sums=lambda *a: called.append(1))
    ops.flare(torch.ones(3, 2, 4), sums=lambda *a: called.append(1))
    assert not called                                                  # neither special case launches the MMD pass


# ---- the host half --------------------------------------------------------------------------------------------------------
def _brute_weights(M, ids, k, tau):
    F = len(ids)
    k = min(F // 2 if k is None else k, F - 1)
    c = [0] * F
    for i in range(F):
        for j in range(F):
            if j == i:
                continue
            # j is among i's k nearest iff fewer than k others come before it (smaller M, or equal M at a lower position)
            before = sum(1 for l in range(F) if l not in (i, j) and (M[i][l] < M[i][j] or (M[i][l] == M[i][j] and ids[l] < ids[j])))
            c[j] += before < k
    mx = max(c)
    e = [math.exp((x - mx) / tau) for x in c]
    return [x / sum(e) for x in e], c


@pytest.mark.parametrize("F,k,tau,ties", [(2, None, 1.0, False), (5, None, 1.0, False), (7, 2, 0.5, True), (9, 8, 3.0, True),
                                          (12, None, 1.0, True), (12, 20, 1.0, False), (16, 1, 0.1, True)])
def test_flare_weights_against_brute_force(F, k, tau, ties):
    rng = np.random.default_rng(F * 31 + (k or 0))
    for trial in range(5):
        A = rng.integers(0, 4, (F, F)).astype(np.float64) if ties else rng.random((F, F))
        M = np.triu(A, 1) + np.triu(A, 1).T
        ids = sorted(rng.choice(100, F, replace=False).tolist())
        ts, c = ops.flare_weights(M, ids, k, tau)
        bts, bc = _brute_weights(M.tolist(), ids, k, tau)
        assert c.tolist() == bc
        np.testing.assert_allclose(ts, bts, rtol=1e-14)
        assert abs(ts.sum() - 1.0) < 1e-14 and c.sum() == F * min(F // 2 if k is None else k, F - 1)


def test_ties_go_to_the_lower_position():
    M = np.zeros((4, 4))
    ts, c = ops.flare_weights(M, [0, 1, 2, 3], 1, 1.0)
    assert c.tolist() == [3, 1, 0, 0]                                  # 0 is everyone else's neighbour; 1 is 0's


# ---- the feature tap ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", [m for m in MODELS if m != "auto"])
def test_feature_tap_is_the_forward_truncated_before_the_head(model):
    from rlr_b200.models import get_layout
    from rlr_b200.models.graph import GraphNet, Node, feature_dim, head_index
    from rlr_b200.trainers import TorchTrainer
    lay = get_layout(model)
    data = "fmnist" if lay.in_shape[0] == 1 else "cifar10"
    w = torch.zeros(lay.n_total)
    lay.init_(w, 1)
    for b in lay.buffers:
        v = lay.view(w, b)
        v.copy_(0.1 * torch.randn(v.shape) if b.kind == "bn_mean" else 0.5 + torch.rand(v.shape))
    C, H, W = lay.in_shape
    x = torch.randn(5, C, H, W, generator=torch.Generator().manual_seed(0))
    tr = TorchTrainer(lay, make_args(data=data, model=model, bs=2, device="cpu"), "cpu", 8)
    z = tr.root_features(w, x)                                         # three chunks of --bs 2
    assert z.shape == (5, feature_dim(lay)) and z.dtype == torch.float32
    # the explicit forward: a GraphNet over the nodes before the head, the head's input moved to the output slot, eval mode
    import copy
    head = head_index(lay)
    short = copy.copy(lay)
    short.nodes = lay.nodes[:head] + [Node("save", inp=lay.nodes[head].inp, out="x")]
    trunc, net = GraphNet(short, w.clone()), GraphNet(lay, w.clone())
    trunc.eval()
    net.eval()
    with torch.no_grad():
        ref = torch.cat([trunc(x[s:s + 2]) for s in range(0, 5, 2)])      # the same --bs chunks
        logits = net(x)
    assert torch.equal(z, ref)
    hw, hb = lay.view(w, lay.by_name[lay.nodes[head].name + ".weight"]), lay.view(w, lay.by_name[lay.nodes[head].name + ".bias"])
    torch.testing.assert_close(torch.nn.functional.linear(z, hw, hb), logits, rtol=1e-5, atol=1e-5)
    w2 = w.clone()
    w2[: lay.n_vote] *= 1.01
    assert not torch.equal(tr.root_features(w2, x), z)                # one executor, rebound to the parameters it is handed
    assert torch.equal(tr.root_features(w, x), z)


# ---- the server step ----------------------------------------------------------------------------------------------------
def _round(K, n, R, d, seed, bad=()):
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(n, generator=gen)
    ws = [g + 0.05 * (1 + k % 3) * torch.randn(n, generator=gen) for k in range(K)]
    centres = torch.randn(3, d, generator=gen)
    Z = torch.stack([torch.relu(centres[k % 3] + 0.5 * torch.randn(R, d, generator=gen)) for k in range(K)])
    for k in bad:
        Z[k, 0, 0] = float("nan")
    return g, ws, Z


def _oracle(g, ws, Z, nv, theta, server_lr, k=None, tau=1.0, opt=None, cand=None):
    K = len(ws)
    cand = list(range(K)) if cand is None else cand
    res = ops.flare_statement(Z[cand], k, tau)
    F = [cand[j] for j in res.members]
    if not F:
        return g.clone(), []
    wts = [float(np.float32(res.weights[m])) for m in res.members]
    ref, _ = ops.aggregate_oracle(g, [ws[j] for j in F], wts, "avg", theta, server_lr, None, nv, None, opt)
    return ref, F


@pytest.mark.parametrize("theta,server_opt,bad,k", [(0, "sgd", (), None), (2, "sgd", (1,), None), (0, "adam", (), 2), (2, "adam", (0, 3), 1),
                                                    (2, "sgd", tuple(range(6)), None)])
def test_aggregate_updates_equals_the_statement_and_the_avg_oracle(theta, server_opt, bad, k):
    K, n, nv = 6, 512, 480
    g, ws, Z = _round(K, n, 7, 16, 7, bad)
    a = make_args(num_agents=K, num_corrupt=2, aggr="flare", robustLR_threshold=theta, server_opt=server_opt, server_lr=0.05, flare_k=k)
    agg = Aggregation({i: 100 + 13 * i for i in range(K)}, n, None, a)
    opt = ops.ServerOptState(server_opt, n, beta1=a.server_beta1, beta2=a.server_beta2, tau=a.server_tau)
    wg = g.clone()
    for rnd in (1, 2):
        ref, F = _oracle(wg, ws, Z, nv, theta, a.server_lr, k, 1.0, opt)
        agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, rnd, n_vote=nv, features=Z)
        torch.testing.assert_close(wg, ref, rtol=0, atol=1e-6)
        assert agg.last_admitted == F == [j for j in range(K) if j not in bad]
        lf = agg.last_flare
        res = ops.flare_statement(Z, k, 1.0)
        assert abs(lf["FLARE/Corrupt_Weight"] - float(res.weights[:2].sum())) < 1e-15
        if F:
            assert lf["FLARE/Bandwidth"] == res.sigma2 and lf["FLARE/Bandwidth"] > 0


def test_aggregate_updates_needs_the_features():
    g, ws, Z = _round(3, 64, 4, 8, 1)
    agg = Aggregation({i: 1 for i in range(3)}, 64, None, make_args(num_agents=3, aggr="flare"))
    with pytest.raises(ValueError, match="features"):
        agg.aggregate_updates(g.clone(), {i: ws[i] for i in range(3)}, 1)


def test_multikrum_then_flare():
    K, n, nv = 7, 256, 240
    g, ws, Z = _round(K, n, 5, 8, 8)
    ws[0] = ws[0] + 3.0                                                  # far from everyone: rejected by multikrum first
    a = make_args(num_agents=K, num_corrupt=1, aggr="flare", robustLR_threshold=2, select="multikrum")
    agg = Aggregation({i: 50 + 7 * i for i in range(K)}, n, None, a)
    wg = g.clone()
    agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv, features=Z)
    ref, F = _oracle(g, ws, Z, nv, 2, a.server_lr, cand=list(range(1, K)))
    assert agg.last_admitted == F == list(range(1, K))
    torch.testing.assert_close(wg, ref, rtol=0, atol=1e-6)


def _local_aggregator(n, nv, slots):
    from rlr_b200.parallel import FusedAggregator, init_distributed
    return FusedAggregator(init_distributed("cpu"), n, nv, slots, "local")


@pytest.mark.parametrize("bad", [(), (2,), tuple(range(5))])
def test_slots_form_equals_the_dict_form(bad):
    K, n, nv = 5, 256, 240
    g, ws, Z = _round(K, n, 6, 8, 10, bad)
    sizes = {i: 50 + 7 * i for i in range(K)}
    a = make_args(num_agents=K, num_corrupt=1, aggr="flare", robustLR_threshold=2, noise=0.1, clip=0.5)
    fa = _local_aggregator(n, nv, K)
    fa.w_global.copy_(g)
    for j in range(K):
        fa.slots[j].copy_(ws[j])
    agg = Aggregation(sizes, n, None, a, fused=fa)
    agg.aggregate_slots(list(range(K)), 1, Z.clone())
    dict_form = Aggregation(sizes, n, None, a)
    wg = g.clone()
    dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv, features=Z)
    assert agg.last_admitted == dict_form.last_admitted == [j for j in range(K) if j not in bad]
    assert agg.last_flare == dict_form.last_flare
    assert torch.equal(fa.w_global, wg)
    fa.close()


# ---- engine runs ----------------------------------------------------------------------------------------------------------
def _engine(**kw):
    base = dict(data="fmnist", synthetic=1200, synthetic_val=300, num_agents=4, local_ep=1, bs=64, device="cpu", num_corrupt=1,
                poison_frac=0.5, aggr="flare", root_size=40, robustLR_threshold=2, log_dir="", seed=5, trainer="torch")
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def test_engine_root_set_and_no_root_job():
    e = _engine(num_corrupt=2)
    poisoned = {i for a in e.agents for i in a.poisoned_idxs}
    assert e.root_agent is None and e.fused.max_slots == 4               # nothing is trained on R
    assert e.flare_x.shape == (40, 1, 28, 28) and e.flare_local.shape == (4, 40, 128)
    from rlr_b200.engine import draw_root_set
    root = draw_root_set(len(e.train_dataset), sorted(poisoned), 40, 5)
    assert not poisoned & set(root.tolist())
    x, _ = e.train_dataset.batch(torch.as_tensor(root))
    assert torch.equal(e.flare_x, x)
    e.close()


def test_engine_logs_the_flare_fields(tmp_path):
    eng = _engine(log_dir=str(tmp_path / "logs"), no_tensorboard=True, rounds=2, attack_boost=5.0)
    hist = eng.fit()
    eng.close()
    run_dirs = os.listdir(tmp_path / "logs")
    recs = [json.loads(l) for d in run_dirs for l in open(tmp_path / "logs" / d / "metrics.jsonl")]
    assert [r["round"] for r in recs] == [1, 2]
    for r, h in zip(recs, hist):
        for key in ("flare_avg_honest", "flare_avg_corrupt", "flare_corrupt_weight", "flare_bandwidth"):
            assert key in r and r[key] == h[key]
        assert 0 <= r["flare_corrupt_weight"] <= 1 and r["flare_bandwidth"] > 0
        assert abs(3 * r["flare_avg_honest"] + r["flare_corrupt_weight"] - 1.0) < 1e-12


def test_engine_writes_the_tensorboard_tags():
    from rlr_b200.aggregation import Aggregation as Agg

    class W:
        def __init__(self):
            self.tags = {}

        def add_scalar(self, k, v, r):
            self.tags[k] = v
    K, n = 4, 64
    g, ws, Z = _round(K, n, 5, 8, 2)
    w = W()
    agg = Agg({i: 1 for i in range(K)}, n, None, make_args(num_agents=K, num_corrupt=1, aggr="flare"), writer=w)
    agg.aggregate_updates(g.clone(), {i: ws[i] for i in range(K)}, 1, features=Z)
    assert set(w.tags) == {"FLARE/Avg_Honest_Trust", "FLARE/Avg_Corrupt_Trust", "FLARE/Corrupt_Weight", "FLARE/Bandwidth"}


def test_resume_equals_an_uninterrupted_run(tmp_path):
    full = _engine(rounds=4)
    full.fit()
    ck = str(tmp_path / "ck.pt")
    first = _engine(rounds=2, checkpoint=ck)
    first.fit()
    second = _engine(rounds=4, resume=ck)
    assert second.start_round == 3
    second.fit()
    assert torch.equal(second.w_global, full.w_global)
    assert second.aggregator.last_flare == full.aggregator.last_flare
    for e in (full, first, second):
        e.close()


# ---- 2 ranks over gloo ---------------------------------------------------------------------------------------------------
CASES = {"mixed": (1, 3), "all": (), "none": (0, 1, 2, 3, 4)}


def _transport_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.aggregation import Aggregation as Agg
    from rlr_b200.options import make_args as mk
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed("cpu")
    K, n, nv = 5, 1024, 1000
    out = {}
    for case, bad in CASES.items():
        g, ws, Z = _round(K, n, 6, 8, 21, bad)
        for transport in ("gather", "reduce"):
            slots = (K + world - 1) // world
            fa = FusedAggregator(ctx, n, nv, slots, "gloo", transport=transport)
            fa.w_global.copy_(g)
            local = torch.zeros(slots, 6, 8)
            for j, w in enumerate(ws):
                r, s = fa.slot_owner(j)
                if r == rank:
                    fa.slots[s].copy_(w)
                    local[s] = Z[j]
            agg = Agg({i: 10 + 3 * i for i in range(K)}, n, None, mk(num_agents=K, num_corrupt=1, aggr="flare", robustLR_threshold=2,
                                                                     noise=0.1, clip=0.5), fused=fa)
            agg.aggregate_slots(list(range(K)), 1, local)
            out[(case, transport)] = (fa.w_global.clone(), list(agg.last_admitted), dict(agg.last_flare))
            fa.close()
    torch.save(out, os.path.join(outdir, f"t{rank}.pt"))
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_transports_match_the_dict_form(tmp_path):
    world = 2
    mp.spawn(_transport_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"t{r}.pt") for r in range(world)]
    K, n, nv = 5, 1024, 1000
    for case, bad in CASES.items():
        g, ws, Z = _round(K, n, 6, 8, 21, bad)
        a = make_args(num_agents=K, num_corrupt=1, aggr="flare", robustLR_threshold=2, noise=0.1, clip=0.5)
        dict_form = Aggregation({i: 10 + 3 * i for i in range(K)}, n, None, a)
        wg = g.clone()
        dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv, features=Z)
        want = [i for i in range(K) if i not in bad]
        for o in outs:
            assert o[(case, "gather")][1] == o[(case, "reduce")][1] == dict_form.last_admitted == want, case
            assert o[(case, "gather")][2] == o[(case, "reduce")][2] == dict_form.last_flare, case       # identical weights everywhere
            assert torch.equal(o[(case, "gather")][0], wg), case
            torch.testing.assert_close(o[(case, "reduce")][0], wg, rtol=1e-6, atol=1e-6)
            assert torch.equal(o[(case, "reduce")][0], outs[0][(case, "reduce")][0])


def _engine_worker(rank, world, port, outdir, kw):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.engine import FLEngine as Engine
    from rlr_b200.options import make_args as mk
    eng = Engine(mk(**kw), verbose=False)
    trust, feats = [], []
    for r in range(1, 3):
        eng.run_round(r)
        trust.append(dict(eng.aggregator.last_flare))
        feats.append(eng.fused.flare_features(eng.n_part, eng.flare_local).clone())
    torch.save({"w": eng.w_global.clone(), "trust": trust, "feats": feats, "backend": eng.fused.backend,
                "transport": eng.fused.transport}, os.path.join(outdir, f"e{rank}_{kw['agg_transport']}.pt"))
    eng.close()
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("transport", ["gather", "reduce"])
def test_gloo_engine_ranks_agree(tmp_path, transport):
    """Two ranks over gloo: every rank holds the same features, weights and parameters.  The features are those of the slots each rank
    trained, ordered by participant position."""
    world = 2
    kw = dict(data="fmnist", synthetic=800, synthetic_val=200, num_agents=5, local_ep=1, bs=64, aggr="flare", root_size=32, log_dir="",
              device="cpu", robustLR_threshold=2, seed=3, agg_transport=transport, no_graphs=True)
    mp.spawn(_engine_worker, args=(world, _free_port(), str(tmp_path), kw), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"e{r}_{transport}.pt") for r in range(world)]
    assert outs[0]["backend"] == "gloo" and outs[0]["transport"] == transport
    for o in outs[1:]:
        assert torch.equal(o["w"], outs[0]["w"]) and o["trust"] == outs[0]["trust"]
        assert all(torch.equal(a, b) for a, b in zip(o["feats"], outs[0]["feats"]))
    # the trust of the last round is the statement's on the gathered features
    res = ops.flare_statement(outs[0]["feats"][-1])
    assert outs[0]["trust"][-1]["FLARE/Bandwidth"] == res.sigma2


def test_gloo_features_match_one_process(tmp_path):
    """The same participant slots and features, placed on two ranks or held by one process, give the same gathered features, the same
    weights and the same step (gather transport)."""
    world = 2
    mp.spawn(_transport_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"t{r}.pt") for r in range(world)]
    K, n, nv = 5, 1024, 1000
    for case, bad in CASES.items():
        g, ws, Z = _round(K, n, 6, 8, 21, bad)
        fa = _local_aggregator(n, nv, K)
        fa.w_global.copy_(g)
        for j in range(K):
            fa.slots[j].copy_(ws[j])
        agg = Aggregation({i: 10 + 3 * i for i in range(K)}, n, None,
                          make_args(num_agents=K, num_corrupt=1, aggr="flare", robustLR_threshold=2, noise=0.1, clip=0.5), fused=fa)
        agg.aggregate_slots(list(range(K)), 1, Z.clone())
        for o in outs:
            assert o[(case, "gather")][2] == agg.last_flare and o[(case, "gather")][1] == agg.last_admitted
            assert torch.equal(o[(case, "gather")][0], fa.w_global), case
        fa.close()
