"""DeepSight (``--aggr deepsight``) without a GPU: the options and the banner; ``hdbscan_labels`` against scikit-learn on tie-free
matrices, against a brute-force level-wise evaluation under permutations of tied and zero-distance matrices, and against FLAME's
``_first_cluster``; the statistics statement's closed forms; constructed rounds (one-label heads, identical colluders, a cluster that
takes a benign-looking member down, non-finite candidates, nobody accepted); the in-process step against the avg oracle; engine runs
(log fields, a bit-for-bit resume) and 2-rank gloo runs on both transports against one process."""
import itertools
import json
import os
import socket
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.aggregation import Aggregation
from rlr_b200.engine import FLEngine
from rlr_b200.models import get_layout
from rlr_b200.models.graph import head_slices
from rlr_b200.options import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S = ops.DEEPSIGHT_SEEDS


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- options ------------------------------------------------------------------------------------------------------------------
def test_defaults():
    a = make_args(aggr="deepsight")
    assert a.deepsight_samples == 256 and abs(a.deepsight_tau - 1 / 3) < 1e-15
    b = make_args(aggr="deepsight", deepsight_samples=7, deepsight_tau=1.0, noise=0.1, clip=1.0, robustLR_threshold=9, num_agents=10)
    assert (b.deepsight_samples, b.deepsight_tau) == (7, 1.0)
    assert make_args().deepsight_samples is None and make_args().deepsight_tau is None
    make_args(aggr="deepsight", select="multikrum", num_agents=10, select_f=2, select_m=5)
    make_args(aggr="deepsight", detect="fldetector", num_agents=5)


@pytest.mark.parametrize("kw", [dict(deepsight_samples=8), dict(deepsight_tau=0.5), dict(aggr="flame", deepsight_tau=0.5),
                                dict(aggr="deepsight", deepsight_samples=0), dict(aggr="deepsight", deepsight_samples=2.5),
                                dict(aggr="deepsight", deepsight_tau=0.0), dict(aggr="deepsight", deepsight_tau=1.5),
                                dict(aggr="deepsight", deepsight_tau=float("nan")), dict(aggr="deepsight", deepsight_tau=float("inf")),
                                dict(aggr="deepsight", server_clip=True, clip=1.0)])
def test_deepsight_options_rejected(kw):
    with pytest.raises(ValueError):
        make_args(**kw)


def test_banner_line(capsys):
    from rlr_b200.options import print_exp_details
    print_exp_details(make_args())
    assert "DeepSight" not in capsys.readouterr().out
    print_exp_details(make_args(aggr="deepsight", deepsight_samples=64, deepsight_tau=0.5))
    assert "    DeepSight (seeds x samples / tau): 3 x 64 / 0.5\n" in capsys.readouterr().out
    print_exp_details(make_args(aggr="deepsight"))
    assert "    DeepSight (seeds x samples / tau): 3 x 256 / 0.3333\n" in capsys.readouterr().out


# ---- hdbscan_labels -----------------------------------------------------------------------------------------------------------
def _partition(labels):
    """The partition of ``labels`` with every noise point (-1) its own part, and the noise points."""
    parts = {}
    for i, lab in enumerate(np.asarray(labels).tolist()):
        parts.setdefault(lab if lab >= 0 else -1 - i, []).append(i)
    return sorted(tuple(p) for p in parts.values()), sorted(i for i, lab in enumerate(np.asarray(labels).tolist()) if lab < 0)


def _tie_free(rng, n):
    if rng.random() < 0.5:
        D = rng.random((n, n))
        D = D + D.T
    else:
        X = rng.normal(size=(n, 3))
        X[: n // 3] += 4.0
        X[n // 3: n // 2] -= 3.0
        D = np.sqrt(((X[:, None] - X[None]) ** 2).sum(-1))
    np.fill_diagonal(D, 0.0)
    return D


def test_hdbscan_labels_equal_sklearn_on_tie_free_matrices():
    sk = pytest.importorskip("sklearn.cluster")
    rng = np.random.default_rng(0)
    cases = 0
    for n in range(2, 61):
        for m in range(2, 6):
            for _ in range(2 if n > 30 else 3):
                D = _tie_free(rng, n)
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    want = sk.HDBSCAN(metric="precomputed", min_samples=1, min_cluster_size=m, allow_single_cluster=True,
                                      copy=True).fit(D).labels_
                assert _partition(ops.hdbscan_labels(D, m)) == _partition(want), (n, m)
                cases += 1
    assert cases > 500
    assert ops.hdbscan_labels(np.zeros((1, 1)), 2).tolist() == [-1]          # one point is noise (scikit-learn refuses n = 1)


def _levelwise(D, m):
    """Brute-force statement of the level-wise definition: at every distinct distance h, from the largest down, the connected
    components of {d < h} (breadth-first on the full matrix) inside each living cluster."""
    n = D.shape[0]
    if n < 2:
        return [-1] * n

    def comps(pts, h):
        left, out = set(pts), []
        while left:
            p = min(left)
            seen, todo = {p}, [p]
            while todo:
                x = todo.pop()
                for y in list(left - seen):
                    if D[x, y] < h:
                        seen.add(y)
                        todo.append(y)
            left -= seen
            out.append(sorted(seen))
        return out
    levels = sorted({float(D[i, j]) for i in range(n) for j in range(n) if i != j}, reverse=True)
    clusters = [dict(pts=list(range(n)), birth=0.0, parent=-1, kids=[], stab=0.0, death=0.0)]
    leave = {}
    alive = [0]
    for h in levels:
        lam = 1.0 / h if h > 0 else float("inf")
        nxt = []
        for c in alive:
            cl = clusters[c]
            parts = comps(cl["pts"], h)
            if len(parts) == 1:
                nxt.append(c)
                continue
            big = [q for q in parts if len(q) >= m]
            for q in parts:
                if len(q) < m:
                    for p in q:
                        leave[p] = (c, lam)
                        cl["stab"] += lam - cl["birth"]
            cl["death"] = lam
            if len(big) == 1:
                cl["pts"] = big[0]
                nxt.append(c)
            elif len(big) >= 2:
                for q in big:
                    cl["stab"] += (lam - cl["birth"]) * len(q)
                    clusters.append(dict(pts=q, birth=lam, parent=c, kids=[], stab=0.0, death=lam))
                    cl["kids"].append(len(clusters) - 1)
                    nxt.append(len(clusters) - 1)
        alive = nxt
    sel, val = [False] * len(clusters), [c["stab"] for c in clusters]

    def desc(c):
        for k in clusters[c]["kids"]:
            yield k
            yield from desc(k)
    for c in range(len(clusters) - 1, -1, -1):
        sub = sum(val[k] for k in clusters[c]["kids"])
        if sub > val[c]:
            val[c] = sub
        else:
            sel[c] = True
            for k in desc(c):
                sel[k] = False
    lab = []
    for p in range(n):
        c, lam = leave[p]
        while c != -1 and not sel[c]:
            c = clusters[c]["parent"]
        lab.append(c if (c > 0 or (c == 0 and lam >= clusters[0]["death"])) else -1)
    return lab


@pytest.mark.parametrize("seed", range(12))
def test_hdbscan_labels_on_ties_are_the_levelwise_definition_in_any_order(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(3, 16))
    m = int(rng.integers(2, 4))
    # a co-association-like matrix: small integer distances with many ties, zeros included (identical points)
    D = rng.integers(0, 4, size=(n, n)).astype(np.float64)
    D = np.minimum(D, D.T)
    np.fill_diagonal(D, 0.0)
    want = _partition(_levelwise(D, m))
    assert _partition(ops.hdbscan_labels(D, m)) == want
    for _ in range(20):
        perm = rng.permutation(n)
        got = ops.hdbscan_labels(D[np.ix_(perm, perm)], m)
        back = np.empty(n, dtype=np.int64)
        back[perm] = got
        assert _partition(back) == want


def test_hdbscan_labels_with_m_above_half_is_flames_first_cluster():
    rng = np.random.default_rng(3)
    for n in range(2, 30):
        for _ in range(5):
            D = _tie_free(rng, n) if rng.random() < 0.5 else np.minimum(*(lambda A: (A, A.T))(rng.integers(0, 3, (n, n)).astype(float)))
            np.fill_diagonal(D, 0.0)
            m = n // 2 + 1
            first = ops._first_cluster(D, m)
            lab = ops.hdbscan_labels(D, max(m, 2))
            if m >= 2:
                assert sorted(np.flatnonzero(lab >= 0).tolist()) == sorted(first), (n, D)


# ---- the statistics statement ---------------------------------------------------------------------------------------------------
LAY = get_layout("cnn_cifar")
HEAD = head_slices(LAY)


def _round(K, seed, corrupt=2, N=16):
    """A round on cnn_cifar's flat vectors: honest candidates move every parameter a little and answer the random inputs like the
    global model; the first ``corrupt`` candidates move only row 0 of the head and its bias and raise logit 0 -- a one-label head."""
    w_off, b_off, P, d = HEAD
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(LAY.n_total, generator=gen)
    zg = torch.randn(S * N, P, generator=gen)
    ws, z = [], []
    for k in range(K):
        w = g + 0.01 * torch.randn(LAY.n_total, generator=gen)
        zk = zg + 0.05 * torch.randn(S * N, P, generator=gen)
        if k < corrupt:
            w[w_off:w_off + P * d] = g[w_off:w_off + P * d]
            w[b_off:b_off + P] = g[b_off:b_off + P]
            w[w_off:w_off + d] += 0.5
            w[b_off] += 0.5
            zk[:, 0] += 2.0
        ws.append(w)
        z.append(zk)
    return g, ws, torch.stack(z), zg


def test_statement_against_the_definitions():
    g, ws, z, zg = _round(3, 1)
    st = ops.deepsight_stats_statement(z, zg, ws, g, HEAD).numpy()
    w_off, b_off, P, d = HEAD
    N = z.shape[1] // S
    zz, gg = z.double().numpy(), zg.double().numpy()
    lse = lambda a: np.log(np.exp(a).sum(-1, keepdims=True))
    ddif = np.exp((zz - lse(zz)) - (gg - lse(gg))[None]).reshape(3, S, N, P).mean(2).reshape(3, -1)
    np.testing.assert_allclose(st[:, :S * P], ddif, rtol=1e-12)
    for k in range(3):
        dW = (ws[k][w_off:w_off + P * d] - g[w_off:w_off + P * d]).reshape(P, d).double()
        db = (ws[k][b_off:b_off + P] - g[b_off:b_off + P]).double()
        np.testing.assert_allclose(st[k, S * P:(S + 1) * P], (db.abs() + dW.abs().sum(1)).numpy(), rtol=1e-13)
        assert np.array_equal(st[k, (S + 1) * P:], db.numpy())


def test_closed_forms():
    g, ws, z, zg = _round(4, 2, corrupt=1)
    ws[3] = g.clone()                                                  # a candidate equal to w_g
    z[3] = zg
    st = ops.deepsight_stats_statement(z, zg, ws, g, HEAD)
    P = HEAD[2]
    assert torch.equal(st[3, :S * P], torch.ones(S * P, dtype=torch.float64)) and not st[3, S * P:].any()
    res = ops.deepsight_decide(st, torch.tensor([1.0, 1.0, 1.0, 0.0]), [0, 1, 2, 3], 1 / 3)
    assert res.te[3] == 0 and res.te[0] == 1 and res.te[1] == res.te[2] == P      # one-class head: TE 1; every class moved: TE P
    assert res.suspicious.tolist() == [True, False, False, True]
    assert float(res.scales[3]) == 1.0                                 # e_k = 0: scale 1
    # all-equal TEs: nobody is suspicious
    g, ws, z, zg = _round(5, 3, corrupt=0)
    res = ops.deepsight_statement(z, zg, ws, g, HEAD, list(range(5)), 1 / 3)
    assert (res.te == P).all() and not res.suspicious.any() and res.members == list(range(5))


# ---- constructed rounds ---------------------------------------------------------------------------------------------------------
def test_one_label_heads_are_rejected_and_honest_ones_accepted():
    g, ws, z, zg = _round(10, 4)
    res = ops.deepsight_statement(z, zg, ws, g, HEAD, list(range(10)), 1 / 3)
    assert res.members == list(range(2, 10)) and res.suspicious.tolist() == [True] * 2 + [False] * 8
    assert res.labels[0] == res.labels[1] and res.labels[0] not in res.labels[2:].tolist()


@pytest.mark.parametrize("poisoned", [False, True])
def test_identical_colluders_form_one_part_and_share_its_fate(poisoned):
    g, ws, z, zg = _round(9, 5, corrupt=3 if poisoned else 0)
    for k in (1, 2):                                                   # ALIE / Min-Max submit one crafted update three times
        ws[k], z[k] = ws[0].clone(), z[0].clone()
    ids = [7, 3, 5, 0, 1, 2, 4, 6, 8]
    res = ops.deepsight_statement(z, zg, ws, g, HEAD, ids, 1 / 3)
    assert res.labels[0] == res.labels[1] == res.labels[2] >= 0
    assert all(k in res.members for k in (0, 1, 2)) == (not poisoned)
    assert all(k not in res.members for k in (0, 1, 2)) == poisoned
    assert res.members == (list(range(3, 9)) if poisoned else list(range(9)))
    for _ in range(4):                                                 # the decision does not depend on the candidates' positions
        perm = np.random.default_rng(_).permutation(9).tolist()
        r2 = ops.deepsight_statement(z[perm], zg, [ws[p] for p in perm], g, HEAD, [ids[p] for p in perm], 1 / 3)
        assert sorted(perm[j] for j in r2.members) == res.members


def _stats(P, rows):
    """Statistics rows from (ddif [S][P] or a scalar, eps [P], db [P])."""
    out = []
    for ddif, eps, db in rows:
        dd = np.broadcast_to(np.asarray(ddif, dtype=np.float64), (S, P)).reshape(-1)
        out.append(np.concatenate([dd, np.asarray(eps, dtype=np.float64), np.asarray(db, dtype=np.float64)]))
    return torch.from_numpy(np.stack(out))


def test_a_suspicious_majority_takes_a_benign_looking_member_down():
    P, rng = 10, np.random.default_rng(7)
    one = np.eye(P)[0]
    rows = [(np.where(np.arange(P) == 0, 3.0, 0.8), one * 5 + 1e-4, one * 0.5 + 0.001 * rng.normal(size=P)) for _ in range(2)]
    # benign-looking: every class of its head moved (TE = P), but it behaves and moves its bias like the two poisoned ones
    rows.append((np.where(np.arange(P) == 0, 3.0, 0.8), np.ones(P), one * 0.5 + 0.001 * rng.normal(size=P)))
    for _ in range(7):
        rows.append((1.0 + 0.001 * rng.normal(size=P), np.ones(P) + 0.01 * rng.normal(size=P), -one * 0.1 + 0.001 * rng.normal(size=P)))
    res = ops.deepsight_decide(_stats(P, rows), torch.ones(10), list(range(10)), 1 / 3)
    assert res.suspicious.tolist() == [True, True] + [False] * 8
    assert res.labels[0] == res.labels[1] == res.labels[2] and res.labels[2] not in res.labels[3:].tolist()
    assert res.members == list(range(3, 10))


def test_non_finite_candidates_are_never_accepted():
    g, ws, z, zg = _round(6, 8, corrupt=0)
    z[1, 5, 3] = float("nan")
    z[2, 0, 0] = -float("inf")
    ws[3] = ws[3].clone()
    ws[3][HEAD[1]] = float("inf")
    norms = ops.update_norms(g, ws, LAY.n_vote)
    st = ops.deepsight_stats_statement(z, zg, ws, g, HEAD)
    res = ops.deepsight_decide(st, norms, list(range(6)), 1.0)
    assert res.finite == [0, 4, 5] and res.members == [0, 4, 5]
    norms[4] = float("nan")
    res = ops.deepsight_decide(st, norms, list(range(6)), 1.0)
    assert res.finite == [0, 5] and res.members == [0, 5] and (res.labels[[1, 2, 3, 4]] == -1).all()
    res = ops.deepsight_decide(st[[1, 2, 3]], norms[[1, 2, 3]], [1, 2, 3], 1.0)
    assert res.members == [] and res.finite == [] and res.clip_bound is None


# ---- the in-process step ----------------------------------------------------------------------------------------------------------
def _agg(K, **kw):
    a = make_args(num_agents=K, num_corrupt=2, aggr="deepsight", **kw)
    return Aggregation({i: 100 + 13 * i for i in range(K)}, LAY.n_params, None, a, layout=LAY), a


@pytest.mark.parametrize("theta,server_opt", [(0, "sgd"), (3, "sgd"), (2, "adam")])
def test_aggregate_updates_equals_the_avg_oracle(theta, server_opt):
    K = 8
    g, ws, z, zg = _round(K, 9)
    ws[5] = g + 5.0 * (ws[5] - g)                                      # a long update: clipped to the median norm
    agg, a = _agg(K, robustLR_threshold=theta, server_opt=server_opt, server_lr=0.5)
    opt = ops.ServerOptState(server_opt, LAY.n_total, beta1=a.server_beta1, beta2=a.server_beta2, tau=a.server_tau)
    wg = g.clone()
    for rnd in (1, 2):
        res = ops.deepsight_statement(z, zg, ws, wg, HEAD, list(range(K)), a.deepsight_tau, LAY.n_vote)
        A = res.members
        ref, _ = ops.aggregate_oracle(wg, [ws[j] for j in A], [1.0] * len(A), "avg", theta, a.server_lr, None, LAY.n_vote,
                                      res.scales[A], opt)
        agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, rnd, logits=z, global_logits=zg)
        torch.testing.assert_close(wg, ref, rtol=0, atol=1e-6)
        assert agg.last_admitted == A == list(range(2, K))
        ld = agg.last_deepsight
        assert ld["DeepSight/Accepted"] == 6 and ld["DeepSight/Corrupt_Accepted"] == 0 and ld["DeepSight/Suspicious"] == 2
        assert ld["DeepSight/Corrupt_Suspicious"] == 2 and ld["DeepSight/Clusters"] >= 2 and ld["DeepSight/Clip_Bound"] == res.clip_bound
        assert float(res.scales[5]) < 1.0


def test_aggregate_updates_needs_the_logits():
    g, ws, z, zg = _round(3, 1)
    agg, _ = _agg(3)
    with pytest.raises(ValueError, match="logits"):
        agg.aggregate_updates(g.clone(), {i: ws[i] for i in range(3)}, 1, logits=z)


def test_nobody_accepted_gives_zero_plus_noise():
    K = 4
    g, ws, z, zg = _round(K, 10, corrupt=0)
    w_off, b_off, P, d = HEAD
    for w in ws:                                                       # no head moved: every TE is 0, so everybody is suspicious
        w[w_off:w_off + P * d] = g[w_off:w_off + P * d]
        w[b_off:b_off + P] = g[b_off:b_off + P]
    agg, _ = _agg(K)
    wg = g.clone()
    agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, logits=z, global_logits=zg)
    assert torch.equal(wg, g) and agg.last_admitted == [] and agg.last_deepsight["DeepSight/Suspicious"] == K
    agg, a = _agg(K, noise=0.1, clip=0.5)
    wg = g.clone()
    agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, logits=z, global_logits=zg)
    ref, _ = ops.aggregate_oracle(g, ws, [0.0] * K, "avg", 0, 1.0, None, LAY.n_vote, None, None, 1.0)
    noise = (wg - ref)[:LAY.n_vote].double()
    assert torch.equal(wg[LAY.n_vote:], g[LAY.n_vote:]) and abs(float(noise.std()) / 0.05 - 1) < 0.05


def test_tensorboard_tags():
    class W:
        def __init__(self):
            self.tags = {}

        def add_scalar(self, k, v, r):
            self.tags[k] = v
    g, ws, z, zg = _round(4, 2)
    w = W()
    agg = Aggregation({i: 1 for i in range(4)}, LAY.n_params, None, make_args(num_agents=4, num_corrupt=2, aggr="deepsight"), writer=w,
                      layout=LAY)
    agg.aggregate_updates(g.clone(), {i: ws[i] for i in range(4)}, 1, logits=z, global_logits=zg)
    assert set(w.tags) == {f"DeepSight/{t}" for t in ("Accepted", "Corrupt_Accepted", "Suspicious", "Corrupt_Suspicious", "Clusters",
                                                      "Clip_Bound")}


# ---- engine runs ----------------------------------------------------------------------------------------------------------
def _engine(**kw):
    base = dict(data="fmnist", synthetic=1200, synthetic_val=300, num_agents=4, local_ep=1, bs=64, device="cpu", num_corrupt=1,
                poison_frac=0.5, aggr="deepsight", deepsight_samples=16, robustLR_threshold=0, log_dir="", seed=5, trainer="torch")
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def test_engine_random_inputs_and_statistics():
    e = _engine()
    from rlr_b200.data import DATASET_META
    assert e.ds_x.shape == (3 * 16, 1, 28, 28) and e.ds_local.shape == (4, (S + 2) * 10) and e.ds_local.dtype == torch.float64
    assert torch.equal(e.ds_x, ops.deepsight_inputs(DATASET_META["fmnist"], 5, 16, "cpu"))
    assert not torch.equal(e.ds_x, ops.deepsight_inputs(DATASET_META["fmnist"], 6, 16, "cpu"))
    e.run_round(1)
    assert torch.isfinite(e.ds_local).all() and e.aggregator.last_deepsight["DeepSight/Clip_Bound"] > 0
    e.close()


def test_engine_logs_the_deepsight_fields(tmp_path):
    eng = _engine(log_dir=str(tmp_path / "logs"), no_tensorboard=True, rounds=2)
    hist = eng.fit()
    eng.close()
    recs = [json.loads(l) for d in os.listdir(tmp_path / "logs") for l in open(tmp_path / "logs" / d / "metrics.jsonl")]
    assert [r["round"] for r in recs] == [1, 2]
    for r, h in zip(recs, hist):
        for key in ("accepted", "corrupt_accepted", "suspicious", "corrupt_suspicious", "clusters", "clip_bound"):
            assert f"deepsight_{key}" in r and r[f"deepsight_{key}"] == h[f"deepsight_{key}"]
        assert 0 <= r["deepsight_corrupt_accepted"] <= r["deepsight_accepted"] <= 4 and r["deepsight_clip_bound"] > 0


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
    assert second.aggregator.last_deepsight == full.aggregator.last_deepsight
    for e in (full, first, second):
        e.close()


# ---- 2 ranks over gloo ---------------------------------------------------------------------------------------------------
CASES = {"mixed": 2, "honest": 0}


def _transport_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.aggregation import Aggregation as Agg
    from rlr_b200.options import make_args as mk
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed("cpu")
    K = 5
    out = {}
    for case, corrupt in CASES.items():
        g, ws, z, zg = _round(K, 21, corrupt)
        for transport in ("gather", "reduce"):
            slots = (K + world - 1) // world
            fa = FusedAggregator(ctx, LAY.n_total, LAY.n_vote, slots, "gloo", transport=transport)
            fa.w_global.copy_(g)
            local = torch.zeros(slots, (S + 2) * HEAD[2], dtype=torch.float64)
            for j, w in enumerate(ws):
                r, s = fa.slot_owner(j)
                if r == rank:
                    fa.slots[s].copy_(w)
                    local[s] = ops.deepsight_stats(z[j:j + 1], zg, [fa.slots[s]], fa.w_global, HEAD)[0]
            agg = Agg({i: 10 + 3 * i for i in range(K)}, LAY.n_params, None,
                      mk(num_agents=K, num_corrupt=2, aggr="deepsight", noise=0.1, clip=0.5), layout=LAY, fused=fa)
            agg.aggregate_slots(list(range(K)), 1, deepsight_local=local)
            out[(case, transport)] = (fa.w_global.clone(), list(agg.last_admitted), dict(agg.last_deepsight))
            fa.close()
    torch.save(out, os.path.join(outdir, f"t{rank}.pt"))
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_transports_match_one_process(tmp_path):
    from rlr_b200.parallel import FusedAggregator, init_distributed
    world = 2
    mp.spawn(_transport_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"t{r}.pt") for r in range(world)]
    K = 5
    for case, corrupt in CASES.items():
        g, ws, z, zg = _round(K, 21, corrupt)
        fa = FusedAggregator(init_distributed("cpu"), LAY.n_total, LAY.n_vote, K, "local")
        fa.w_global.copy_(g)
        for j in range(K):
            fa.slots[j].copy_(ws[j])
        agg = Aggregation({i: 10 + 3 * i for i in range(K)}, LAY.n_params, None,
                          make_args(num_agents=K, num_corrupt=2, aggr="deepsight", noise=0.1, clip=0.5), layout=LAY, fused=fa)
        agg.aggregate_slots(list(range(K)), 1, deepsight_local=ops.deepsight_stats(z, zg, ws, g, HEAD))
        assert agg.last_admitted == list(range(corrupt, K))
        for o in outs:
            for transport in ("gather", "reduce"):
                assert o[(case, transport)][1] == agg.last_admitted and o[(case, transport)][2] == agg.last_deepsight, (case, transport)
            assert torch.equal(o[(case, "gather")][0], fa.w_global), case
            torch.testing.assert_close(o[(case, "reduce")][0], fa.w_global, rtol=1e-6, atol=1e-6)
            assert torch.equal(o[(case, "reduce")][0], outs[0][(case, "reduce")][0])
        fa.close()
