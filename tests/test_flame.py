"""FLAME aggregation (``--aggr flame``) on CPU: option validation and the banner, the fp64 Gram statement against numpy, the clustering
rule against a brute-force evaluation of its definition and against scikit-learn's HDBSCAN, its properties, constructed rounds (colluders,
a boosted update, the clip bound and the noise), the server step against the oracle, the slots form, 2-rank gloo runs on both transports,
and engine runs (JSONL fields, TensorBoard tags, resume)."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.aggregation import Aggregation
from rlr_b200.options import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- options ------------------------------------------------------------------------------------------------------------
def test_defaults():
    a = make_args(aggr="flame")
    assert a.flame_lambda == 1e-3 and a.server_lr == 1.0
    assert make_args(aggr="flame", flame_lambda=0.0).flame_lambda == 0.0
    assert make_args().flame_lambda is None
    assert make_args(aggr="flame", num_agents=10, robustLR_threshold=6).robustLR_threshold == 6        # floor(10 / 2) + 1
    assert make_args(aggr="flame", num_agents=7, num_corrupt=1, select="multikrum", robustLR_threshold=4).select_m == 6


@pytest.mark.parametrize("kw", [
    dict(aggr="avg", flame_lambda=1e-3),
    dict(aggr="rfa", flame_lambda=0.0),
    dict(aggr="flame", flame_lambda=-1e-3),
    dict(aggr="flame", flame_lambda=float("inf")),
    dict(aggr="flame", flame_lambda=float("nan")),
    dict(aggr="flame", server_clip=True, clip=1.0),
    dict(aggr="flame", noise=0.1, clip=1.0),
    dict(aggr="flame", num_agents=10, robustLR_threshold=7),
    dict(aggr="flame", num_agents=7, num_corrupt=1, select="multikrum", robustLR_threshold=5),   # 6 candidates admit at least 4
])
def test_flame_options_rejected(kw):
    with pytest.raises(ValueError):
        make_args(**kw)


def test_command_line_flags_and_banner(capsys):
    from rlr_b200.options import args_parser, finalize_args, print_exp_details
    a = finalize_args(args_parser(["--aggr", "flame", "--flame_lambda", "0.01"]))
    assert a.flame_lambda == 0.01
    with pytest.raises(ValueError):
        finalize_args(args_parser(["--flame_lambda", "0.01"]))
    print_exp_details(make_args())
    assert "FLAME" not in capsys.readouterr().out
    print_exp_details(a)
    out = capsys.readouterr().out
    assert "FLAME lambda: 0.01" in out and "Aggregation Function: flame" in out


# ---- the Gram statement -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,n,n_vote", [(1, 16, 16), (5, 64, 48), (9, 200, 180)])
def test_gram_statement_matches_numpy(K, n, n_vote):
    gen = torch.Generator().manual_seed(K * n)
    g = torch.randn(n, generator=gen)
    ws = [g + 0.1 * (k + 1) * torch.randn(n, generator=gen) for k in range(K)]
    for w in ws:
        w[n_vote:] += 1e3                                                 # tail coordinates do not count
    G = ops.pairwise_gram(ws, g, n_vote)
    assert G.dtype == torch.float64 and G.shape == (K, K)
    assert torch.equal(G, ops.gram_statement(ws, g, 0, n_vote))
    x = np.stack([np.asarray(w[:n_vote], dtype=np.float64) - np.asarray(g[:n_vote], dtype=np.float64) for w in ws])
    np.testing.assert_allclose(G.numpy(), x @ x.T, rtol=1e-12, atol=1e-12)


# ---- the clustering rule ------------------------------------------------------------------------------------------------
def _brute_force(G, lam=0.0):
    """FLAME's admission straight from its definition, in position order: every candidate threshold h (each distinct distance), the graph
    of the edges d_ij <= h over the candidates with a finite norm, its connected components by search."""
    G = np.asarray(G, dtype=np.float64)
    K = G.shape[0]
    e = np.sqrt(np.diag(G))
    d = np.full((K, K), np.inf)
    for i in range(K):
        for j in range(K):
            if e[i] > 0 and e[j] > 0:
                c = G[i, j] / np.sqrt(G[i, i] * G[j, j])
                c = min(1.0, max(-1.0, c)) if c == c else c
            else:
                c = 0.0
            d[i, j] = np.inf if np.isnan(1.0 - c) else 1.0 - c
    ok = [k for k in range(K) if np.isfinite(e[k])]
    m = K // 2 + 1
    admitted = []
    if K == 1:
        admitted = ok
    else:
        for h in sorted({d[i, j] for i in ok for j in ok if i != j}):
            seen, best = set(), []
            for s in ok:
                if s in seen:
                    continue
                comp, stack = [], [s]
                seen.add(s)
                while stack:
                    u = stack.pop()
                    comp.append(u)
                    for v in ok:
                        if v not in seen and d[u, v] <= h:
                            seen.add(v); stack.append(v)
                if len(comp) > len(best):
                    best = comp
            if len(best) >= m:
                admitted = sorted(best)
                break
    S = float(np.median(np.where(np.isnan(e), np.inf, e)))
    sc = np.array([np.float32(min(1.0, S / x)) if x > 0 else np.float32(1.0) for x in e], dtype=np.float32)
    return admitted, sc, S, lam * S


def _gram(X):
    G = X @ X.T
    return np.triu(G) + np.triu(G, 1).T                                  # exactly symmetric


def _random_gram(rng, sybils=False):
    K = int(rng.integers(1, 24))
    d = int(rng.integers(2, 12))
    X = rng.standard_normal((K, d))
    c = int(rng.integers(0, K // 2 + 1))
    X[:c] += rng.standard_normal(d) * rng.uniform(0, 4)
    if sybils and K >= 3:
        b = int(rng.integers(2, K + 1))                                   # a block of identical updates: tied (zero) distances
        X[K - b:] = X[K - 1]
        if rng.random() < 0.5:
            X[0] = X[1]
    if rng.random() < 0.2:
        X[int(rng.integers(0, K))] = 0.0                                  # a zero update: cosine 0 with everyone
    return _gram(X)


@pytest.mark.parametrize("sybils", [False, True])
def test_admission_equals_the_brute_force_definition(sybils):
    rng = np.random.default_rng(17 + sybils)
    for _ in range(150):
        G = _random_gram(rng, sybils)
        K = G.shape[0]
        members, sc, S, noise = ops.flame_admit(torch.from_numpy(G), list(range(100, 100 + K)), 0.25)
        want, want_sc, want_S, want_noise = _brute_force(G, 0.25)
        assert members == want
        assert S == want_S and noise == want_noise
        assert sc.dtype == torch.float32 and np.array_equal(sc.numpy(), want_sc)


@pytest.mark.filterwarnings("ignore::FutureWarning")
def test_admission_equals_sklearn_hdbscan():
    sk = pytest.importorskip("sklearn.cluster")
    rng = np.random.default_rng(3)
    for _ in range(100):
        K = int(rng.integers(3, 40))
        X = rng.standard_normal((K, int(rng.integers(2, 30))))
        c = int(rng.integers(0, K // 2 + 1))
        X[:c] += rng.standard_normal(X.shape[1]) * rng.uniform(0, 5)
        G = _gram(X)
        e = np.sqrt(np.diag(G))
        D = np.clip(1.0 - G / np.outer(e, e), 0.0, 2.0)
        np.fill_diagonal(D, 0.0)
        labels = sk.HDBSCAN(min_cluster_size=K // 2 + 1, min_samples=1, allow_single_cluster=True,
                            metric="precomputed").fit(D).labels_
        members, _, _, _ = ops.flame_admit(G, list(range(K)), 1e-3)
        assert members == np.flatnonzero(labels >= 0).tolist()


def test_admission_properties():
    rng = np.random.default_rng(5)
    for _ in range(100):
        G = _random_gram(rng, sybils=rng.random() < 0.5)
        K = G.shape[0]
        ids = rng.permutation(1000)[:K].tolist()
        members, sc, S, _ = ops.flame_admit(G, ids, 1e-3)
        assert len(members) >= K // 2 + 1                                # every norm is finite
        p = rng.permutation(K)
        members_p, sc_p, S_p, _ = ops.flame_admit(G[np.ix_(p, p)], [ids[k] for k in p], 1e-3)
        assert sorted(ids[j] for j in members) == sorted(ids[p[j]] for j in members_p)
        assert S_p == S and np.array_equal(sc_p.numpy(), sc.numpy()[p])
        bad = int(rng.integers(0, K))
        Gn = G.copy()
        Gn[bad, :] = np.nan
        Gn[:, bad] = np.nan
        members_n, sc_n, _, _ = ops.flame_admit(Gn, ids, 1e-3)
        assert bad not in members_n and sc_n[bad] == 1.0


def test_nobody_admitted_when_too_few_finite_norms():
    G = _gram(np.eye(3))
    G[0, 0] = G[1, 1] = np.inf
    members, _, S, noise = ops.flame_admit(G, [0, 1, 2], 0.5)
    assert members == [] and S == np.inf and noise == np.inf
    assert ops.flame_admit(np.array([[4.0]]), [7], 0.5)[:1] == ([0],)
    assert ops.flame_admit(np.array([[np.nan]]), [7], 0.5)[0] == []


# ---- constructed rounds -------------------------------------------------------------------------------------------------
def _round(K, n, seed, colluders=(), boost=(), spread=0.3):
    """w_global and K participants whose updates point near one direction; the colluders' near another; boosted updates scaled x100."""
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(n, generator=gen)
    honest, evil = torch.randn(n, generator=gen), torch.randn(n, generator=gen)
    ws = []
    for k in range(K):
        u = (evil if k in colluders else honest) + spread * torch.randn(n, generator=gen)
        ws.append(g + 0.01 * (1 + 0.2 * k) * (100.0 if k in boost else 1.0) * u)
    if spread == 0:
        ws = [ws[0].clone() for _ in ws]
    return g, ws


def test_colluders_rejected_and_boosted_update_clipped():
    K, n, nv = 10, 1024, 1000
    g, ws = _round(K, n, 1, colluders=(0, 1, 2), boost=(5,))
    G = ops.gram_statement(ws, g, 0, nv)
    members, sc, S, noise = ops.flame_admit(G, list(range(K)), 1e-3)
    assert len(members) >= K // 2 + 1 and not {0, 1, 2} & set(members) and 5 in members
    e = torch.sqrt(torch.diagonal(G)).numpy()
    assert S == float(np.median(e)) and noise == 1e-3 * S
    assert sc[5] < 0.05 and abs(float(sc[5]) * e[5] - S) <= 1e-6 * S   # the boosted update is admitted and clipped to S
    assert all(float(sc[k]) == min(1.0, np.float32(S / e[k])) for k in range(K))


@pytest.mark.parametrize("norms,S,scales", [
    ([1.0, 2.0, 3.0, 4.0, 5.0], 3.0, [1.0, 1.0, 1.0, 0.75, 0.6]),
    ([1.0, 2.0, 3.0, 4.0], 2.5, [1.0, 1.0, np.float32(2.5 / 3.0), 0.625]),
])
@pytest.mark.parametrize("lam", [0.0, 0.1])
def test_clip_bound_scales_and_noise_by_hand(norms, S, scales, lam):
    K = len(norms)
    e = np.asarray(norms)
    G = 0.9 * np.outer(e, e)                                              # every pair at cosine 0.9
    np.fill_diagonal(G, e * e)
    members, sc, S_got, noise = ops.flame_admit(G, list(range(K)), lam)
    assert members == list(range(K)) and S_got == S and noise == lam * S
    assert sc.tolist() == [float(np.float32(s)) for s in scales]
    if lam == 0.0:
        assert noise == 0.0


# ---- the server step ----------------------------------------------------------------------------------------------------
def _oracle(g, ws, ids, nv, a, rnd, opt=None, cand=None):
    cand = list(range(len(ws))) if cand is None else cand
    members, sc, S, noise_std = ops.flame_admit(ops.gram_statement([ws[j] for j in cand], g, 0, nv), [ids[j] for j in cand],
                                                a.flame_lambda)
    adm = [cand[j] for j in members]
    n = g.numel()
    gen = torch.Generator().manual_seed(int(a.seed) * 1000003 + rnd)
    noise = torch.randn(n, generator=gen, dtype=torch.float64) * noise_std
    noise[nv:] = 0
    ref, _ = ops.aggregate_oracle(g, [ws[j] for j in adm], [1.0] * len(adm), "avg", a.robustLR_threshold, a.server_lr, noise, nv,
                                  [float(sc[j]) for j in members], opt, float(len(adm)))
    return ref, [ids[j] for j in adm], S, noise_std


@pytest.mark.parametrize("theta,server_opt", [(0, "sgd"), (2, "sgd"), (0, "adam"), (2, "adam")])
def test_aggregate_updates_equals_the_oracle_on_the_admitted_set(theta, server_opt):
    K, n, nv = 8, 512, 480
    g, ws = _round(K, n, 7, colluders=(0, 1), boost=(4,))
    a = make_args(num_agents=K, num_corrupt=2, aggr="flame", robustLR_threshold=theta, server_opt=server_opt, server_lr=0.05)
    agg = Aggregation({i: 100 + 13 * i for i in range(K)}, n, None, a)
    opt = ops.ServerOptState(server_opt, n, beta1=a.server_beta1, beta2=a.server_beta2, tau=a.server_tau)
    wg = g.clone()
    for rnd in (1, 2):                                                   # two rounds: the optimizer state carries over
        ref, adm, S, noise_std = _oracle(wg, ws, list(range(K)), nv, a, rnd, opt)
        agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, rnd, n_vote=nv)
        torch.testing.assert_close(wg, ref, rtol=0, atol=1e-6)
        assert agg.last_admitted == adm and len(adm) >= K // 2 + 1
        if rnd == 1:                                                     # (round 2 measures the updates from the new w_global)
            assert not {0, 1} & set(adm)
        assert agg.last_flame == {"FLAME/Admitted": len(adm), "FLAME/Corrupt_Admitted": sum(1 for i in adm if i < 2),
                                  "FLAME/Clip_Bound": S,
                                  "FLAME/Noise_Std": noise_std}


def test_multikrum_then_flame():
    K, n, nv = 7, 256, 240
    g, ws = _round(K, n, 8, colluders=(1, 2))
    ws[0] = ws[0] + 3.0                                                  # far from everyone: rejected by multikrum first
    a = make_args(num_agents=K, num_corrupt=3, aggr="flame", robustLR_threshold=2, select="multikrum", select_f=1)
    agg = Aggregation({i: 50 + 7 * i for i in range(K)}, n, None, a)
    wg = g.clone()
    agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
    ref, adm, _, _ = _oracle(g, ws, list(range(K)), nv, a, 1, cand=list(range(1, K)))
    assert agg.last_admitted == adm == [3, 4, 5, 6]
    torch.testing.assert_close(wg, ref, rtol=0, atol=1e-6)


def _local_aggregator(n, nv, slots):
    from rlr_b200.parallel import FusedAggregator, init_distributed
    return FusedAggregator(init_distributed("cpu"), n, nv, slots, "local")


@pytest.mark.parametrize("select", ["none", "multikrum"])
def test_slots_form_equals_the_dict_form(select):
    K, n, nv = 7, 256, 240
    g, ws = _round(K, n, 10, colluders=(0, 1), boost=(3,))
    sizes = {i: 50 + 7 * i for i in range(K)}
    a = make_args(num_agents=K, num_corrupt=2, aggr="flame", robustLR_threshold=2, select=select, flame_lambda=0.01)
    fa = _local_aggregator(n, nv, K)
    fa.w_global.copy_(g)
    for j in range(K):
        fa.slots[j].copy_(ws[j])
    agg = Aggregation(sizes, n, None, a, fused=fa)
    agg.aggregate_slots(list(range(K)), 1)
    dict_form = Aggregation(sizes, n, None, a)
    wg = g.clone()
    dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
    assert agg.last_admitted == dict_form.last_admitted and agg.last_flame == dict_form.last_flame
    assert 0 not in agg.last_admitted and 1 not in agg.last_admitted
    assert torch.equal(fa.w_global, wg)
    fa.close()


# ---- 2 ranks over gloo ---------------------------------------------------------------------------------------------------
CASES = [("none", (0, 1), 0.3), ("multikrum", (0, 1), 0.3), ("none", (), 0.0)]       # spread 0: identical updates, everyone admitted


def _transport_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.aggregation import Aggregation as Agg
    from rlr_b200.options import make_args as mk
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed("cpu")
    K, n, nv = 7, 1024, 1000
    out = {}
    for select, colluders, spread in CASES:
        g, ws = _round(K, n, 21, colluders=colluders, boost=(4,), spread=spread)
        for transport in ("gather", "reduce"):
            fa = FusedAggregator(ctx, n, nv, (K + world - 1) // world, "gloo", transport=transport)
            fa.w_global.copy_(g)
            for j, w in enumerate(ws):
                r, s = fa.slot_owner(j)
                if r == rank:
                    fa.slots[s].copy_(w)
            agg = Agg({i: 10 + 3 * i for i in range(K)}, n, None, mk(num_agents=K, num_corrupt=2, aggr="flame", robustLR_threshold=2,
                                                                     select=select, flame_lambda=0.01), fused=fa)
            agg.aggregate_slots(list(range(K)), 1)
            out[(select, colluders, transport)] = (fa.w_global.clone(), dict(agg.last_flame), agg.last_admitted)
            fa.close()
    torch.save(out, os.path.join(outdir, f"t{rank}.pt"))
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_transports_match_the_dict_form(tmp_path):
    world = 2
    mp.spawn(_transport_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"t{r}.pt") for r in range(world)]
    K, n, nv = 7, 1024, 1000
    for select, colluders, spread in CASES:
        g, ws = _round(K, n, 21, colluders=colluders, boost=(4,), spread=spread)
        a = make_args(num_agents=K, num_corrupt=2, aggr="flame", robustLR_threshold=2, select=select, flame_lambda=0.01)
        dict_form = Aggregation({i: 10 + 3 * i for i in range(K)}, n, None, a)
        wg = g.clone()
        dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
        if spread == 0:
            assert dict_form.last_admitted == list(range(K))              # everyone admitted: the reduce step all-reduces
        for o in outs:
            for transport in ("gather", "reduce"):
                w, last, adm = o[(select, colluders, transport)]
                assert torch.equal(w, outs[0][(select, colluders, transport)][0]), (select, colluders, transport)
                assert adm == dict_form.last_admitted and last == dict_form.last_flame, (select, colluders, transport)
                if transport == "gather":                                  # the same pass and step on the same copies: the dict form's bits
                    assert torch.equal(w, wg), (select, colluders)
                else:                                                      # all-reduced partial sums: another order of adds
                    torch.testing.assert_close(w, wg, rtol=1e-6, atol=1e-6)


# ---- engine runs -----------------------------------------------------------------------------------------------------------
def test_federated_py_writes_the_flame_fields_and_tags(tmp_path):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "federated.py", "--data=fmnist", "--local_ep=1", "--bs=64", "--num_agents=4", "--rounds=2",
                        "--num_corrupt=1", "--poison_frac=0.5", "--robustLR_threshold=2", "--synthetic=400", "--synthetic_val=80",
                        "--aggr=flame", "--flame_lambda=0.01", f"--log_dir={tmp_path}", "--device=cpu"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "Aggregation Function: flame" in r.stdout and "FLAME lambda: 0.01" in r.stdout
    run_dirs = os.listdir(tmp_path)
    assert len(run_dirs) == 1
    recs = [json.loads(l) for l in open(tmp_path / run_dirs[0] / "metrics.jsonl")]
    assert [rec["round"] for rec in recs] == [1, 2]
    for rec in recs:
        assert 3 <= rec["flame_admitted"] <= 4 and 0 <= rec["flame_corrupt_admitted"] <= 1
        assert rec["flame_clip_bound"] > 0 and rec["flame_noise_std"] == 0.01 * rec["flame_clip_bound"]
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    acc = EventAccumulator(str(tmp_path / run_dirs[0]))
    acc.Reload()
    tags = {"FLAME/Admitted", "FLAME/Corrupt_Admitted", "FLAME/Clip_Bound", "FLAME/Noise_Std"}
    assert tags <= set(acc.Tags()["scalars"])
    for t in tags:
        assert [e.step for e in acc.Scalars(t)] == [1, 2]


def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="fmnist", synthetic=800, synthetic_val=200, num_agents=5, local_ep=1, bs=64, device="cpu", num_corrupt=1,
                poison_frac=0.5, aggr="flame", robustLR_threshold=2, log_dir="", seed=5, trainer="torch", flame_lambda=0.01)
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


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
    assert second.aggregator.last_admitted == full.aggregator.last_admitted
    assert second.aggregator.last_flame == full.aggregator.last_flame
    for e in (full, first, second):
        e.close()
