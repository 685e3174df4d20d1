"""FoolsGold aggregation (``--aggr foolsgold``) on CPU: the weights against a numpy transcription of the authors' ``foolsgold()`` and against the
rules that define its divisions by zero, the history against the fp32 statement over engine rounds, constructed rounds (sybils, every weight 1,
nobody weighted), composition with ``--select``, ``--server_clip`` and ``--attack_boost``, 2-rank gloo runs on both transports, checkpoints
(bitwise resume, 1 rank -> 2 ranks, a checkpoint without history), options, logging, a CLI run and the memory refusal."""
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


# ---- the weights --------------------------------------------------------------------------------------------------------------
def _authors_foolsgold(G):
    """The authors' released ``foolsgold(grads)`` (Fung et al., RAID 2020) line by line, on the cosines ``G_ij / sqrt(G_ii G_jj)`` of the
    Gram matrix ``G`` in place of sklearn's ``cosine_similarity(grads)`` (a zero vector has cosine 0 with everything, itself included, as
    there; a nonzero vector's cosine with itself is taken as exactly 1, which sklearn gives up to rounding)."""
    n_clients = G.shape[0]
    q = np.diag(G)
    outer = np.sqrt(np.outer(q, q))
    cs = np.where(outer > 0, G / np.where(outer > 0, outer, 1.0), 0.0)
    np.fill_diagonal(cs, np.where(q > 0, 1.0, 0.0))
    cs = cs - np.eye(n_clients)
    maxcs = np.max(cs, axis=1)
    # pardoning
    for i in range(n_clients):
        for j in range(n_clients):
            if i == j:
                continue
            if maxcs[i] < maxcs[j]:
                cs[i][j] = cs[i][j] * maxcs[i] / maxcs[j]
    wv = 1 - (np.max(cs, axis=1))
    wv[wv > 1] = 1
    wv[wv < 0] = 0
    # rescale so that the max value is 1
    wv = wv / np.max(wv)
    wv[(wv == 1)] = .99
    # logit function
    wv = (np.log(wv / (1 - wv)) + .5)
    wv[(np.isinf(wv) + wv > 1)] = 1
    wv[(wv < 0)] = 0
    return wv


def _random_gram(rng, against=0):
    K = int(rng.integers(2 + against, 30))
    d = int(rng.integers(K, 4 * K + 8))
    X = rng.standard_normal((K, d)) + rng.uniform(0.2, 1.5) * rng.standard_normal(d)       # a shared direction: positive cosines
    b = int(rng.integers(0, K // 2 + 1))
    X[:b] = X[0] + rng.uniform(0, 0.3) * rng.standard_normal((b, d))                     # a near-sybil block
    for k in range(K - against, K):                                                       # candidates pointing against everyone else
        X[k] = -X[:K - against].mean(axis=0) + rng.uniform(0, 0.2) * rng.standard_normal(d)
    G = X @ X.T
    return np.triu(G) + np.triu(G, 1).T


def test_weights_equal_the_authors_function():
    """On finite Gram matrices of distinct updates the authors' function divides by no zero (its row maxima include the diagonal 0, so a
    pardoning divisor is v_j > v_i >= 0), and the weights equal it bit for bit -- including candidates whose every cosine is negative."""
    rng = np.random.default_rng(11)
    checked = pardoned = negative = 0
    for t in range(600):
        G = _random_gram(rng, against=t % 3)
        K = G.shape[0]
        cs = G / np.sqrt(np.outer(np.diag(G), np.diag(G)))
        v = np.where(~np.eye(K, dtype=bool), cs, -np.inf).max(axis=1)
        want = _authors_foolsgold(G)
        got = ops.foolsgold_weights(torch.from_numpy(G))
        assert got.dtype == np.float64 and np.array_equal(got, want), (got, want)
        checked += 1
        pardoned += int((v[:, None] < v[None, :]).any())
        negative += int((v < 0).any())
    assert checked == 600 and pardoned >= 500 and negative >= 150     # pardoning (both ways: v_i < v_j and v_j < v_i), anti-correlated candidates


def test_a_candidate_against_everyone_keeps_its_weight():
    """A candidate whose every cosine is negative has v = 0: the pardoning factor v_i / v_j is 0, not negative, so its cosines are not
    turned positive and it is not zeroed for being anti-correlated with everyone."""
    G = np.array([[1.0, 0.05, -0.5], [0.05, 1.0, -0.5], [-0.5, -0.5, 1.0]])
    assert ops.foolsgold_weights(G).tolist() == [1.0, 1.0, 1.0]
    np.testing.assert_array_equal(ops.foolsgold_weights(G), _authors_foolsgold(G))
    G = np.array([[1.0, 0.6, -0.5, 0.1], [0.6, 1.0, -0.5, 0.2], [-0.5, -0.5, 1.0, -0.1], [0.1, 0.2, -0.1, 1.0]])
    alpha = ops.foolsgold_weights(G)
    np.testing.assert_array_equal(alpha, _authors_foolsgold(G))
    assert alpha[2] == 1.0 and alpha[0] < 1.0


def test_weight_edge_cases():
    assert ops.foolsgold_weights(np.array([[4.0]])).tolist() == [1.0]              # one candidate: v = 0
    assert ops.foolsgold_weights(np.array([[0.0]])).tolist() == [1.0]              # ... also with a zero history
    assert ops.foolsgold_weights(np.ones((4, 4))).tolist() == [0.0] * 4            # all duplicates: max wv = 0, every alpha 0
    # a zero-norm history has cosine 0 with everyone: wv = 1 for it (the authors' function agrees)
    X = np.array([[1.0, 1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 0.0]])
    G = X @ X.T
    np.testing.assert_array_equal(ops.foolsgold_weights(G), _authors_foolsgold(G))
    alpha = ops.foolsgold_weights(G)
    assert alpha.tolist() == [0.0, 0.0, 1.0]                                       # cos_01 = 0.71: wv 0.29 of the zero row's 1
    # every cosine of candidate 0 negative, the best of the others 0: v = 0 for all three, no pardoning (the authors' function agrees)
    C = np.array([[1.0, -0.5, -0.2], [-0.5, 1.0, 0.0], [-0.2, 0.0, 1.0]])
    assert ops.foolsgold_weights(C).tolist() == [1.0, 1.0, 1.0]
    np.testing.assert_array_equal(ops.foolsgold_weights(C), _authors_foolsgold(C))
    # non-finite G_kk: alpha_k = 0 and its cosines count as 0, exactly as a zero history would for the others
    rng = np.random.default_rng(2)
    for bad in (np.inf, np.nan):
        for _ in range(20):
            G = _random_gram(rng)
            k = int(rng.integers(0, G.shape[0]))
            Gz, Gb = G.copy(), G.copy()
            Gz[k, :] = Gz[:, k] = 0.0
            Gb[k, :] = Gb[:, k] = bad
            a, z = ops.foolsgold_weights(Gb), ops.foolsgold_weights(Gz)
            assert a[k] == 0.0 and np.array_equal(np.delete(a, k), np.delete(z, k))
    assert np.all(np.isfinite(ops.foolsgold_weights(np.full((3, 3), np.nan))))


# ---- constructed rounds ---------------------------------------------------------------------------------------------------------
N, NV = 256, 240


def _disjoint_round(g, sybils, honest, seed):
    """Parameters of the sybils (one shared update on block 0) and honest agents (each on a block of its own) around ``g``: updates with
    disjoint supports, so every cosine between different blocks is exactly 0."""
    gen = torch.Generator().manual_seed(seed)
    blk = NV // (len(honest) + 1)
    ws = {}
    shared = torch.zeros(N)
    shared[:blk] = torch.randn(blk, generator=gen)
    for a in sybils:
        ws[a] = g + shared
    for b, a in enumerate(honest, 1):
        u = torch.zeros(N)
        u[b * blk:(b + 1) * blk] = torch.randn(blk, generator=gen)
        u[NV:] = torch.randn(N - NV, generator=gen)                     # the BatchNorm tail has no history
        ws[a] = g + u
    return dict(sorted(ws.items()))


@pytest.mark.parametrize("theta", [0, 2])
def test_sybils_get_zero_weight_and_the_round_is_avg_over_the_honest(theta):
    sizes = {i: 40 + 9 * i for i in range(7)}
    fg = Aggregation(sizes, N, None, make_args(num_agents=7, num_corrupt=3, aggr="foolsgold", robustLR_threshold=theta))
    avg = Aggregation(sizes, N, None, make_args(num_agents=7, num_corrupt=3, aggr="avg", robustLR_threshold=theta))
    g = torch.randn(N, generator=torch.Generator().manual_seed(0))
    wf, wa = g.clone(), g.clone()
    for rnd in (1, 2, 3):
        ws = _disjoint_round(wf, [0, 1, 2], [3, 4, 5, 6], rnd)                 # wf == wa: the same parameters for both
        honest = {a: w.clone() for a, w in ws.items() if a >= 3}
        fg.aggregate_updates(wf, ws, rnd, n_vote=NV)
        avg.aggregate_updates(wa, honest, rnd, n_vote=NV)
        assert fg.last_admitted == [3, 4, 5, 6]
        assert fg.last_foolsgold == {"FoolsGold/Avg_Honest_Weight": 1.0, "FoolsGold/Avg_Corrupt_Weight": 0.0, "FoolsGold/Admitted": 4}
        assert torch.equal(wf, wa), rnd
    assert torch.equal(fg.history[0], fg.history[1]) and fg.history[:, :NV].shape == (7, NV)


def test_every_weight_one_is_avg_bit_for_bit():
    sizes = {i: 40 + 9 * i for i in range(5)}
    for server_opt in ("sgd", "adam"):
        fg = Aggregation(sizes, N, None, make_args(num_agents=5, aggr="foolsgold", robustLR_threshold=2, server_opt=server_opt, server_lr=0.1))
        avg = Aggregation(sizes, N, None, make_args(num_agents=5, aggr="avg", robustLR_threshold=2, server_opt=server_opt, server_lr=0.1))
        wf = torch.randn(N, generator=torch.Generator().manual_seed(1))
        wa = wf.clone()
        for rnd in (1, 2):
            ws = _disjoint_round(wf, [], [0, 1, 2, 3, 4], 10 + rnd)
            fg.aggregate_updates(wf, ws, rnd, n_vote=NV)
            avg.aggregate_updates(wa, {a: w.clone() for a, w in ws.items()}, rnd, n_vote=NV)
            assert fg.last_foolsgold["FoolsGold/Admitted"] == 5 and fg.last_foolsgold["FoolsGold/Avg_Corrupt_Weight"] is None
            assert torch.equal(wf, wa), (server_opt, rnd)


def test_nobody_weighted_is_zero_plus_noise():
    K = 4
    a = make_args(num_agents=K, aggr="foolsgold", noise=0.5, clip=0.2, seed=9)
    agg = Aggregation({i: 10 + i for i in range(K)}, N, None, a)
    g = torch.randn(N, generator=torch.Generator().manual_seed(3))
    u = torch.randn(N, generator=torch.Generator().manual_seed(4))
    w = g.clone()
    agg.aggregate_updates(w, {i: g + u for i in range(K)}, 5, n_vote=NV)
    assert agg.last_admitted == [] and agg.last_foolsgold["FoolsGold/Admitted"] == 0
    gen = torch.Generator().manual_seed(9 * 1000003 + 5)
    noise = torch.randn(N, generator=gen, dtype=torch.float64) * (0.5 * 0.2)
    noise[NV:] = 0
    assert torch.equal(w, (g.double() + noise).float())


# ---- the history over engine rounds, with the attackers ------------------------------------------------------------------------
def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="fmnist", synthetic=960, synthetic_val=200, num_agents=12, agent_frac=0.5, local_ep=1, bs=64, device="cpu",
                num_corrupt=2, poison_frac=0.5, aggr="foolsgold", log_dir="", seed=5, trainer="torch")
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def _capture(eng):
    """Wrap the engine's server step to record (participants, w_global, slots) of every round."""
    seen, orig = [], eng.aggregator.aggregate_slots

    def aggregate_slots(participants, rnd):
        ws = [w.clone() for w in eng.fused.gather_participants(len(participants))]       # collective across ranks
        seen.append((list(participants), eng.fused.w_global.clone(), ws))
        orig(participants, rnd)
    eng.aggregator.aggregate_slots = aggregate_slots
    return seen


def test_history_equals_the_fp32_statement_over_engine_rounds():
    eng = _engine(attack_boost=5.0, rounds=3)
    seen = _capture(eng)
    eng.fit()
    nv = eng.layout.n_vote
    H = torch.zeros(12, nv)
    for participants, wg, slots in seen:
        for a, w in zip(participants, slots):
            H[a] = H[a] + (w[:nv] - wg[:nv])                             # fp32: one rounding per operation
    assert torch.equal(eng.fused.history, H)
    sampled = {a for p, _, _ in seen for a in p}
    never = [a for a in range(12) if a not in sampled]
    assert never and all(not eng.fused.history[a].any() for a in never)
    assert eng.aggregator.last_foolsgold["FoolsGold/Admitted"] >= 1
    eng.close()


def test_multikrum_candidates_only_and_server_clip_on_the_step():
    K = 7
    sizes = {i: 30 + 5 * i for i in range(K)}
    a = make_args(num_agents=K, num_corrupt=1, aggr="foolsgold", select="multikrum", select_f=1, robustLR_threshold=2, server_clip=True,
                  clip=0.5)
    agg = Aggregation(sizes, N, None, a)
    g = torch.randn(N, generator=torch.Generator().manual_seed(6))
    gen = torch.Generator().manual_seed(7)
    common = torch.randn(N, generator=gen)
    ws = {i: g + 0.1 * (common + torch.randn(N, generator=gen)) for i in range(K)}
    ws[0] = g - 0.3 * common                                            # against everyone: rejected by multikrum even after clipping
    w = g.clone()
    agg.aggregate_updates(w, ws, 1, n_vote=NV)
    clip = (1.0 / torch.clamp(ops.update_norms(g, list(ws.values()), NV) / a.clip, min=1.0)).float()
    cand = ops.krum_select(ops.sqdist_statement(list(ws.values()), 0, NV, g, clip), list(range(K)), a.select_f, a.select_m)
    assert 0 not in cand and not agg.history[0].any()                   # only the candidates enter the history
    for i in cand:
        assert torch.equal(agg.history[i], ws[i][:NV] - g[:NV])         # unclipped updates
    alpha = ops.foolsgold_weights(ops.history_gram_statement([agg.history[i] for i in cand], 0, NV))
    members = [i for i, al in zip(cand, alpha) if al > 0]
    assert agg.last_admitted == members
    norms = ops.update_norms(g, [ws[i] for i in members], NV)
    scales = (1.0 / torch.clamp(norms / a.clip, min=1.0)).float()
    ref, _ = ops.aggregate_oracle(g, [ws[i] for i in members], [float(al) * sizes[i] for i, al in zip(cand, alpha) if al > 0], "avg",
                                  2, a.server_lr, None, NV, scales.tolist(), None,
                                  sum(float(al) * sizes[i] for i, al in zip(cand, alpha) if al > 0))
    assert torch.equal(w, ref)


# ---- 2 ranks over gloo ---------------------------------------------------------------------------------------------------------
def _gloo_case(rnd):
    g = torch.randn(1024, generator=torch.Generator().manual_seed(50))
    gen = torch.Generator().manual_seed(rnd)
    evil = torch.randn(1024, generator=gen)
    ids = [int(i) for i in torch.randperm(10, generator=gen)[:7]]
    ws = [g + 0.01 * ((evil if a < 3 else 0) + torch.randn(1024, generator=gen)) for a in ids]
    return g, ids, ws


def _transport_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.aggregation import Aggregation as Agg
    from rlr_b200.options import make_args as mk
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed("cpu")
    out = {}
    for select in ("none", "multikrum"):
        for transport in ("gather", "reduce"):
            fa = FusedAggregator(ctx, 1024, 1000, 4, "gloo", transport=transport, history_agents=10)
            agg = Agg({i: 10 + 3 * i for i in range(10)}, 1024, None,
                      mk(num_agents=10, agent_frac=0.7, num_corrupt=3, aggr="foolsgold", robustLR_threshold=2, select=select,
                                select_f=1 if select != "none" else -1), fused=fa)
            res = []
            w = None
            for rnd in (1, 2, 3):
                g, ids, ws = _gloo_case(rnd)
                fa.w_global.copy_(g if w is None else w)
                for j, wj in enumerate(ws):
                    r, s = fa.slot_owner(j)
                    if r == rank:
                        fa.slots[s].copy_(wj - g + fa.w_global)
                agg.aggregate_slots(ids, rnd)
                w = fa.w_global.clone()
                res.append((w, dict(agg.last_foolsgold), list(agg.last_admitted)))
            out[(select, transport)] = (res, fa.history.clone(), fa.foolsgold_history())       # every rank's table; the main rank's copy
            fa.close()
    torch.save(out, os.path.join(outdir, f"t{rank}.pt"))
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_transports_match_the_dict_form(tmp_path):
    world = 2
    mp.spawn(_transport_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"t{r}.pt") for r in range(world)]
    for select in ("none", "multikrum"):
        dict_form = Aggregation({i: 10 + 3 * i for i in range(10)}, 1024, None,
                                make_args(num_agents=10, agent_frac=0.7, num_corrupt=3, aggr="foolsgold", robustLR_threshold=2, select=select,
                                select_f=1 if select != "none" else -1))
        w, want = None, []
        for rnd in (1, 2, 3):
            g, ids, ws = _gloo_case(rnd)
            w = g.clone() if w is None else w
            dict_form.aggregate_updates(w, {a: wj - g + w for a, wj in zip(ids, ws)}, rnd, n_vote=1000)
            want.append((w.clone(), dict(dict_form.last_foolsgold), list(dict_form.last_admitted)))
        assert any(last["FoolsGold/Avg_Corrupt_Weight"] < last["FoolsGold/Avg_Honest_Weight"] for _, last, _ in want)
        for o in outs:
            for transport in ("gather", "reduce"):
                res, hist, host = o[(select, transport)]
                assert torch.equal(hist, dict_form.history), (select, transport)
                assert (torch.equal(host, hist) if o is outs[0] else host is None), (select, transport)
                for rnd, ((w_, last, adm), (ww, wl, wa)) in enumerate(zip(res, want)):
                    assert last == wl and adm == wa, (select, transport, rnd)
                    assert torch.equal(w_, outs[0][(select, transport)][0][rnd][0])
                    if transport == "gather":
                        assert torch.equal(w_, ww), (select, rnd)
                    else:
                        torch.testing.assert_close(w_, ww, rtol=1e-6, atol=1e-6)


def _sharded_worker(rank, world, port, outdir):
    """The fused multi-GPU path's history layout on gloo ranks: each rank holds the columns of its coordinate slice below n_vote (the
    last rank's slice lies past n_vote: no columns), loads them from a full table and gathers the table back in several chunks."""
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed("cpu")
    n, nv, A = 1024, 600, 10
    fa = FusedAggregator(ctx, n, nv, 2, "gloo")
    fa.sharded, fa.per = True, (n // 4 + world - 1) // world * 4           # the slices FusedAggregator gives the fused path
    fa.begin = min(n, rank * fa.per)
    fa.end = min(n, fa.begin + fa.per)
    fa._alloc_history(A)
    full = torch.randn(A, nv, generator=torch.Generator().manual_seed(4))
    fa.load_foolsgold_history(full)
    local = fa.history.clone()
    host = fa.foolsgold_history(chunk_bytes=4 * fa.per * world * 3)       # 3 rows per chunk: 4 chunks, the last one partial
    torch.save(dict(lo=fa.hist_lo, hi=fa.hist_hi, local=local, host=host, full=full), os.path.join(outdir, f"s{rank}.pt"))
    fa.close()
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_sharded_history_layout_loads_and_gathers_the_full_table(tmp_path):
    world = 3
    mp.spawn(_sharded_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"s{r}.pt") for r in range(world)]
    full = outs[0]["full"]
    assert [(o["lo"], o["hi"]) for o in outs] == [(0, 344), (344, 600), (688, 688)]
    for o in outs:
        assert torch.equal(o["local"], full[:, o["lo"]:o["hi"]])
    assert torch.equal(outs[0]["host"], full) and outs[1]["host"] is None and outs[2]["host"] is None


# ---- checkpoints ---------------------------------------------------------------------------------------------------------------
def test_resume_equals_an_uninterrupted_run(tmp_path):
    full = _engine(rounds=4)
    full.fit()
    ck = str(tmp_path / "ck.pt")
    first = _engine(rounds=2, checkpoint=ck)
    first.fit()
    saved = torch.load(ck, weights_only=False)["extra"]["foolsgold_history"]
    assert saved.dtype == torch.float32 and saved.shape == (12, first.layout.n_vote) and torch.equal(saved, first.fused.history)
    second = _engine(rounds=4, resume=ck)
    assert second.start_round == 3 and torch.equal(second.fused.history, saved)
    second.fit()
    assert torch.equal(second.w_global, full.w_global) and torch.equal(second.fused.history, full.fused.history)
    assert second.aggregator.last_foolsgold == full.aggregator.last_foolsgold
    for e in (full, first, second):
        e.close()


def test_checkpoint_without_history_is_rejected(tmp_path):
    ck = str(tmp_path / "avg.pt")
    _engine(aggr="avg", rounds=1, checkpoint=ck).fit()
    with pytest.raises(ValueError, match="no FoolsGold history"):
        _engine(rounds=2, resume=ck)


def _resume_worker(rank, world, port, outdir, ck):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    eng = _engine(rounds=4, resume=ck)
    loaded = eng.fused.history.clone()
    seen = _capture(eng)
    eng.fit()
    torch.save(dict(loaded=loaded, history=eng.fused.history.clone(), w=eng.w_global.clone(), seen=seen if rank == 0 else None,
                    admitted=eng.aggregator.last_admitted, backend=eng.fused.backend), os.path.join(outdir, f"r{rank}.pt"))
    eng.close()
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_one_rank_checkpoint_resumes_at_two_ranks(tmp_path):
    ck = str(tmp_path / "ck.pt")
    first = _engine(rounds=2, checkpoint=ck)
    first.fit()
    saved = first.fused.history.clone()
    first.close()
    mp.spawn(_resume_worker, args=(2, _free_port(), str(tmp_path), ck), nprocs=2, join=True)
    outs = [torch.load(tmp_path / f"r{r}.pt", weights_only=False) for r in range(2)]
    assert outs[0]["backend"] == "gloo"
    for o in outs:
        assert torch.equal(o["loaded"], saved)
        assert torch.equal(o["w"], outs[0]["w"]) and torch.equal(o["history"], outs[0]["history"]) and o["admitted"] == outs[0]["admitted"]
    # rounds 3-4 folded into the resumed history: the fp32 statement over the updates both ranks submitted
    H = saved.clone()
    nv = H.shape[1]
    for participants, wg, ws in outs[0]["seen"]:
        for a, w in zip(participants, ws):
            H[a] = H[a] + (w[:nv] - wg[:nv])
    assert torch.equal(outs[0]["history"], H)


# ---- options, logging, CLI, memory ---------------------------------------------------------------------------------------------
def test_options_and_banner(capsys):
    from rlr_b200.options import AGGREGATORS, args_parser, build_parser, finalize_args, print_exp_details
    assert "foolsgold" in AGGREGATORS and "foolsgold" in build_parser().format_help()
    a = finalize_args(args_parser(["--aggr", "foolsgold", "--select", "multikrum", "--num_agents", "10", "--num_corrupt", "2",
                                   "--server_clip", "--clip", "1.0", "--noise", "0.1", "--attack_boost", "3"]))
    assert a.aggr == "foolsgold" and a.select == "multikrum" and a.server_clip and a.attack_boost == 3.0
    print_exp_details(a)
    assert "Aggregation Function: foolsgold" in capsys.readouterr().out


def test_federated_py_writes_the_foolsgold_fields_and_tags(tmp_path):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "federated.py", "--data=fmnist", "--local_ep=1", "--bs=64", "--num_agents=4", "--rounds=2",
                        "--num_corrupt=1", "--poison_frac=0.5", "--synthetic=400", "--synthetic_val=80", "--aggr=foolsgold",
                        "--agent_frac=0.5", f"--log_dir={tmp_path}", "--device=cpu"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "Aggregation Function: foolsgold" in r.stdout
    run_dirs = os.listdir(tmp_path)
    assert len(run_dirs) == 1
    recs = [json.loads(l) for l in open(tmp_path / run_dirs[0] / "metrics.jsonl")]
    assert [rec["round"] for rec in recs] == [1, 2]
    for rec in recs:
        assert {"foolsgold_avg_honest", "foolsgold_avg_corrupt", "foolsgold_admitted"} <= set(rec)
        assert 0 <= rec["foolsgold_admitted"] <= 2
        for k in ("foolsgold_avg_honest", "foolsgold_avg_corrupt"):
            assert rec[k] is None or 0.0 <= rec[k] <= 1.0
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    acc = EventAccumulator(str(tmp_path / run_dirs[0]))
    acc.Reload()
    tags = set(acc.Tags()["scalars"])
    assert "FoolsGold/Admitted" in tags and [e.step for e in acc.Scalars("FoolsGold/Admitted")] == [1, 2]
    for t, key in (("FoolsGold/Avg_Honest_Weight", "foolsgold_avg_honest"), ("FoolsGold/Avg_Corrupt_Weight", "foolsgold_avg_corrupt")):
        steps = [rec["round"] for rec in recs if rec[key] is not None]
        assert (t in tags) == bool(steps) and (not steps or [e.step for e in acc.Scalars(t)] == steps)


def test_diagnostics_cover_every_participant():
    eng = _engine(rounds=1, diagnostics=True)
    eng.fit()
    assert set(eng.aggregator.last_norms) <= {"Norms/Avg_Honest_L2", "Norms/Avg_Corrupt_L2"} and eng.aggregator.last_norms
    eng.close()


def test_memory_refusal_names_the_bytes_and_num_agents():
    from rlr_b200.parallel.fused_agg import check_history_memory
    assert check_history_memory(3383, 1200128, 1 << 40) == 4 * 3383 * 1200128
    with pytest.raises(ValueError) as e:
        check_history_memory(3383, 1200128, 8 << 30)
    msg = str(e.value)
    assert str(4 * 3383 * 1200128) in msg and "--num_agents 3383" in msg and str(8 << 30) in msg
