"""FLTrust aggregation (``--aggr fltrust``) on CPU: option validation and the banner, the fp64 trust statistics against brute-force
numpy, trust scores and rescaling on constructed cases, the server step against the oracle on the trusted set (RLR, adam, multikrum),
the root set, engine runs (root job, JSONL fields, reproducibility, resume) and 2-rank gloo runs on both transports."""
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
from rlr_b200.engine import FLEngine, draw_root_set
from rlr_b200.options import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- options ------------------------------------------------------------------------------------------------------------
def test_defaults_and_server_lr():
    a = make_args(aggr="fltrust", server_lr=0.3)
    assert a.root_size == 100 and a.server_lr == 1.0              # the plain sgd step keeps the forced server_lr = 1
    assert make_args(aggr="fltrust", root_size=7).root_size == 7
    assert make_args().root_size is None


@pytest.mark.parametrize("kw", [
    dict(aggr="fltrust", server_clip=True, clip=1.0),
    dict(aggr="avg", root_size=100),
    dict(aggr="comed", root_size=5),
    dict(aggr="fltrust", root_size=0),
    dict(aggr="fltrust", root_size=-3),
])
def test_fltrust_options_rejected(kw):
    with pytest.raises(ValueError):
        make_args(**kw)


def test_banner_line(capsys):
    from rlr_b200.options import print_exp_details
    print_exp_details(make_args())
    assert "Root set" not in capsys.readouterr().out
    print_exp_details(make_args(aggr="fltrust", root_size=64))
    out = capsys.readouterr().out
    assert "Root set: 64" in out and "Aggregation Function: fltrust" in out


# ---- statistics ---------------------------------------------------------------------------------------------------------
def _numpy_stats(ws, root, g, n_vote):
    g = np.asarray(g[:n_vote], dtype=np.float64)
    d0 = np.asarray(root[:n_vote], dtype=np.float64) - g
    xs = [np.asarray(w[:n_vote], dtype=np.float64) - g for w in ws]
    d = [math.fsum(float(a) * float(b) for a, b in zip(x, d0)) for x in xs]
    q = [math.fsum(float(a) * float(a) for a in x) for x in xs]
    return np.array(d + q + [math.fsum(float(a) * float(a) for a in d0)])


@pytest.mark.parametrize("K,n,n_vote", [(1, 16, 16), (5, 64, 48), (9, 200, 180)])
def test_trust_statement_matches_numpy(K, n, n_vote):
    gen = torch.Generator().manual_seed(K * n)
    g = torch.randn(n, generator=gen)
    root = g + 0.1 * torch.randn(n, generator=gen)
    ws = [g + 0.1 * (k + 1) * torch.randn(n, generator=gen) for k in range(K)]
    for w in (*ws, root):
        w[n_vote:] += 1e3                                               # tail coordinates do not count
    s = ops.trust_stats(ws, root, g, n_vote)
    assert s.dtype == torch.float64 and s.shape == (2 * K + 1,)
    assert torch.equal(s, ops.trust_statement(ws, root, g, 0, n_vote))
    np.testing.assert_allclose(s.numpy(), _numpy_stats(ws, root, g, n_vote), rtol=1e-12, atol=1e-12)


def _weights(ws, root, g, n_vote=None):
    K = len(ws)
    s = ops.trust_stats(ws, root, g, n_vote)
    return ops.fltrust_weights(s[:K], s[K:2 * K], s[2 * K])


def test_constructed_trust_scores_and_scales():
    n = 64
    g = torch.zeros(n)
    d0 = torch.randn(n, generator=torch.Generator().manual_seed(2))
    orth = torch.zeros(n)
    orth[0], orth[1] = d0[1], -d0[0]                                   # exactly orthogonal to Δ0
    ws = [0.5 * d0, 2.0 * d0, -d0, orth, 100.0 * d0, d0, torch.zeros(n)]
    ts, sc, adm = _weights(ws, d0, g)
    assert ts.dtype == torch.float64 and sc.dtype == torch.float32
    for k, c in ((0, 0.5), (1, 2.0), (4, 100.0), (5, 1.0)):
        assert abs(float(ts[k]) - 1.0) < 1e-12 and abs(float(sc[k]) - 1.0 / c) <= 1e-6 / c
    assert float(ts[2]) == 0.0 and float(ts[3]) == 0.0                 # opposite and orthogonal: no weight
    assert float(ts[6]) == 0.0 and float(sc[6]) == 1.0                 # a zero update: no weight, scale 1
    assert adm == [0, 1, 4, 5]
    # a boosted copy contributes exactly what Δ0 itself does
    torch.testing.assert_close(ws[4] * sc[4], ws[5] * sc[5], rtol=1e-6, atol=0)
    ts0, sc0, adm0 = ops.fltrust_weights([1.0, -1.0], [1.0, 1.0], 0.0)   # a zero root update trusts nobody
    assert adm0 == [] and ts0.tolist() == [0.0, 0.0] and sc0.tolist() == [0.0, 0.0]
    ts1, _, adm1 = ops.fltrust_weights([float("nan")], [1.0], 1.0)
    assert adm1 == [] and ts1.tolist() == [0.0]


# ---- the server step ----------------------------------------------------------------------------------------------------
def _round(K, n, seed, flip=(1,)):
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(n, generator=gen)
    d0 = 0.05 * torch.randn(n, generator=gen)
    root = g + d0
    ws = [g + d0 * (0.5 + 0.3 * k) + 0.05 * torch.randn(n, generator=gen) for k in range(K)]
    for k in flip:
        ws[k] = g - (ws[k] - g)                                         # points away from the root update: distrusted
    return g, root, ws


def _oracle(g, root, ws, ids, nv, theta, server_lr, opt=None, select_keep=None):
    K = len(ws)
    s = ops.trust_statement(ws, root, g, 0, nv)
    ts, sc, adm = ops.fltrust_weights(s[:K], s[K:2 * K], s[2 * K])
    if select_keep is not None:
        adm = [j for j in adm if j in select_keep]
    ref, _ = ops.aggregate_oracle(g, [ws[j] for j in adm], [float(ts[j]) for j in adm], "avg", theta, server_lr, None, nv,
                                  [float(sc[j]) for j in adm], opt)
    return ref, [ids[j] for j in adm]


@pytest.mark.parametrize("theta,server_opt", [(0, "sgd"), (2, "sgd"), (0, "adam"), (2, "adam")])
def test_aggregate_updates_equals_the_oracle_on_the_trusted_set(theta, server_opt):
    K, n, nv = 6, 512, 480
    g, root, ws = _round(K, n, 7, flip=(1, 4))
    a = make_args(num_agents=K, num_corrupt=2, aggr="fltrust", robustLR_threshold=theta, server_opt=server_opt, server_lr=0.05)
    sizes = {i: 100 + 13 * i for i in range(K)}
    agg = Aggregation(sizes, n, None, a)
    opt = ops.ServerOptState(server_opt, n, beta1=a.server_beta1, beta2=a.server_beta2, tau=a.server_tau)
    wg = g.clone()
    for rnd in (1, 2):                                                   # two rounds: the optimizer state carries over
        ref, adm = _oracle(wg, root, ws, list(range(K)), nv, theta, a.server_lr, opt)
        agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, rnd, n_vote=nv, root_params=root)
        torch.testing.assert_close(wg, ref, rtol=0, atol=1e-6)
        assert agg.last_admitted == adm and agg.last_trust["Trust/Admitted"] == len(adm)
        if rnd == 1:
            assert adm == [0, 2, 3, 5]
            assert agg.last_trust["Trust/Avg_Corrupt"] > 0 and agg.last_trust["Trust/Avg_Honest"] > 0


def test_aggregate_updates_needs_the_root():
    g, root, ws = _round(3, 64, 1)
    agg = Aggregation({i: 1 for i in range(3)}, 64, None, make_args(num_agents=3, aggr="fltrust"))
    with pytest.raises(ValueError, match="root"):
        agg.aggregate_updates(g.clone(), {i: ws[i] for i in range(3)}, 1)


def test_multikrum_then_fltrust():
    K, n, nv = 7, 256, 240
    g, root, ws = _round(K, n, 8, flip=(3,))
    ws[0] = ws[0] + 3.0                                                  # far from everyone: rejected by multikrum first
    a = make_args(num_agents=K, num_corrupt=1, aggr="fltrust", robustLR_threshold=2, select="multikrum")
    assert (a.select_f, a.select_m) == (1, 6)
    agg = Aggregation({i: 50 + 7 * i for i in range(K)}, n, None, a)
    wg = g.clone()
    agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv, root_params=root)
    ref, adm = _oracle(g, root, ws, list(range(K)), nv, 2, a.server_lr, select_keep=list(range(1, K)))
    assert agg.last_select["Select/Corrupt_Admitted"] == 0
    assert agg.last_admitted == adm == [1, 2, 4, 5, 6]
    torch.testing.assert_close(wg, ref, rtol=0, atol=1e-6)


@pytest.mark.parametrize("theta", [0, 2])
def test_every_participant_distrusted_keeps_w_global(theta):
    K, n, nv = 5, 256, 224
    g, root, ws = _round(K, n, 9, flip=range(K))
    a = make_args(num_agents=K, aggr="fltrust", robustLR_threshold=theta)
    agg = Aggregation({i: 10 for i in range(K)}, n, None, a)
    wg = g.clone()
    agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv, root_params=root)
    assert agg.last_admitted == [] and agg.last_trust["Trust/Admitted"] == 0
    assert torch.equal(wg, g)


def _local_aggregator(n, nv, slots):
    from rlr_b200.parallel import FusedAggregator, init_distributed
    return FusedAggregator(init_distributed("cpu"), n, nv, slots, "local")


@pytest.mark.parametrize("flip", [(1,), (), tuple(range(5))])
def test_slots_form_equals_the_dict_form(flip):
    K, n, nv = 5, 256, 240
    g, root, ws = _round(K, n, 10, flip=flip)
    sizes = {i: 50 + 7 * i for i in range(K)}
    a = make_args(num_agents=K, num_corrupt=1, aggr="fltrust", robustLR_threshold=2)
    fa = _local_aggregator(n, nv, K + 1)
    fa.w_global.copy_(g)
    for j in range(K):
        fa.slots[j].copy_(ws[j])
    fa.slots[K].copy_(root)                                              # the root job is position K
    agg = Aggregation(sizes, n, None, a, fused=fa)
    agg.aggregate_slots(list(range(K)), 1)
    dict_form = Aggregation(sizes, n, None, a)
    wg = g.clone()
    dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv, root_params=root)
    assert agg.last_admitted == dict_form.last_admitted
    assert torch.equal(fa.w_global, wg)
    fa.close()


# ---- the root set ---------------------------------------------------------------------------------------------------------
def test_draw_root_set():
    r = draw_root_set(1000, [3, 5, 7], 100, 4)
    assert r.dtype == np.int64 and len(set(r.tolist())) == 100 and not {3, 5, 7} & set(r.tolist())
    assert np.array_equal(r, draw_root_set(1000, [3, 5, 7], 100, 4)) and not np.array_equal(r, draw_root_set(1000, [3, 5, 7], 100, 5))
    assert sorted(draw_root_set(10, [0, 9], 8, 1).tolist()) == list(range(1, 9))
    with pytest.raises(ValueError):
        draw_root_set(10, [0, 9], 9, 1)


def _engine(**kw):
    base = dict(data="fmnist", synthetic=1200, synthetic_val=300, num_agents=4, local_ep=1, bs=64, device="cpu", num_corrupt=1,
                poison_frac=0.5, aggr="fltrust", root_size=80, robustLR_threshold=2, log_dir="", seed=5, trainer="torch")
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


@pytest.mark.parametrize("data", ["fmnist", "cifar10"])
def test_root_set_excludes_poisoned_samples_and_is_seeded(data):
    e1, e2 = _engine(data=data, num_corrupt=2), _engine(data=data, num_corrupt=2)
    poisoned = {i for a in e1.agents for i in a.poisoned_idxs}
    root = e1.root_agent.idxs.tolist()
    assert poisoned and len(set(root)) == len(root) == 80 and not poisoned & set(root)
    assert e1.root_agent.id == 4 and not e1.root_agent.is_corrupt and e1.root_agent.poisoned_idxs == []
    assert torch.equal(e1.root_agent.idxs, e2.root_agent.idxs)
    n_clean = len(e1.train_dataset) - len(poisoned)
    everything = _engine(data=data, num_corrupt=2, root_size=n_clean)        # the whole clean set is still drawable
    assert set(everything.root_agent.idxs.tolist()) == set(range(len(e1.train_dataset))) - poisoned
    with pytest.raises(ValueError, match="root_size"):
        _engine(data=data, num_corrupt=2, root_size=n_clean + 1)
    for e in (e1, e2, everything):
        e.close()


def test_other_rules_have_no_root_job():
    e = _engine(aggr="avg", root_size=None)
    assert e.root_agent is None and e.fused.max_slots == 4
    e.close()


def test_engine_trains_the_root_job_logs_and_is_reproducible(tmp_path):
    eng = _engine(log_dir=str(tmp_path / "logs"), no_tensorboard=True, rounds=2)
    K = eng.n_part
    assert eng.fused.max_slots == K + 1
    w_start = eng.w_global.clone()
    info = eng.run_round(1)
    assert info["steps"] == sum((eng.agents[a].n_data + 63) // 64 for a in info["chosen"])      # clients only
    assert not torch.equal(eng.fused.slots[K], w_start)                  # the root job trained into position K
    root_again = eng.fused.slots[K].clone()
    eng.close()
    eng = _engine(log_dir=str(tmp_path / "logs"), no_tensorboard=True, rounds=2)
    hist = eng.fit()
    eng.close()
    run_dirs = os.listdir(tmp_path / "logs")
    recs = [json.loads(l) for d in run_dirs for l in open(tmp_path / "logs" / d / "metrics.jsonl")]
    assert [r["round"] for r in recs] == [1, 2]
    for r, h in zip(recs, hist):
        assert 0 <= r["trust_admitted"] <= K and h["trust_admitted"] == r["trust_admitted"]
        assert 0 <= r["trust_avg_honest"] <= 1 and 0 <= r["trust_avg_corrupt"] <= 1
    again = _engine(rounds=2)
    again.run_round(1)
    assert torch.equal(again.fused.slots[K], root_again)
    again.run_round(2)
    assert torch.equal(again.w_global, eng.w_global)
    again.close()


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
    for e in (full, first, second):
        e.close()


# ---- 2 ranks over gloo ---------------------------------------------------------------------------------------------------
def _engine_worker(rank, world, port, outdir, kw):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.engine import FLEngine as Engine
    from rlr_b200.options import make_args as mk
    eng = Engine(mk(**kw), verbose=False)
    admitted = []
    for r in range(1, 3):
        eng.run_round(r)
        admitted.append(list(eng.aggregator.last_admitted))
    ev = eng.evaluate(2)
    torch.save({"w": eng.w_global.clone(), "val_acc": ev["val_acc"], "admitted": admitted, "backend": eng.fused.backend},
               os.path.join(outdir, f"e{rank}.pt"))
    eng.close()
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_engine_ranks_agree_and_match_single_process(tmp_path):
    world = 2
    kw = dict(data="fmnist", synthetic=800, synthetic_val=200, num_agents=5, local_ep=1, bs=64, aggr="fltrust", root_size=64,
              log_dir="", device="cpu", robustLR_threshold=2, seed=3)
    mp.spawn(_engine_worker, args=(world, _free_port(), str(tmp_path), kw), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"e{r}.pt") for r in range(world)]
    assert outs[0]["backend"] == "gloo"
    for o in outs[1:]:
        assert torch.equal(o["w"], outs[0]["w"]) and o["val_acc"] == outs[0]["val_acc"] and o["admitted"] == outs[0]["admitted"]
    solo = FLEngine(make_args(**kw), verbose=False)            # dropout masks differ across process layouts: compare in distribution
    for r in range(1, 3):
        solo.run_round(r)
    assert abs(solo.evaluate(2)["val_acc"] - outs[0]["val_acc"]) < 0.25
    solo.close()


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
    for case, flip in CASES.items():
        g, root, ws = _round(K, n, 21, flip=flip)
        for transport in ("gather", "reduce"):
            fa = FusedAggregator(ctx, n, nv, (K + 1 + world - 1) // world, "gloo", transport=transport)
            fa.w_global.copy_(g)
            for j, w in enumerate(ws + [root]):
                r, s = fa.slot_owner(j)
                if r == rank:
                    fa.slots[s].copy_(w)
            agg = Agg({i: 10 + 3 * i for i in range(K)}, n, None, mk(num_agents=K, num_corrupt=1, aggr="fltrust", robustLR_threshold=2,
                                                                     noise=0.1, clip=0.5), fused=fa)
            agg.aggregate_slots(list(range(K)), 1)
            out[(case, transport)] = (fa.w_global.clone(), list(agg.last_admitted))
            fa.close()
    torch.save(out, os.path.join(outdir, f"t{rank}.pt"))
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_transports_match_the_dict_form(tmp_path):
    world = 2
    mp.spawn(_transport_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"t{r}.pt") for r in range(world)]
    K, n, nv = 5, 1024, 1000
    for case, flip in CASES.items():
        g, root, ws = _round(K, n, 21, flip=flip)
        a = make_args(num_agents=K, num_corrupt=1, aggr="fltrust", robustLR_threshold=2, noise=0.1, clip=0.5)
        dict_form = Aggregation({i: 10 + 3 * i for i in range(K)}, n, None, a)
        wg = g.clone()
        dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv, root_params=root)
        want = [i for i in range(K) if i not in flip]
        for o in outs:
            assert o[(case, "gather")][1] == o[(case, "reduce")][1] == dict_form.last_admitted == want, case
            assert torch.equal(o[(case, "gather")][0], wg), case                   # the gathered step is the dict form's
            torch.testing.assert_close(o[(case, "reduce")][0], wg, rtol=1e-6, atol=1e-6)
            assert torch.equal(o[(case, "reduce")][0], outs[0][(case, "reduce")][0])
