"""Krum / Multi-Krum participant selection (``--select``) on CPU: option validation and defaults, the fp64 distance statement against
brute-force numpy, Krum scores on constructed cases, the admitted-set server step, multikrum with M = K against no selection bit for
bit, the per-round JSONL fields, and a 2-rank gloo run on both transports."""
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
from rlr_b200.options import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- options ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,f,m", [
    (dict(data="fmnist", num_agents=10, num_corrupt=1), 1, 9),                              # scripts/runner.sh fmnist
    (dict(data="cifar10", num_agents=40, num_corrupt=4), 4, 36),
    (dict(data="fedemnist", num_agents=3383, agent_frac=0.01, num_corrupt=338), 4, 29),    # K = 33
    (dict(data="fmnist", num_agents=10, num_corrupt=0), 0, 10),
    (dict(data="fmnist", num_agents=10, num_corrupt=1, select_f=3, select_m=4), 3, 4),
])
def test_default_f_and_m(kw, f, m):
    a = make_args(select="multikrum", **kw)
    assert (a.select_f, a.select_m) == (f, m)
    k = make_args(select="krum", **{key: v for key, v in kw.items() if key != "select_m"})
    assert (k.select_f, k.select_m) == (f, 1)


@pytest.mark.parametrize("kw", [
    dict(select="multikrum", num_agents=4, num_corrupt=1),                  # K = 4 < 2F + 3 = 5
    dict(select="krum", num_agents=10, select_f=4),                         # 10 < 11
    dict(select="multikrum", num_agents=10, select_m=11),                   # M > K
    dict(select="multikrum", num_agents=10, select_m=-2),
    dict(select="multikrum", num_agents=10, select_m=3, robustLR_threshold=4),
    dict(select="krum", num_agents=10, robustLR_threshold=2),               # krum admits one participant
    dict(select="krum", num_agents=10, select_m=3),
    dict(select="none", select_f=1),
    dict(select="none", select_m=3),
    dict(select="multikrum", num_agents=10, select_f=-3),
    dict(select="bulyan"),
])
def test_select_options_rejected(kw):
    with pytest.raises(ValueError):
        make_args(**kw)


def test_banner_line(capsys):
    from rlr_b200.options import print_exp_details
    print_exp_details(make_args())
    assert "Selection" not in capsys.readouterr().out
    print_exp_details(make_args(select="multikrum", num_agents=10, num_corrupt=1))
    assert "Selection (F / M): multikrum (1 / 9)" in capsys.readouterr().out


# ---- distances ----------------------------------------------------------------------------------------------------------
def _numpy_sqdist(ws, g, n_vote, scales):
    x = [np.asarray(w[:n_vote], dtype=np.float64) for w in ws]
    if scales is not None:
        x = [(xi - np.asarray(g[:n_vote], dtype=np.float64)) * float(s) for xi, s in zip(x, np.asarray(scales, dtype=np.float32))]
    K = len(x)
    D = np.zeros((K, K))
    for i in range(K):
        for j in range(K):
            D[i, j] = sum((a - b) ** 2 for a, b in zip(x[i].tolist(), x[j].tolist()))
    return D


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("K,n,n_vote", [(5, 64, 48), (3, 40, 40), (9, 128, 100)])
def test_pairwise_sqdist_matches_numpy(K, n, n_vote, scaled):
    gen = torch.Generator().manual_seed(K * n + scaled)
    g = torch.randn(n, generator=gen)
    ws = [g + torch.randn(n, generator=gen) * (0.1 + k) for k in range(K)]
    ws[1] = ws[0].clone()                                             # a Sybil pair
    for w in ws:
        w[n_vote:] += 1e3                                               # tail coordinates do not count
    scales = torch.rand(K, generator=gen).float() + 0.1 if scaled else None
    D = ops.pairwise_sqdist(ws, n_vote, g if scaled else None, scales)
    assert D.dtype == torch.float64 and D.shape == (K, K)
    np.testing.assert_allclose(D.numpy(), _numpy_sqdist(ws, g, n_vote, scales), rtol=1e-12, atol=1e-12)
    assert torch.equal(D, D.T) and torch.equal(D.diagonal(), torch.zeros(K, dtype=torch.float64))
    if not scaled:
        assert D[0, 1] == 0.0


def test_pairwise_sqdist_scales_need_w_global():
    with pytest.raises(ValueError):
        ops.pairwise_sqdist([torch.zeros(4)] * 3, 4, None, [1.0, 1.0, 1.0])


# ---- Krum scores ---------------------------------------------------------------------------------------------------------
def test_multikrum_rejects_a_far_cluster_of_identical_updates():
    gen = torch.Generator().manual_seed(1)
    n, honest, bad = 200, 7, 3
    g = torch.zeros(n)
    ws = [torch.full((n,), 5.0) for _ in range(bad)] + [torch.randn(n, generator=gen) for _ in range(honest)]
    ids = list(range(len(ws)))                                        # corrupt agents have the lowest ids, as in the engine
    D = ops.pairwise_sqdist(ws, n)
    assert D[0, 1] == 0.0 and D[1, 2] == 0.0
    assert ops.krum_select(D, ids, 3, len(ws) - 3) == list(range(bad, len(ws)))
    assert ops.krum_select(D, ids, 3, 1)[0] >= bad


def test_krum_picks_the_central_honest_update():
    n = 8
    pts = [torch.eye(n)[k] for k in range(5)]                           # five unit vectors: 2 apart from each other
    pts.insert(2, torch.zeros(n))                                       # the centre: 1 from each of them
    pts.append(10.0 * torch.ones(n))                                    # an outlier
    D = ops.pairwise_sqdist(pts, n)
    assert ops.krum_select(D, list(range(len(pts))), 1, 1) == [2]


def test_ties_go_to_the_lower_id():
    ws = [torch.ones(16) for _ in range(5)]
    D = ops.pairwise_sqdist(ws, 16)
    ids = [7, 3, 9, 1, 5]
    assert ops.krum_select(D, ids, 1, 1) == [3]                          # id 1
    assert ops.krum_select(D, ids, 1, 2) == [1, 3]                       # ids 3 and 1, positions ascending
    assert ops.krum_select(D, ids, 1, 5) == [0, 1, 2, 3, 4]


def test_krum_scores_sum_the_k_minus_f_minus_2_nearest():
    D = torch.tensor([[0, 1, 4, 9, 16], [1, 0, 1, 4, 9], [4, 1, 0, 1, 4], [9, 4, 1, 0, 1], [16, 9, 4, 1, 0]], dtype=torch.float64)
    # f = 1: K - f - 2 = 2 nearest -> scores 5, 2, 2, 2, 5; m = 3 keeps positions 1, 2, 3; m = 1 keeps the lowest id of the ties
    assert ops.krum_select(D, [0, 1, 2, 3, 4], 1, 3) == [1, 2, 3]
    assert ops.krum_select(D, [4, 3, 2, 1, 0], 1, 1) == [3]
    D[2, 4] = D[4, 2] = float("nan")                                   # a NaN distance counts as +inf
    assert ops.krum_select(D, [0, 1, 2, 3, 4], 1, 1) == [1]
    with pytest.raises(ValueError):
        ops.krum_select(D, [0, 1, 2, 3, 4], 2, 1)                       # 5 < 2 * 2 + 3
    with pytest.raises(ValueError):
        ops.krum_select(D, [0, 1, 2, 3, 4], 1, 6)


def _loop_select(D, ids, f, m):
    """Krum / Multi-Krum as a plain Python loop: neighbours sorted, added one by one in ascending order."""
    K = len(ids)
    scores = []
    for i in range(K):
        s = 0.0
        for v in sorted(float(D[i][j]) for j in range(K) if j != i)[: K - f - 2]:
            s += v
        scores.append(s)
    return sorted(sorted(range(K), key=lambda i: (scores[i], ids[i]))[:m])


@pytest.mark.parametrize("K,f", [(5, 1), (12, 3), (40, 4), (97, 20)])
def test_krum_select_matches_a_sequential_loop(K, f):
    gen = torch.Generator().manual_seed(K)
    x = torch.randn(K, 6, generator=gen, dtype=torch.float64) * torch.logspace(-3, 3, K, dtype=torch.float64)[:, None]
    x[1] = x[0]                                                         # exact ties
    D = torch.cdist(x, x, compute_mode="donot_use_mm_for_euclid_dist") ** 2
    ids = torch.randperm(K, generator=gen).tolist()
    for m in (1, K - f, K):
        assert ops.krum_select(D, ids, f, m) == _loop_select(D, ids, f, m)


# ---- the server step over the admitted set -------------------------------------------------------------------------------
def _updates(K, n, seed):
    gen = torch.Generator().manual_seed(seed)
    w0 = torch.randn(n, generator=gen)
    ws = [w0 + 0.05 * (k + 1) * torch.randn(n, generator=gen) for k in range(K)]
    ws[0] = w0 + 3.0                                                    # far from everyone: rejected by F >= 1
    return w0, ws


@pytest.mark.parametrize("aggr,theta,clip", [("avg", 0, 0.0), ("avg", 3, 0.0), ("comed", 2, 0.0), ("sign", 3, 0.0), ("avg", 2, 5.0)])
def test_multikrum_all_admitted_equals_no_selection_bitwise(aggr, theta, clip):
    K, n, nv = 6, 512, 480
    w0, ws = _updates(K, n, 11)
    sizes = {i: 100 + 13 * i for i in range(K)}
    base = dict(num_agents=K, aggr=aggr, robustLR_threshold=theta, server_lr=0.01, clip=clip, server_clip=clip > 0)
    out = {}
    for sel in ("none", "multikrum"):
        extra = dict(select=sel, select_m=K) if sel != "none" else {}
        a = make_args(**base, **extra)
        agg = Aggregation(sizes, n, None, a)
        wg = w0.clone()
        agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
        out[sel] = wg
        if sel != "none":
            assert agg.last_admitted == list(range(K))
    assert torch.equal(out["none"], out["multikrum"])


@pytest.mark.parametrize("aggr,theta", [("avg", 0), ("avg", 2), ("comed", 2), ("sign", 2)])
def test_rejected_participants_take_no_part(aggr, theta):
    K, n, nv = 7, 256, 240
    w0, ws = _updates(K, n, 12)
    sizes = {i: 50 + 7 * i for i in range(K)}
    a = make_args(num_agents=K, num_corrupt=1, aggr=aggr, robustLR_threshold=theta, server_lr=0.01, select="multikrum")
    assert (a.select_f, a.select_m) == (1, 6)
    agg = Aggregation(sizes, n, None, a)
    wg = w0.clone()
    agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
    assert agg.last_admitted == list(range(1, K))
    assert agg.last_select == {"Select/Corrupt_Participants": 1, "Select/Corrupt_Admitted": 0}
    ref, _ = ops.aggregate_oracle(w0, ws[1:], [sizes[i] for i in range(1, K)], aggr, theta, a.server_lr, None, nv)
    assert torch.equal(wg, ref)


def _local_aggregator(n, nv, K):
    from rlr_b200.parallel import FusedAggregator, init_distributed
    return FusedAggregator(init_distributed("cpu"), n, nv, K, "local")


def test_slots_form_selects_like_the_dict_form():
    K, n, nv = 7, 256, 240
    w0, ws = _updates(K, n, 13)
    sizes = {i: 50 + 7 * i for i in range(K)}
    for m in (4, K):
        a = make_args(num_agents=K, num_corrupt=1, aggr="avg", robustLR_threshold=2, select="multikrum", select_m=m)
        fa = _local_aggregator(n, nv, K)
        fa.w_global.copy_(w0)
        for j in range(K):
            fa.slots[j].copy_(ws[j])
        agg = Aggregation(sizes, n, None, a, fused=fa)
        agg.aggregate_slots(list(range(K)), 1)
        dict_form = Aggregation(sizes, n, None, a)
        wg = w0.clone()
        dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
        assert agg.last_admitted == dict_form.last_admitted and len(agg.last_admitted) == m
        assert torch.equal(fa.w_global, wg)
        fa.close()


def test_engine_logs_selection_fields(tmp_path):
    kw = dict(data="fmnist", synthetic=1200, synthetic_val=300, num_agents=5, local_ep=1, bs=64, device="cpu", num_corrupt=1,
              poison_frac=0.5, select="multikrum", log_dir=str(tmp_path / "logs"), no_tensorboard=True, rounds=2)
    eng = FLEngine(make_args(**kw), verbose=False)
    hist = eng.fit()
    eng.close()
    run_dirs = os.listdir(tmp_path / "logs")
    recs = [json.loads(l) for l in open(tmp_path / "logs" / run_dirs[0] / "metrics.jsonl")]
    assert [r["round"] for r in recs] == [1, 2]
    for r, h in zip(recs, hist):
        assert r["select_corrupt_participants"] == 1 and 0 <= r["select_corrupt_admitted"] <= 1
        assert h["select_corrupt_admitted"] == r["select_corrupt_admitted"]
    assert len(eng.aggregator.last_admitted) == eng.args.select_m == 4


# ---- 2 ranks over gloo ---------------------------------------------------------------------------------------------------
def _gloo_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200 import ops as ops_
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed("cpu")
    n, nv, n_part = 1024, 1000, 7
    w0, ws = _updates(n_part, n, 21)
    weights = [float(10 + 3 * j) for j in range(n_part)]
    out = {}
    for transport in ("gather", "reduce"):
        for scaled in (False, True):
            fa = FusedAggregator(ctx, n, nv, (n_part + world - 1) // world, "gloo", transport=transport)
            fa.w_global.copy_(w0)
            for j in range(n_part):
                r, s = fa.slot_owner(j)
                if r == rank:
                    fa.slots[s].copy_(ws[j])
            scales = torch.linspace(0.5, 1.0, n_part) if scaled else None
            assert fa.gathers(n_part)
            copies = fa.gather_participants(n_part) if scaled else None     # both passes on one gather, or each pass gathers
            D = fa.pairwise_sqdist(n_part, scales, copies)
            keep = ops_.krum_select(D, list(range(n_part)), 1, 5)
            fa.aggregate(weights, "avg", 2, 1.0, 0.0, 0, 1, scales, members=keep, participants=copies)
            out[(transport, scaled)] = (D.clone(), keep, fa.w_global.clone())
            fa.close()
    torch.save(out, os.path.join(outdir, f"s{rank}.pt"))
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_ranks_agree_on_distances_selection_and_step(tmp_path):
    world = 2
    mp.spawn(_gloo_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"s{r}.pt") for r in range(world)]
    n, nv, n_part = 1024, 1000, 7
    w0, ws = _updates(n_part, n, 21)
    weights = [float(10 + 3 * j) for j in range(n_part)]
    for (transport, scaled), (D, keep, wg) in outs[0].items():
        for o in outs[1:]:
            D1, keep1, wg1 = o[(transport, scaled)]
            assert torch.equal(D1, D) and keep1 == keep and torch.equal(wg1, wg)
        scales = torch.linspace(0.5, 1.0, n_part) if scaled else None
        torch.testing.assert_close(D, ops.pairwise_sqdist(ws, nv, w0 if scaled else None, scales), rtol=0, atol=0)
        assert keep == ops.krum_select(D, list(range(n_part)), 1, 5) and 0 not in keep
        ref, _ = ops.aggregate_oracle(w0, [ws[j] for j in keep], [weights[j] for j in keep], "avg", 2, 1.0, None, nv,
                                      scales[keep] if scaled else None)
        assert torch.equal(wg, ref)
    for scaled in (False, True):    # the reduce transport selects over the gather transport
        assert torch.equal(outs[0][("reduce", scaled)][2], outs[0][("gather", scaled)][2])
