"""DnC participant selection (``--select dnc``) on CPU: option validation, defaults and the banner, the coordinate subsample, the host
rule against an independent numpy DnC (explicit gather, centring and SVD), a planted malicious direction, ties and NaN updates, the
no-op case against ``--select none`` bit for bit, the slots form against the dict form, and a 2-rank gloo run on both transports."""
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
from rlr_b200.options import DNC_DIM, DNC_FRAC, DNC_ITERS, make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- options ------------------------------------------------------------------------------------------------------------
def test_defaults_resolve():
    a = make_args(select="dnc", num_agents=10, num_corrupt=2)
    assert (a.select_f, a.dnc_dim, a.dnc_iters, a.dnc_frac) == (2, DNC_DIM, DNC_ITERS, DNC_FRAC) == (2, 10000, 1, 1.0)
    assert a.select_m == 0
    b = make_args(select="dnc", num_agents=10, num_corrupt=2, select_f=3, dnc_dim=500, dnc_iters=2, dnc_frac=0.5)
    assert (b.select_f, b.dnc_dim, b.dnc_iters, b.dnc_frac) == (3, 500, 2, 0.5)
    n = make_args()
    assert (n.dnc_dim, n.dnc_iters, n.dnc_frac) == (None, None, None)
    # DnC does not need Krum's K >= 2F + 3: 5 participants, F = 2, one removed per iteration
    assert make_args(select="dnc", num_agents=5, select_f=2, dnc_frac=0.5).select_f == 2


@pytest.mark.parametrize("kw", [
    dict(dnc_dim=100),                                                      # flags without --select dnc
    dict(dnc_iters=2),
    dict(dnc_frac=0.5),
    dict(select="multikrum", num_agents=10, num_corrupt=1, dnc_dim=100),
    dict(select="dnc", num_agents=10, num_corrupt=1, select_m=5),           # --select_m with dnc
    dict(select="dnc", num_agents=10, select_f=5, dnc_frac=1.0, dnc_iters=2),   # 10 - 2 x 5 = 0 could be admitted
    dict(select="dnc", num_agents=10, select_f=10),                         # 10 - 10 = 0
    dict(select="dnc", num_agents=10, select_f=2, dnc_iters=3, robustLR_threshold=5),   # fewest admitted 10 - 6 = 4 < 5
    dict(select="dnc", num_agents=10, num_corrupt=1, dnc_dim=0),
    dict(select="dnc", num_agents=10, num_corrupt=1, dnc_iters=0),
    dict(select="dnc", num_agents=10, num_corrupt=1, dnc_frac=-0.5),
    dict(select="dnc", num_agents=10, num_corrupt=1, dnc_frac=float("inf")),
    dict(select="dnc", num_agents=10, num_corrupt=1, dnc_frac=float("nan")),
    dict(select="dnc", num_agents=10, num_corrupt=1, detect="fldetector"),
    dict(select="dnc", num_agents=10, select_f=4, aggr="flame", robustLR_threshold=5),  # FLAME over the 6 admitted: 4 voters
])
def test_dnc_options_rejected(kw):
    with pytest.raises(ValueError):
        make_args(**kw)


def test_threshold_at_the_fewest_admitted_is_accepted():
    a = make_args(select="dnc", num_agents=10, select_f=2, dnc_iters=3, robustLR_threshold=4)
    assert a.robustLR_threshold == 4


def test_banner_line(capsys):
    from rlr_b200.options import print_exp_details
    print_exp_details(make_args(select="dnc", num_agents=10, num_corrupt=2, dnc_dim=500, dnc_iters=3, dnc_frac=0.5))
    out = capsys.readouterr().out
    assert "Selection DnC (F / c / b / T): 2 / 0.5 / 500 / 3" in out and "Selection (F / M)" not in out
    print_exp_details(make_args(select="multikrum", num_agents=10, num_corrupt=1))
    out = capsys.readouterr().out
    assert "Selection (F / M): multikrum (1 / 9)" in out and "DnC" not in out


# ---- the subsample -------------------------------------------------------------------------------------------------------
def test_sample_is_sorted_distinct_and_seeded_by_seed_round_and_iteration():
    s = ops.dnc_sample(3, 7, 0, 1000, 123457)
    assert s.shape == (1000,) and s.dtype == np.int64
    assert np.all(np.diff(s) > 0) and s[0] >= 0 and s[-1] < 123457
    assert np.array_equal(s, ops.dnc_sample(3, 7, 0, 1000, 123457))
    assert not np.array_equal(s, ops.dnc_sample(3, 7, 1, 1000, 123457))
    assert not np.array_equal(s, ops.dnc_sample(3, 8, 0, 1000, 123457))
    assert not np.array_equal(s, ops.dnc_sample(4, 7, 0, 1000, 123457))


@pytest.mark.parametrize("b", [101, 102, 10 ** 6])
def test_a_sample_of_at_least_n_vote_takes_every_coordinate(b):
    assert np.array_equal(ops.dnc_sample(0, 1, 0, b, 101), np.arange(101))


def test_sample_refuses_n_vote_beyond_int32():
    with pytest.raises(ValueError):
        ops.dnc_sample(0, 1, 0, 10, 1 << 31)


# ---- the host rule against an independent numpy DnC ------------------------------------------------------------------------
def _numpy_dnc(ws, g, n_vote, samples, scales, ids, f, c):
    """DnC as the paper writes it: gather, centre, SVD, score <x_k - mu, v1>^2, keep the K - floor(c f) lowest, intersect."""
    K = len(ws)
    W = np.stack([np.asarray(w, dtype=np.float32) for w in ws]).astype(np.float64)
    G = np.asarray(g, dtype=np.float32).astype(np.float64)
    keep, all_scores = set(range(K)), []
    for r in samples:
        assert r.max() < n_vote
        x = W[:, r] - G[r]
        if scales is not None:
            x = x * np.asarray(scales, dtype=np.float32).astype(np.float64)[:, None]
        mu = np.zeros(len(r))
        for k in range(K):                                              # the mean adds in ascending k
            mu = mu + x[k]
        mu = mu / K
        y = (x - mu).astype(np.float32).astype(np.float64)              # rounded once to fp32
        v = np.linalg.svd(y, full_matrices=False)[2][0]
        s = (y @ v) ** 2
        all_scores.append(s)
        keep &= set(sorted(range(K), key=lambda k: (s[k], ids[k]))[: K - math.floor(c * f)])
    return sorted(keep), all_scores


def _random_updates(K, n, seed):
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(n, generator=gen)
    ws = [g + 0.02 * (1 + k % 4) * torch.randn(n, generator=gen) for k in range(K)]
    return g, ws


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("c", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("T", [1, 3])
def test_dnc_select_matches_numpy_dnc(T, c, scaled):
    K, n, nv, b, f = 14, 700, 689, 150, 2
    g, ws = _random_updates(K, n, 100 * T + int(10 * c) + scaled)
    scales = torch.linspace(0.3, 1.0, K).float() if scaled else None
    samples = np.stack([ops.dnc_sample(5, 2, t, b, nv) for t in range(T)])
    ids = np.random.default_rng(T).permutation(K).tolist()
    grams = ops.dnc_grams(ws, g, samples, nv, scales)
    assert grams.shape == (T, K, K) and grams.dtype == torch.float64
    keep = ops.dnc_select(grams, ids, f, c)
    want, want_scores = _numpy_dnc([w.numpy() for w in ws], g.numpy(), nv, samples, scales, ids, f, c)
    for t in range(T):
        s = ops.dnc_scores(grams[t])
        np.testing.assert_allclose(s, want_scores[t], rtol=1e-9, atol=1e-12 * want_scores[t].max())
    assert keep == want
    assert len(keep) >= K - T * math.floor(c * f)


def test_gram_statement_is_the_gram_of_the_centred_gather():
    K, n, nv = 5, 64, 61
    g, ws = _random_updates(K, n, 4)
    s = ops.dnc_sample(0, 1, 0, 20, nv)
    y = ops.dnc_gather_statement(ws, g, s)
    assert y.dtype == torch.float32 and y.shape == (K, 20)
    torch.testing.assert_close(y.double().sum(0), torch.zeros(20, dtype=torch.float64), rtol=0, atol=1e-6)
    assert torch.equal(ops.dnc_gram_statement(ws, g, s[None])[0], y.double() @ y.double().T)


def test_planted_direction_is_removed_in_every_iteration():
    K, n, nv, bad = 10, 4000, 3996, 3
    gen = torch.Generator().manual_seed(9)
    g = torch.randn(n, generator=gen)
    honest = [0.01 * torch.randn(n, generator=gen) for _ in range(K)]
    d = torch.randn(n, generator=gen)
    d = d / d.norm() * 2.0 * float(torch.stack(honest).norm(dim=1).mean())     # about twice an honest update's norm
    ws = [g + honest[k] + (d if k < bad else 0.0) for k in range(K)]
    samples = np.stack([ops.dnc_sample(1, 3, t, 800, nv) for t in range(4)])
    grams = ops.dnc_grams(ws, g, samples, nv)
    for t in range(4):
        assert ops.dnc_select(grams[t:t + 1], list(range(K)), bad, 1.0) == list(range(bad, K)), t
    assert ops.dnc_select(grams, list(range(K)), bad, 1.0) == list(range(bad, K))


def test_ties_go_to_the_lower_id():
    ws = [torch.ones(16) for _ in range(5)]                             # every centred update 0: every score 0
    grams = ops.dnc_grams(ws, torch.zeros(16), np.arange(16)[None], 16)
    assert not grams.any()
    ids = [7, 3, 9, 1, 5]
    assert ops.dnc_select(grams, ids, 2, 1.0) == [1, 3, 4]              # ids 3, 1, 5 kept
    assert ops.dnc_select(grams, ids, 1, 1.0) == [0, 1, 3, 4]


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("bad_id", [0, 3])
def test_nan_updates_are_never_admitted_ahead_of_finite_ones(bad_id, every):
    K, n = 6, 256
    g, ws = _random_updates(K, n, 17)
    ws[bad_id] = ws[bad_id].clone()
    ws[bad_id][::every] = float("nan")
    grams = ops.dnc_grams(ws, g, np.arange(n)[None], n)
    s = ops.dnc_scores(grams[0])
    assert s[bad_id] == np.inf and np.all(np.isfinite(np.delete(s, bad_id)))
    for f in (1, 2, 4):
        keep = ops.dnc_select(grams, list(range(K)), f, 1.0)
        assert bad_id not in keep and len(keep) == K - f
    if every > 1:
        return
    # a participant that is NaN everywhere stays out of the mean: the others' block is the Gram matrix without it
    others = [w for k, w in enumerate(ws) if k != bad_id]
    clean = ops.dnc_grams(others, g, np.arange(n)[None], n)
    assert torch.equal(torch.as_tensor(np.delete(np.delete(grams[0].numpy(), bad_id, 0), bad_id, 1)), clean[0])


def test_dnc_select_refuses_an_empty_iteration():
    with pytest.raises(ValueError):
        ops.dnc_select(torch.zeros(1, 3, 3, dtype=torch.float64), [0, 1, 2], 3, 1.0)


# ---- the server step ------------------------------------------------------------------------------------------------------
def _updates(K, n, seed):
    gen = torch.Generator().manual_seed(seed)
    w0 = torch.randn(n, generator=gen)
    ws = [w0 + 0.05 * (1 + k % 3) * torch.randn(n, generator=gen) for k in range(K)]
    ws[0] = w0 + 0.05 * torch.randn(n, generator=gen) + 0.4             # a shared offset far along one direction
    ws[1] = w0 + 0.05 * torch.randn(n, generator=gen) + 0.4
    return w0, ws


@pytest.mark.parametrize("aggr,theta,clip", [("avg", 0, 0.0), ("avg", 3, 0.0), ("sign", 3, 0.0), ("avg", 2, 5.0), ("sign", 2, 5.0)])
def test_no_removal_equals_no_selection_bitwise(aggr, theta, clip):
    K, n, nv = 6, 512, 480
    w0, ws = _updates(K, n, 11)
    sizes = {i: 100 + 13 * i for i in range(K)}
    base = dict(num_agents=K, num_corrupt=2, aggr=aggr, robustLR_threshold=theta, server_lr=0.01, clip=clip, server_clip=clip > 0)
    out = {}
    for sel, extra in (("none", {}), ("dnc", dict(select="dnc", dnc_frac=0.0)), ("dnc_f0", dict(select="dnc", select_f=0))):
        a = make_args(**base, **extra)
        agg = Aggregation(sizes, n, None, a)
        wg = w0.clone()
        agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
        out[sel] = wg
        if sel != "none":
            assert agg.last_admitted == list(range(K))
            assert agg.last_select == {"Select/Corrupt_Participants": 2, "Select/Corrupt_Admitted": 2}
    assert torch.equal(out["none"], out["dnc"]) and torch.equal(out["none"], out["dnc_f0"])


@pytest.mark.parametrize("aggr,theta,clip", [("avg", 0, 0.0), ("sign", 2, 0.0), ("avg", 2, 5.0)])
def test_removed_participants_take_no_part(aggr, theta, clip):
    K, n, nv = 8, 512, 500
    w0, ws = _updates(K, n, 12)
    sizes = {i: 50 + 7 * i for i in range(K)}
    a = make_args(num_agents=K, num_corrupt=2, aggr=aggr, robustLR_threshold=theta, server_lr=0.01, select="dnc", dnc_dim=200,
                  clip=clip, server_clip=clip > 0)
    agg = Aggregation(sizes, n, None, a)
    wg = w0.clone()
    agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
    assert agg.last_admitted == list(range(2, K))
    assert agg.last_select == {"Select/Corrupt_Participants": 2, "Select/Corrupt_Admitted": 0}
    scales = None
    if clip > 0:
        scales = (1.0 / torch.clamp(ops.update_norms(w0, ws, nv) / clip, min=1.0)).float()[2:]
    ref, _ = ops.aggregate_oracle(w0, ws[2:], [sizes[i] for i in range(2, K)], aggr, theta, a.server_lr, None, nv, scales)
    assert torch.equal(wg, ref)


def _local_aggregator(n, nv, K):
    from rlr_b200.parallel import FusedAggregator, init_distributed
    return FusedAggregator(init_distributed("cpu"), n, nv, K, "local")


@pytest.mark.parametrize("clip", [0.0, 5.0])
def test_slots_form_selects_like_the_dict_form(clip):
    K, n, nv = 7, 256, 243
    w0, ws = _updates(K, n, 13)
    sizes = {i: 50 + 7 * i for i in range(K)}
    for T, c in ((1, 1.0), (3, 0.5)):
        a = make_args(num_agents=K, num_corrupt=2, aggr="avg", robustLR_threshold=2, select="dnc", dnc_dim=60, dnc_iters=T, dnc_frac=c,
                      clip=clip, server_clip=clip > 0)
        fa = _local_aggregator(n, nv, K)
        fa.w_global.copy_(w0)
        for j in range(K):
            fa.slots[j].copy_(ws[j])
        agg = Aggregation(sizes, n, None, a, fused=fa)
        agg.aggregate_slots(list(range(K)), 4)
        dict_form = Aggregation(sizes, n, None, a)
        wg = w0.clone()
        dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 4, n_vote=nv)
        assert agg.last_admitted == dict_form.last_admitted and len(agg.last_admitted) < K
        assert torch.equal(fa.w_global, wg)
        fa.close()


# ---- 2 ranks over gloo ---------------------------------------------------------------------------------------------------
N, NV, N_PART = 1024, 999, 7


def _gloo_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200 import ops as ops_
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed("cpu")
    w0, ws = _updates(N_PART, N, 21)
    weights = [float(10 + 3 * j) for j in range(N_PART)]
    samples = np.stack([ops_.dnc_sample(0, 1, t, 300, NV) for t in range(2)])
    out = {}
    for transport in ("gather", "reduce"):
        for scaled in (False, True):
            fa = FusedAggregator(ctx, N, NV, (N_PART + world - 1) // world, "gloo", transport=transport)
            fa.w_global.copy_(w0)
            for j in range(N_PART):
                r, s = fa.slot_owner(j)
                if r == rank:
                    fa.slots[s].copy_(ws[j])
            scales = torch.linspace(0.5, 1.0, N_PART) if scaled else None
            assert fa.gathers(N_PART)
            copies = fa.gather_participants(N_PART) if scaled else None     # both passes on one gather, or each pass gathers
            G = fa.dnc_grams(N_PART, samples, scales, None, copies)
            keep = ops_.dnc_select(G, list(range(N_PART)), 2, 1.0)
            fa.aggregate(weights, "avg", 2, 1.0, 0.0, 0, 1, scales, members=keep, participants=copies)
            out[(transport, scaled)] = (G.clone(), keep, fa.w_global.clone())
            fa.close()
    torch.save(out, os.path.join(outdir, f"s{rank}.pt"))
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_ranks_agree_on_grams_selection_and_step(tmp_path):
    world = 2
    mp.spawn(_gloo_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"s{r}.pt") for r in range(world)]
    w0, ws = _updates(N_PART, N, 21)
    weights = [float(10 + 3 * j) for j in range(N_PART)]
    samples = np.stack([ops.dnc_sample(0, 1, t, 300, NV) for t in range(2)])
    for (transport, scaled), (G, keep, wg) in outs[0].items():
        for o in outs[1:]:
            G1, keep1, wg1 = o[(transport, scaled)]
            assert torch.equal(G1, G) and keep1 == keep and torch.equal(wg1, wg)
        scales = torch.linspace(0.5, 1.0, N_PART) if scaled else None
        assert torch.equal(G, ops.dnc_grams(ws, w0, samples, NV, scales))
        assert keep == ops.dnc_select(G, list(range(N_PART)), 2, 1.0) and 0 not in keep and 1 not in keep
        ref, _ = ops.aggregate_oracle(w0, [ws[j] for j in keep], [weights[j] for j in keep], "avg", 2, 1.0, None, NV,
                                      scales[keep] if scaled else None)
        assert torch.equal(wg, ref)
    for scaled in (False, True):    # the reduce transport selects over the gather transport
        assert torch.equal(outs[0][("reduce", scaled)][2], outs[0][("gather", scaled)][2])
