"""RFA aggregation (``--aggr rfa``) on CPU: option validation and the banner, the fp64 distance statement against brute-force numpy, the
Weiszfeld loop against an independent numpy smoothed geometric median, the objective's descent, ``--rfa_iters 0`` against ``--aggr avg``,
a boosted participant, one participant, 2-rank gloo runs on both transports (with Multi-Krum and server clipping) and the JSONL fields of
a ``federated.py`` run."""
import json
import math
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
    a = make_args(aggr="rfa")
    assert (a.rfa_iters, a.rfa_nu) == (3, 1e-6) and a.server_lr == 1.0
    b = make_args(aggr="rfa", rfa_iters=0, rfa_nu=0.5)
    assert (b.rfa_iters, b.rfa_nu) == (0, 0.5)
    c = make_args()
    assert c.rfa_iters is None and c.rfa_nu is None


@pytest.mark.parametrize("kw", [
    dict(aggr="avg", rfa_iters=3),
    dict(aggr="comed", rfa_nu=1e-6),
    dict(aggr="fltrust", rfa_iters=1),
    dict(aggr="rfa", rfa_iters=-1),
    dict(aggr="rfa", rfa_nu=0.0),
    dict(aggr="rfa", rfa_nu=-1e-3),
    dict(aggr="rfa", rfa_nu=float("inf")),
])
def test_rfa_options_rejected(kw):
    with pytest.raises(ValueError):
        make_args(**kw)


def test_command_line_flags_and_banner(capsys):
    from rlr_b200.options import args_parser, finalize_args, print_exp_details
    a = finalize_args(args_parser(["--aggr", "rfa", "--rfa_iters", "5", "--rfa_nu", "0.01"]))
    assert (a.rfa_iters, a.rfa_nu) == (5, 0.01)
    with pytest.raises(ValueError):
        finalize_args(args_parser(["--rfa_iters", "5"]))
    print_exp_details(make_args())
    assert "RFA" not in capsys.readouterr().out
    print_exp_details(a)
    out = capsys.readouterr().out
    assert "RFA passes / nu: 5 / 0.01" in out and "Aggregation Function: rfa" in out


# ---- the distance pass and the loop --------------------------------------------------------------------------------------
def _numpy_sqdist(ws, b, n_vote, g=None, scales=None):
    x = np.stack([np.asarray(w[:n_vote], dtype=np.float64) for w in ws])
    if scales is not None:
        x = (x - np.asarray(g[:n_vote], dtype=np.float64)) * np.asarray(scales, dtype=np.float32).astype(np.float64)[:, None]
    z = np.asarray(b, dtype=np.float64) @ x
    return np.array([math.fsum(float(v) for v in (r - z) ** 2) for r in x])


@pytest.mark.parametrize("K,n,n_vote,clip", [(1, 16, 16, False), (5, 64, 48, False), (9, 200, 180, True), (4, 96, 96, True)])
def test_statement_matches_numpy(K, n, n_vote, clip):
    gen = torch.Generator().manual_seed(K * n)
    g = torch.randn(n, generator=gen)
    ws = [g + 0.1 * (k + 1) * torch.randn(n, generator=gen) for k in range(K)]
    for w in ws:
        w[n_vote:] += 1e3                                                 # tail coordinates do not count
    b = np.random.default_rng(K).random(K) + 0.1
    b /= b.sum()
    sc = torch.linspace(0.3, 1.0, K) if clip else None
    d2 = ops.rfa_sqdist(ws, b, n_vote, g if clip else None, sc)
    assert d2.dtype == torch.float64 and d2.shape == (K,)
    assert torch.equal(d2, ops.rfa_statement(ws, b, 0, n_vote, g if clip else None, sc))
    np.testing.assert_allclose(d2.numpy(), _numpy_sqdist(ws, b, n_vote, g, sc), rtol=1e-12, atol=1e-12)
    with pytest.raises(ValueError):
        ops.rfa_sqdist(ws, b, n_vote, None, torch.ones(K))


def _numpy_weiszfeld(X, alpha, T, nu):
    """Smoothed Weiszfeld (Pillutla et al., Algorithm 3) from the alpha-weighted mean, written independently of ops: the final weights
    and the objective sum_k alpha_k ||z - x_k|| at every iterate z_0 .. z_T."""
    alpha = np.asarray(alpha, dtype=np.float64)
    beta, F = alpha.copy(), []
    for t in range(T + 1):
        z = (beta / beta.sum()) @ X
        d = np.linalg.norm(X - z, axis=1)
        F.append(float(alpha @ d))
        if t < T:
            beta = alpha / np.maximum(nu, d)
    return beta, F, z


@pytest.mark.parametrize("K,T,nu", [(2, 3, 1e-6), (7, 3, 1e-6), (10, 8, 1e-6), (6, 4, 0.5)])
def test_loop_matches_numpy_weiszfeld(K, T, nu):
    rng = np.random.default_rng(K + T)
    n = 300
    X = rng.standard_normal((K, n)) * rng.uniform(0.2, 3.0, (K, 1)) + rng.standard_normal(n)
    ws = [torch.from_numpy(x.astype(np.float32)) for x in X]
    X32 = np.stack([w.numpy().astype(np.float64) for w in ws])
    alpha = rng.integers(50, 500, K).astype(float)
    beta, F = ops.rfa(alpha, lambda b: ops.rfa_sqdist(ws, b, n), T, nu)
    want_beta, want_F, _ = _numpy_weiszfeld(X32, alpha, T, nu)
    np.testing.assert_allclose(beta, want_beta, rtol=1e-10)
    np.testing.assert_allclose(F, want_F[:T], rtol=1e-12)
    assert all(type(x) is float for x in beta)


@pytest.mark.parametrize("seed", range(4))
def test_objective_does_not_increase(seed):
    rng = np.random.default_rng(seed)
    K, n = 9, 256
    X = rng.standard_normal((K, n))
    X[seed % K] *= 50.0                                                    # one far-off participant
    ws = [torch.from_numpy(x.astype(np.float32)) for x in X]
    _, F = ops.rfa(rng.integers(10, 100, K), lambda b: ops.rfa_sqdist(ws, b, n), 12, 1e-6)
    assert len(F) == 12
    assert all(F[t + 1] <= F[t] * (1 + 1e-12) for t in range(11)), F
    assert F[-1] < F[0]


def test_weights_and_zero_passes():
    beta = ops.rfa_weights([2.0, 4.0, 6.0], [4.0, 0.0, 1e-14], 1e-6)
    np.testing.assert_array_equal(beta, [1.0, 4.0 / 1e-6, 6.0 / 1e-6])
    calls = []
    beta, F = ops.rfa([3, 5.5, 7], lambda b: calls.append(b), 0, 1e-6)
    assert beta == [3.0, 5.5, 7.0] and F == [] and calls == []


# ---- the server step ------------------------------------------------------------------------------------------------------
def _round(K, n, seed, boost=()):
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(n, generator=gen)
    mean = 0.05 * torch.randn(n, generator=gen)
    ws = [g + mean + 0.02 * torch.randn(n, generator=gen) for _ in range(K)]
    for k in boost:
        ws[k] = g + 100.0 * (ws[k] - g)
    return g, mean, ws


@pytest.mark.parametrize("theta,clip,server_opt", [(0, 0.0, "sgd"), (3, 0.0, "sgd"), (2, 0.5, "sgd"), (2, 0.0, "adam")])
def test_zero_passes_equal_avg_bitwise(theta, clip, server_opt):
    K, n, nv = 7, 512, 480
    g, _, ws = _round(K, n, 3, boost=(1,))
    sizes = {i: 100 + 13 * i for i in range(K)}
    base = dict(num_agents=K, num_corrupt=1, robustLR_threshold=theta, clip=clip, server_clip=clip > 0, server_opt=server_opt,
                server_lr=0.05)
    rfa = Aggregation(sizes, n, None, make_args(aggr="rfa", rfa_iters=0, **base))
    avg = Aggregation(sizes, n, None, make_args(aggr="avg", **base))
    w_rfa, w_avg = g.clone(), g.clone()
    for rnd in (1, 2):
        rfa.aggregate_updates(w_rfa, {i: ws[i] for i in range(K)}, rnd, n_vote=nv)
        avg.aggregate_updates(w_avg, {i: ws[i] for i in range(K)}, rnd, n_vote=nv)
        assert torch.equal(w_rfa, w_avg)
        assert int(rfa.last_flipped) == int(avg.last_flipped)
    assert rfa.last_rfa["RFA/Passes"] == 0
    assert rfa.last_rfa["RFA/Corrupt_Weight"] == sizes[0] / sum(sizes.values())


def test_boosted_participant_cannot_drag_the_aggregate():
    K, n, nv = 10, 2048, 2000
    g, mean, ws = _round(K, n, 5, boost=(0,))
    sizes = {i: 100 for i in range(K)}
    honest = torch.stack([w[:nv] - g[:nv] for w in ws[1:]]).double().mean(0)
    out = {}
    for aggr in ("avg", "rfa"):
        agg = Aggregation(sizes, n, None, make_args(num_agents=K, num_corrupt=1, aggr=aggr))
        wg = g.clone()
        agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
        out[aggr] = float(((wg[:nv] - g[:nv]).double() - honest).norm() / honest.norm())
        if aggr == "rfa":
            assert agg.last_rfa["RFA/Corrupt_Weight"] < 0.01 and agg.last_rfa["RFA/Passes"] == 3
    print(f"relative distance from the honest mean: avg {out['avg']:.3f}, rfa {out['rfa']:.4f}")
    assert out["avg"] > 5.0 and out["rfa"] < 0.1                        # measured: avg 10.8, rfa 0.046


def test_one_participant_equals_avg():
    g, _, ws = _round(1, 256, 11)
    res = {}
    for aggr in ("avg", "rfa"):
        agg = Aggregation({0: 37}, 256, None, make_args(num_agents=1, aggr=aggr, robustLR_threshold=1))
        wg = g.clone()
        agg.aggregate_updates(wg, {0: ws[0]}, 1, n_vote=240)
        res[aggr] = wg
    assert torch.equal(res["rfa"], res["avg"])


def test_multikrum_then_rfa_keeps_the_admitted_members():
    K, n, nv = 7, 256, 240
    g, _, ws = _round(K, n, 8, boost=(0,))
    sizes = {i: 50 + 7 * i for i in range(K)}
    a = make_args(num_agents=K, num_corrupt=1, aggr="rfa", robustLR_threshold=2, select="multikrum")
    agg = Aggregation(sizes, n, None, a)
    wg = g.clone()
    agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
    assert agg.last_admitted == list(range(1, K)) and agg.last_rfa["RFA/Corrupt_Weight"] == 0.0
    keep = list(range(1, K))
    beta, _ = ops.rfa([sizes[i] for i in keep], lambda b: ops.rfa_statement([ws[i] for i in keep], b, 0, nv), 3, 1e-6)
    ref, _ = ops.aggregate_oracle(g, [ws[i] for i in keep], beta, "avg", 2, 1.0, None, nv)
    torch.testing.assert_close(wg, ref, rtol=0, atol=1e-6)


@pytest.mark.parametrize("select,clip", [("none", 0.0), ("multikrum", 0.0), ("none", 0.5), ("multikrum", 0.5)])
def test_slots_form_equals_the_dict_form(select, clip):
    from rlr_b200.parallel import FusedAggregator, init_distributed
    K, n, nv = 7, 256, 240
    g, _, ws = _round(K, n, 10, boost=(0,))
    sizes = {i: 50 + 7 * i for i in range(K)}
    a = make_args(num_agents=K, num_corrupt=1, aggr="rfa", robustLR_threshold=2, select=select, clip=clip, server_clip=clip > 0)
    fa = FusedAggregator(init_distributed("cpu"), n, nv, K, "local")
    fa.w_global.copy_(g)
    for j in range(K):
        fa.slots[j].copy_(ws[j])
    agg = Aggregation(sizes, n, None, a, fused=fa)
    agg.aggregate_slots(list(range(K)), 1)
    dict_form = Aggregation(sizes, n, None, a)
    wg = g.clone()
    dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
    assert agg.last_rfa == dict_form.last_rfa and agg.last_admitted == dict_form.last_admitted
    assert torch.equal(fa.w_global, wg)
    fa.close()


# ---- 2 ranks over gloo ---------------------------------------------------------------------------------------------------
CASES = [("none", 0.0), ("multikrum", 0.0), ("none", 0.5), ("multikrum", 0.5)]


def _transport_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.aggregation import Aggregation as Agg
    from rlr_b200.options import make_args as mk
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed("cpu")
    K, n, nv = 7, 1024, 1000
    g, _, ws = _round(K, n, 21, boost=(0,))
    out = {}
    for select, clip in CASES:
        for transport in ("gather", "reduce"):
            fa = FusedAggregator(ctx, n, nv, (K + world - 1) // world, "gloo", transport=transport)
            fa.w_global.copy_(g)
            for j, w in enumerate(ws):
                r, s = fa.slot_owner(j)
                if r == rank:
                    fa.slots[s].copy_(w)
            agg = Agg({i: 10 + 3 * i for i in range(K)}, n, None, mk(num_agents=K, num_corrupt=1, aggr="rfa", robustLR_threshold=2,
                                                                     select=select, clip=clip, server_clip=clip > 0), fused=fa)
            agg.aggregate_slots(list(range(K)), 1)
            out[(select, clip, transport)] = (fa.w_global.clone(), dict(agg.last_rfa), agg.last_admitted)
            fa.close()
    torch.save(out, os.path.join(outdir, f"t{rank}.pt"))
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_transports_match_the_dict_form(tmp_path):
    world = 2
    mp.spawn(_transport_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"t{r}.pt") for r in range(world)]
    K, n, nv = 7, 1024, 1000
    g, _, ws = _round(K, n, 21, boost=(0,))
    for select, clip in CASES:
        a = make_args(num_agents=K, num_corrupt=1, aggr="rfa", robustLR_threshold=2, select=select, clip=clip, server_clip=clip > 0)
        dict_form = Aggregation({i: 10 + 3 * i for i in range(K)}, n, None, a)
        wg = g.clone()
        dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
        for o in outs:
            for transport in ("gather", "reduce"):
                w, last, adm = o[(select, clip, transport)]
                assert torch.equal(w, outs[0][(select, clip, transport)][0]), (select, clip, transport)
                assert adm == dict_form.last_admitted and last["RFA/Passes"] == 3
                assert abs(last["RFA/Corrupt_Weight"] - dict_form.last_rfa["RFA/Corrupt_Weight"]) < 1e-9
                if transport == "gather" and clip == 0:                 # the same kernel on the same copies: the dict form's bits
                    assert torch.equal(w, wg) and last == dict_form.last_rfa, (select, transport)
                else:                                                   # all-reduced clip norms / partial sums: another order of adds
                    torch.testing.assert_close(w, wg, rtol=1e-6, atol=1e-6)


# ---- the command line ------------------------------------------------------------------------------------------------------
def test_federated_py_writes_the_rfa_fields(tmp_path):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "federated.py", "--data=fmnist", "--local_ep=1", "--bs=64", "--num_agents=4", "--rounds=2",
                        "--num_corrupt=1", "--poison_frac=0.5", "--robustLR_threshold=2", "--synthetic=400", "--synthetic_val=80",
                        "--aggr=rfa", "--rfa_iters=2", f"--log_dir={tmp_path}", "--no_tensorboard", "--device=cpu"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "Aggregation Function: rfa" in r.stdout and "RFA passes / nu: 2 / 1e-06" in r.stdout
    recs = [json.loads(l) for d in os.listdir(tmp_path) for l in open(tmp_path / d / "metrics.jsonl")]
    assert [rec["round"] for rec in recs] == [1, 2]
    for rec in recs:
        assert rec["rfa_passes"] == 2 and 0.0 <= rec["rfa_corrupt_weight"] <= 1.0
