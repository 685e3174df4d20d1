"""FLDetector (``--detect fldetector``) on CPU: options and the banner, the L-BFGS Hessian-vector coefficients against the dense compact
L-BFGS matrix, the exact 1-D k-means against brute force, the detection decision, and engine runs -- the defaults unchanged, the corrupt
agents flagged, the step after detection, bitwise resume, two gloo ranks, every --aggr rule and the memory refusal."""
import itertools
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.options import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- options ---------------------------------------------------------------------------------------------------------------------
def test_options_and_banner(capsys):
    from rlr_b200.options import args_parser, build_parser, finalize_args, print_exp_details
    assert "fldetector" in build_parser().format_help()
    a = make_args(num_agents=6, detect="fldetector")
    assert (a.fld_window, a.fld_start) == (10, 0)
    a = finalize_args(args_parser(["--detect", "fldetector", "--num_agents", "8", "--fld_window", "3", "--fld_start", "12",
                                   "--robustLR_threshold", "5"]))
    print_exp_details(a)
    assert "Detection (window / start): fldetector (3 / 12)" in capsys.readouterr().out
    print_exp_details(make_args())
    assert "Detection" not in capsys.readouterr().out
    bad = [(dict(fld_window=3), "need --detect fldetector"), (dict(fld_start=1), "need --detect fldetector"),
           (dict(detect="fldetector", fld_window=0), "--fld_window 0"), (dict(detect="fldetector", fld_start=-1), "--fld_start -1"),
           (dict(detect="fldetector", agent_frac=0.5), "every agent in every round"),
           (dict(detect="fldetector", num_agents=2), "at least 3 agents"),
           (dict(detect="fldetector", select="multikrum", num_agents=10), "does not combine with --select"),
           (dict(detect="fldetector", robustLR_threshold=7, num_agents=10), "7 > 6"),
           (dict(detect="fldetector", aggr="flame", robustLR_threshold=5, num_agents=10), "5 > 4.*under --aggr flame")]
    for kw, msg in bad:
        kw.setdefault("num_agents", 6)
        with pytest.raises(ValueError, match=msg):
            make_args(**kw)
    make_args(detect="fldetector", num_agents=10, robustLR_threshold=6)                    # floor(10/2) + 1 = 6 voters at least
    make_args(detect="fldetector", aggr="flame", num_agents=10, robustLR_threshold=4)       # FLAME on 6 candidates admits 4


# ---- the Hessian-vector product --------------------------------------------------------------------------------------------------
def _dense(R):
    """Dense compact L-BFGS B = sigma I - W M^-1 W^T, W = [sigma S, Y], of the ring R = [s_{r-N} .. s_r] (columns)."""
    N = R.shape[1] - 1
    S, Y = R[:, :N], R[:, 1:] - R[:, :N]
    sigma = (Y[:, -1] @ S[:, -1]) / (S[:, -1] @ S[:, -1])
    StY = S.T @ Y
    M = np.block([[sigma * S.T @ S, np.tril(StY, -1)], [np.tril(StY, -1).T, -np.diag(np.diag(StY))]])
    W = np.hstack([sigma * S, Y])
    return sigma * np.eye(R.shape[0]) - W @ np.linalg.solve(M, W.T), S, Y


@pytest.mark.parametrize("N", range(1, 11))
def test_hvp_coefficients_equal_the_dense_lbfgs_product(N):
    rng = np.random.default_rng(N)
    for _ in range(5):
        d = int(rng.integers(2 * N + 3, 60))
        R = rng.standard_normal((d, N + 1)) * rng.uniform(0.1, 10.0, N + 1)
        c = ops.fld_hvp_coefficients(torch.from_numpy(R.T @ R))
        assert c.dtype == np.float64 and c.shape == (N + 1,) and np.any(c)
        B, S, Y = _dense(R)
        scale = np.abs(B @ R[:, N]).max()
        assert np.abs(R @ c - B @ R[:, N]).max() <= 1e-10 * max(1.0, scale)
        assert np.abs(B @ S[:, -1] - Y[:, -1]).max() <= 1e-10 * max(1.0, np.abs(Y[:, -1]).max())          # the secant condition


def test_hvp_coefficient_fallbacks():
    rng = np.random.default_rng(3)
    R = rng.standard_normal((20, 4))
    R[:, 2] = 0.0                                                      # s_{r-1} = 0
    assert not np.any(ops.fld_hvp_coefficients(R.T @ R))
    R = rng.standard_normal((20, 4))
    G = R.T @ R
    for bad in (np.nan, np.inf):
        Gb = G.copy()
        Gb[0, 1] = Gb[1, 0] = bad
        assert not np.any(ops.fld_hvp_coefficients(Gb))
    R = rng.standard_normal((20, 3))
    R = np.hstack([R, R[:, :1]])                                       # rank-deficient ring: a singular system
    R[:, 1] = R[:, 0]                                                  # y_0 = 0: D has a zero and L a zero row
    assert not np.any(ops.fld_hvp_coefficients(R.T @ R))
    assert not np.any(ops.fld_hvp_coefficients(np.zeros((3, 3))))
    with pytest.raises(ValueError):
        ops.fld_hvp_coefficients(np.ones((1, 1)))


# ---- exact 1-D k-means and the decision ------------------------------------------------------------------------------------------
def _brute(x, k):
    n = len(x)
    best = np.inf
    for cuts in itertools.combinations(range(1, n), k - 1):
        b = (0, *cuts, n)
        best = min(best, sum(float(np.sum((x[b[i]:b[i + 1]] - x[b[i]:b[i + 1]].mean()) ** 2)) for i in range(k)))
    return best


def test_kmeans_is_exact_against_brute_force():
    rng = np.random.default_rng(0)
    for t in range(60):
        n = int(rng.integers(1, 10))
        x = np.sort(rng.uniform(0, 1, n) if t % 3 else np.round(rng.uniform(0, 1, n), 1))      # ties too
        W = ops.fld_kmeans_sse(x, n)
        for k in range(1, n + 1):
            assert abs(W[k - 1] - _brute(x, k)) <= 1e-12, (x, k)
        assert np.all(np.diff(W) <= 1e-15) and W[-1] == 0.0


def test_two_means_split_and_its_tie_rule():
    rng = np.random.default_rng(1)
    for _ in range(40):
        x = np.sort(rng.uniform(0, 1, int(rng.integers(2, 10))))
        i = ops.fld_two_means(x)
        costs = [_brute(x[:j], 1) + _brute(x[j:], 1) for j in range(1, len(x))]
        assert abs(costs[i - 1] - min(costs)) <= 1e-12
    assert ops.fld_two_means(np.array([0.0, 1.0, 2.0])) == 1              # splits 1 and 2 cost the same: the lowest wins
    assert ops.fld_two_means(np.array([0.0, 0.0, 1.0, 1.0])) == 2


def test_detect_decisions():
    rng = np.random.default_rng(2)
    two = np.r_[rng.uniform(0.0, 0.05, 8), rng.uniform(0.9, 1.0, 3)]
    flagged, k = ops.fld_detect(two, 7, 30)
    assert flagged == [8, 9, 10] and k > 1
    assert ops.fld_detect(two, 7, 30) == (flagged, k)                   # deterministic in (seed, round)
    perm = rng.permutation(11)
    assert sorted(perm[ops.fld_detect(two[perm], 7, 30)[0]].tolist()) == [8, 9, 10]
    # one tight group: one cluster, nobody flagged
    tight = 1.0 + 1e-3 * rng.standard_normal(12)
    assert ops.fld_detect(tight, 7, 30) == ([], 1)
    # the upper group a majority: refused
    major = np.r_[rng.uniform(0.0, 0.05, 4), rng.uniform(0.9, 1.0, 6)]
    flagged, k = ops.fld_detect(major, 7, 30)
    assert flagged == [] and k > 1
    # small and degenerate inputs
    assert ops.fld_detect([], 0, 1) == ([], 1)
    assert ops.fld_detect([0.3], 0, 1) == ([], 1)
    assert ops.fld_detect([0.1, 0.9], 0, 1) == ([], 1)                  # K_max = 1
    assert ops.fld_detect([0.5] * 6, 0, 1) == ([], 1)
    assert ops.fld_gap_clusters(np.array([0.0, 1.0]), 0, 1) == 1


# ---- engine runs -----------------------------------------------------------------------------------------------------------------
def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="fmnist", synthetic=300, synthetic_val=60, num_agents=5, agent_frac=1.0, local_ep=1, bs=64, device="cpu",
                num_corrupt=2, poison_frac=0.5, attack_boost=10.0, log_dir="", seed=5, trainer="torch", detect="fldetector", fld_window=2,
                snap=100)
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def test_detect_none_keeps_records_and_checkpoint_keys(tmp_path):
    ck = str(tmp_path / "ck.pt")
    eng = _engine(detect="none", fld_window=None, rounds=2, checkpoint=ck)
    hist = eng.fit()
    assert eng.fused.fld_table is None and eng.aggregator.fld_tables is None
    assert all(not any(k.startswith("fld") for k in rec) for rec in hist)
    assert set(torch.load(ck, weights_only=False)["extra"]) == {"cum_poison_acc_mean"}
    eng.close()


def _capture(eng):
    seen, orig = [], eng.aggregator.aggregate_slots

    def aggregate_slots(participants, rnd):
        ws = [w.clone() for w in eng.fused.gather_participants(len(participants))]
        wg = eng.fused.w_global.clone()
        orig(participants, rnd)
        seen.append((rnd, list(participants), wg, ws, eng.fused.w_global.clone()))
    eng.aggregator.aggregate_slots = aggregate_slots
    return seen


@pytest.fixture(scope="module")
def full_run():
    eng = _engine(rounds=8)
    seen = _capture(eng)
    hist = eng.fit()
    yield eng, seen, hist
    eng.close()


def test_boosted_corrupt_agents_are_flagged_and_the_step_drops_them(full_run):
    eng, seen, hist = full_run
    N = 2
    assert eng.aggregator.fld_flagged == [0, 1]
    det = eng.aggregator.fld_detect_round
    assert det == 2 * N + 1 == next(r["round"] for r in hist if "fld_flagged" in r)
    rec = hist[det - 1]
    assert rec["fld_flagged"] == [0, 1] and rec["fld_corrupt_flagged"] == 2 and rec["fld_detect_round"] == det and rec["fld_clusters"] > 1
    assert rec["fld_avg_corrupt_score"] > rec["fld_avg_honest_score"]
    for r in hist:
        assert ("fld_fallback" in r) == (N + 2 <= r["round"] <= det)
        assert ("fld_excluded" in r) == (r["round"] >= det) and r.get("fld_excluded", 2) == 2
    nv = eng.layout.n_vote
    args = eng.args
    for rnd, participants, wg, ws, after in seen:
        if rnd < det:
            continue
        keep = [j for j, a in enumerate(participants) if a >= 2]
        want = ops.fused_aggregate(wg.clone(), [ws[j] for j in keep], [float(eng.agent_data_sizes[participants[j]]) for j in keep], "avg",
                                   args.robustLR_threshold, args.server_lr, 0.0, args.seed, rnd, nv)
        assert torch.equal(after, want), rnd


def test_table_and_ring_equal_the_statements(full_run):
    eng, seen, _ = full_run
    nv = eng.layout.n_vote
    det = eng.aggregator.fld_detect_round
    table = torch.zeros(5, nv)
    ring = []
    for rnd, participants, wg, ws, _ in seen:
        if rnd > det:
            break
        for a, w in zip(participants, ws):
            table[a] = w[:nv] - wg[:nv]
        if rnd >= 2:
            ring.append(wg[:nv] - prev[:nv])
        prev = wg
    assert torch.equal(eng.fused.fld_table, table)
    chron = [eng.fused.fld_ring[(eng.aggregator.fld_pos + i) % 3] for i in range(3)]
    assert all(torch.equal(a, b) for a, b in zip(chron, ring[-3:]))
    assert torch.equal(eng.fused.fld_w_prev, seen[det - 1][2][:nv])


@pytest.mark.parametrize("stop", [3, 6])
def test_resume_is_bitwise(full_run, tmp_path, stop):
    """From a checkpoint in the warm-up (round 3: no scores yet) and from one after the detection (round 6)."""
    eng, _, hist = full_run
    ck = str(tmp_path / "ck.pt")
    first = _engine(rounds=stop, checkpoint=ck)
    first.fit()
    first.close()
    saved = torch.load(ck, weights_only=False)["extra"]["fldetector"]
    assert set(saved) == {"table", "ring", "w_prev", "count", "pos", "window", "flagged", "detect_round"}
    assert saved["table"].shape == (5, eng.layout.n_vote) and saved["ring"].shape == (3, eng.layout.n_vote)
    second = _engine(rounds=8, resume=ck)
    h2 = second.fit()
    assert torch.equal(second.w_global, eng.w_global)
    assert second.aggregator.fld_flagged == [0, 1] and second.aggregator.fld_detect_round == eng.aggregator.fld_detect_round
    assert [{k: v for k, v in r.items() if k.startswith("fld")} for r in h2] == \
           [{k: v for k, v in r.items() if k.startswith("fld")} for r in hist[stop:]]
    assert torch.equal(second.fused.fld_table, eng.fused.fld_table) and torch.equal(second.fused.fld_ring, eng.fused.fld_ring)
    second.close()


def test_checkpoint_without_state_is_rejected(tmp_path):
    ck = str(tmp_path / "none.pt")
    _engine(detect="none", fld_window=None, rounds=1, checkpoint=ck).fit()
    with pytest.raises(ValueError, match="no FLDetector state"):
        _engine(rounds=2, resume=ck)


@pytest.mark.parametrize("aggr", ["avg", "comed", "sign", "fltrust", "rfa", "flame", "foolsgold"])
def test_every_rule_runs_with_the_flagged_agents_excluded(aggr):
    kw = dict(aggr=aggr, rounds=6)
    if aggr == "sign":                   # a step of +-1 per coordinate moves every update far from its prediction: a sign-sized step
        kw.update(robustLR_threshold=2, server_lr=1e-3)
    eng = _engine(**kw)
    seen = _capture(eng)
    hist = eng.fit()
    assert eng.aggregator.fld_flagged == [0, 1], aggr
    assert hist[-1]["fld_excluded"] == 2 and torch.isfinite(eng.w_global).all()
    if aggr == "foolsgold":                                           # the flagged agents' histories stop changing
        det = eng.aggregator.fld_detect_round
        assert det < 6
        h = eng.fused.history
        nv = eng.layout.n_vote
        want = torch.zeros(2, nv)
        for rnd, participants, wg, ws, _ in seen:
            if rnd < det:
                for a, w in zip(participants, ws):
                    if a < 2:
                        want[a] = want[a] + (w[:nv] - wg[:nv])
        assert torch.equal(h[:2], want)
    if aggr in ("fltrust", "flame", "foolsgold"):
        assert all(i >= 2 for i in eng.aggregator.last_admitted)
    eng.close()


def _gloo_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    eng = _engine(rounds=6)
    hist = eng.fit()
    torch.save(dict(w=eng.w_global.clone(), hist=[{k: v for k, v in r.items() if k.startswith("fld")} for r in hist],
                    window=[torch.from_numpy(w) for w in eng.aggregator.fld_window], flagged=eng.aggregator.fld_flagged,
                    backend=eng.fused.backend), os.path.join(outdir, f"g{rank}.pt"))
    eng.close()
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_two_gloo_ranks_agree(tmp_path, full_run):
    mp.spawn(_gloo_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    outs = [torch.load(tmp_path / f"g{r}.pt", weights_only=False) for r in range(2)]
    assert outs[0]["backend"] == "gloo"
    for o in outs:
        assert torch.equal(o["w"], outs[0]["w"]) and o["hist"] == outs[0]["hist"] and o["flagged"] == [0, 1]
        assert all(torch.equal(a, b) for a, b in zip(o["window"], outs[0]["window"]))
    eng, _, hist = full_run
    assert outs[0]["hist"][eng.aggregator.fld_detect_round - 1]["fld_flagged"] == [0, 1]


def test_memory_refusal_names_the_bytes_and_the_flags():
    from rlr_b200.parallel.fused_agg import check_history_memory
    A, W, N = 3383, 1200128, 10
    assert check_history_memory(A, W, 1 << 40, N, foolsgold=False) == 4 * A * W + 4 * (N + 2) * W
    assert check_history_memory(A, W, 1 << 40, N) == 8 * A * W + 4 * (N + 2) * W
    with pytest.raises(ValueError) as e:
        check_history_memory(A, W, 8 << 30, N, foolsgold=False)
    msg = str(e.value)
    assert str(4 * A * W + 4 * (N + 2) * W) in msg and "--num_agents 3383" in msg and "--fld_window 10" in msg and str(8 << 30) in msg
