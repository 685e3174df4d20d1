"""Colluding attackers (``--attack_collude alie|minmax|minsum``) on CPU: option validation, defaults and the banner, the statement against
a per-coordinate numpy transcription of each paper's definition, the closed-form gamma* against the authors' bisection, the constraint
being met and tight, scale invariance in u, ALIE's z against scipy, every edge rule, engine rounds bit for bit against the statement,
quiet rounds, 2 ranks over gloo against one process, and the logged fields."""
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
from rlr_b200.options import make_args, print_exp_details

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIRS = ("backdoor", "std", "sign", "unit")


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- options ------------------------------------------------------------------------------------------------------------
def test_defaults_and_banner(capsys):
    a = make_args()
    assert (a.attack_collude, a.collude_dir, a.alie_z) == ("none", None, None)
    print_exp_details(a)
    assert "collude" not in capsys.readouterr().out
    b = make_args(num_corrupt=1, attack_collude="minmax")
    assert b.collude_dir == "backdoor" and b.alie_z is None
    c = make_args(num_corrupt=1, attack_collude="alie", collude_dir="std", alie_z=1.5)
    assert (c.collude_dir, c.alie_z) == ("std", 1.5)
    print_exp_details(b); print_exp_details(c); print_exp_details(make_args(num_corrupt=1, attack_collude="alie"))
    out = capsys.readouterr().out
    assert "Attack (collude / dir / z): minmax / backdoor / -" in out
    assert "Attack (collude / dir / z): alie / std / 1.5" in out
    assert "Attack (collude / dir / z): alie / backdoor / per round" in out


@pytest.mark.parametrize("kw", [
    dict(attack_collude="alie"),                                            # no corrupt agents
    dict(attack_collude="minmax", num_corrupt=1, attack_boost=2.0),
    dict(attack_collude="bogus", num_corrupt=1),
    dict(collude_dir="std"),                                                # direction without a mode
    dict(alie_z=1.0),
    dict(attack_collude="minsum", num_corrupt=1, alie_z=1.0),               # z without alie
    dict(attack_collude="alie", num_corrupt=1, collude_dir="sign"),
    dict(attack_collude="alie", num_corrupt=1, collude_dir="unit"),
    dict(attack_collude="minmax", num_corrupt=1, collude_dir="bogus"),
    dict(attack_collude="alie", num_corrupt=1, alie_z=-0.5),
    dict(attack_collude="alie", num_corrupt=1, alie_z=float("inf")),
    dict(attack_collude="alie", num_corrupt=1, alie_z=float("nan")),
])
def test_rejected(kw):
    with pytest.raises(ValueError):
        make_args(**kw)


def test_composes_with_neurotoxin_selection_detection_and_schedules():
    make_args(num_corrupt=1, attack_collude="minsum", collude_dir="sign", attack_neurotoxin=0.01, select="multikrum", num_agents=10)
    make_args(num_corrupt=1, attack_collude="alie", aggr="rfa", attack_start=2, attack_every=2)
    make_args(num_corrupt=1, attack_collude="minmax", detect="fldetector", num_agents=5)


# ---- the statement --------------------------------------------------------------------------------------------------------
def _vectors(K, nv, seed, scale=1e-2):
    g = torch.Generator().manual_seed(seed)
    w_g = torch.randn(nv + 8, generator=g)
    return w_g, [w_g + scale * torch.randn(nv + 8, generator=g) * (1 + k % 3) for k in range(K)]


def _numpy_paper(honest, corrupt, w_g, nv, mode, direction, z=None, gamma=None):
    """Per-coordinate transcription: mean, sample std, corrupt mean, direction and crafted value in float64, one coordinate at a time."""
    X = np.stack([w[:nv].numpy().astype(np.float64) for w in honest]) - w_g[:nv].numpy().astype(np.float64)
    Y = np.stack([w[:nv].numpy().astype(np.float64) for w in corrupt]) - w_g[:nv].numpy().astype(np.float64)
    H = len(honest)
    m = np.empty(nv)
    for c in range(nv):
        s = 0.0
        for j in range(H):
            s = s + X[j, c]
        mu = s / H
        v = 0.0
        for j in range(H):
            v = v + (X[j, c] - mu) * (X[j, c] - mu)
        sig = float(np.sqrt(v / (H - 1))) if H > 1 else 0.0
        t = 0.0
        for j in range(len(corrupt)):
            t = t + Y[j, c]
        xc = t / len(corrupt)
        u = {"std": sig, "sign": float(np.sign(mu)) + 0.0, "unit": mu, "backdoor": mu - xc}[direction]
        if mode == "alie":
            m[c] = mu - z * sig if direction == "std" else min(max(xc, mu - z * sig), mu + z * sig)
        else:
            m[c] = mu - gamma * u
    return (w_g[:nv].numpy().astype(np.float64) + m).astype(np.float32), X, m


@pytest.mark.parametrize("mode,direction", [("alie", "std"), ("alie", "backdoor")] + [(m, d) for m in ("minmax", "minsum") for d in DIRS])
def test_statement_matches_the_paper_definitions(mode, direction):
    nv = 64
    w_g, ws = _vectors(7, nv, 1)
    honest, corrupt = ws[:5], ws[5:]
    st = ops.collude_statement(honest, corrupt, w_g, nv, mode, direction)
    slot, X, m = _numpy_paper(honest, corrupt, w_g, nv, mode, direction, st["z"], st["gamma"])
    assert np.array_equal(st["slot"].numpy().view(np.uint32), slot.view(np.uint32))
    mu = X.mean(0)
    assert st["dev2"] == pytest.approx(float(((m - mu) ** 2).sum()), rel=1e-9, abs=1e-30)
    if mode != "alie":
        assert st["gamma"] > 0
        np.testing.assert_allclose(st["a"].numpy(), ((mu - X) ** 2).sum(1), rtol=1e-12)
    else:
        assert st["z"] == pytest.approx(ops.collude_z(5, 2))


def _bisection(constraint, mu, u):
    """The authors' search for gamma (initial 10, threshold 1e-5)."""
    lam, step, succ = 10.0, 10.0, 0.0
    while abs(succ - lam) > 1e-5:
        if constraint(mu - lam * u):
            succ = lam
            lam = lam + step / 2
        else:
            lam = lam - step / 2
        step /= 2
    return succ


def _dist_setup(K, nv, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(K, nv)) * rng.uniform(0.5, 2.0, size=(K, 1))
    mu = X.mean(0)
    D = ((X[:, None] - X[None]) ** 2).sum(-1)
    return X, mu, D


@pytest.mark.parametrize("mode", ["minmax", "minsum"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_closed_form_matches_the_bisection(mode, seed):
    X, mu, D = _dist_setup(6, 40, seed)
    a = ((mu - X) ** 2).sum(1)
    u = X.std(0, ddof=1)
    u = u * ops.collude_gamma(mode, a, ((mu - X) * u).sum(1), float((u * u).sum()), D) / 5.3   # gamma* near 5.3: inside the search
    e, q = ((mu - X) * u).sum(1), float((u * u).sum())
    g = ops.collude_gamma(mode, a, e, q, D)
    if mode == "minmax":
        ok = lambda m: ((m - X) ** 2).sum(1).max() <= D.max()              # noqa: E731
    else:
        ok = lambda m: ((m - X) ** 2).sum() <= D.sum(1).max()               # noqa: E731
    assert 0 < g < 10
    # the search stops once its step is below 1e-5; its last feasible gamma lies below gamma* by less than its last two steps
    assert 0 <= g - _bisection(ok, mu, u) <= 2e-5


@pytest.mark.parametrize("mode", ["minmax", "minsum"])
@pytest.mark.parametrize("seed", range(6))
def test_constraint_holds_and_is_tight(mode, seed):
    X, mu, D = _dist_setup(3 + seed, 30, seed)
    u = np.random.default_rng(100 + seed).normal(size=mu.size) * 3.0
    a, e, q = ((mu - X) ** 2).sum(1), ((mu - X) * u).sum(1), float((u * u).sum())
    m = mu - ops.collude_gamma(mode, a, e, q, D) * u
    lhs, rhs = (((m - X) ** 2).sum(1).max(), D.max()) if mode == "minmax" else (((m - X) ** 2).sum(), D.sum(1).max())
    assert lhs <= rhs * (1 + 1e-9)
    assert abs(lhs - rhs) <= 1e-6 * rhs


@pytest.mark.parametrize("mode", ["minmax", "minsum"])
def test_scaling_u_leaves_m_unchanged(mode):
    X, mu, D = _dist_setup(5, 30, 7)
    u = np.random.default_rng(3).normal(size=mu.size)
    ms = []
    for s in (1e-3, 1.0, 250.0):
        us = u * s
        g = ops.collude_gamma(mode, ((mu - X) ** 2).sum(1), ((mu - X) * us).sum(1), float((us * us).sum()), D)
        ms.append(mu - g * us)
    np.testing.assert_allclose(ms[0], ms[1], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(ms[2], ms[1], rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("H,C", [(1, 1), (3, 1), (7, 3), (10, 10), (2, 8), (27, 13), (4, 30)])
def test_alie_z_matches_scipy(H, C):
    from scipy.stats import norm
    K = H + C
    s = max(1, K // 2 + 1 - C)                                              # clamped at 1 once C > floor(K / 2)
    assert ops.collude_z(H, C) == pytest.approx(max(0.0, norm.ppf((K - s) / K)), abs=1e-12)


# ---- edge rules -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,direction", [("alie", "std"), ("alie", "backdoor"), ("minmax", "backdoor"), ("minsum", "std")])
def test_one_honest_participant_gives_its_update(mode, direction):
    nv = 32
    w_g, ws = _vectors(3, nv, 2)
    st = ops.collude_statement(ws[:1], ws[1:], w_g, nv, mode, direction, z=1.0 if mode == "alie" else None)
    assert st["dev2"] == 0.0 and (st["gamma"] in (None, 0.0))
    assert torch.equal(st["slot"], ws[0][:nv])


def test_gamma_edge_rules():
    a, e, D = np.array([1.0, 2.0]), np.array([0.5, -0.5]), np.array([[0.0, 4.0], [4.0, 0.0]])
    for mode in ("minmax", "minsum"):
        assert ops.collude_gamma(mode, a, e, 0.0, D) == 0.0                 # q = 0
        assert ops.collude_gamma(mode, a, e, float("nan"), D) == 0.0
        assert ops.collude_gamma(mode, a, e, 1.0, np.full((2, 2), np.nan)) == 0.0
        assert ops.collude_gamma(mode, np.array([np.inf, 1.0]), e, 1.0, D) == 0.0
    # a_k above Dmax by rounding and e_k < 0: the discriminant is clamped at 0 and gamma* stays >= 0
    assert ops.collude_gamma("minmax", np.array([4.0 + 1e-12, 0.0]), np.array([-1e-9, 0.0]), 1.0, D) == 0.0
    with pytest.raises(ValueError):
        ops.collude_gamma("alie", a, e, 1.0, D)


def test_a_non_finite_honest_value_is_left_out():
    nv = 16
    w_g, ws = _vectors(5, nv, 4)
    bad = [w.clone() for w in ws]
    bad[1][3] = float("nan")
    bad[2][5] = float("inf")
    ref = ops.collude_statement([ws[0], ws[3]] + [], ws[4:], w_g, nv, "alie", "std", z=1.0)
    st = ops.collude_statement(bad[:4], bad[4:], w_g, nv, "alie", "std", z=1.0)
    assert torch.isfinite(st["slot"]).all()
    # coordinate 3 keeps honest 0, 2, 3 and coordinate 5 keeps 0, 1, 3
    for c, keep in ((3, [0, 2, 3]), (5, [0, 1, 3])):
        one = ops.collude_statement([bad[j] for j in keep], bad[4:], w_g, nv, "alie", "std", z=1.0)
        assert st["slot"][c] == one["slot"][c]
    assert ref["slot"].shape == st["slot"].shape


# ---- engine runs ----------------------------------------------------------------------------------------------------------
def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="fmnist", synthetic=800, synthetic_val=200, num_agents=6, local_ep=1, bs=64, device="cpu", num_corrupt=2,
                poison_frac=0.5, robustLR_threshold=0, log_dir="", seed=5, trainer="torch")
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def _slots(eng, chosen):
    return {a: eng.fused.slots[eng.fused.slot_owner(j)[1]].clone() for j, a in enumerate(chosen)}


@pytest.mark.parametrize("mode,direction", [("alie", "backdoor"), ("alie", "std")] + [(m, d) for m in ("minmax", "minsum") for d in DIRS])
def test_engine_round_against_the_statement(mode, direction):
    a, b = _engine(), _engine(attack_collude=mode, collude_dir=direction)
    w_g = a.w_global.clone()
    ca, cb = a.run_round(1)["chosen"], b.run_round(1)["chosen"]
    assert ca == cb
    sa, sb = _slots(a, ca), _slots(b, cb)
    nv = a.layout.n_vote
    honest = [sa[x] for x in ca if x >= 2]
    corrupt = [sa[x] for x in ca if x < 2]
    assert honest and corrupt
    st = ops.collude_statement(honest, corrupt, w_g, nv, mode, direction)
    for agent in ca:
        if agent < 2:
            assert torch.equal(sb[agent][:nv], st["slot"])
            assert torch.equal(sb[agent][nv:], sa[agent][nv:])             # BatchNorm tail untouched
        else:
            assert torch.equal(sb[agent], sa[agent])
    rec = b.last_collude
    assert rec["collude_honest"] == len(honest)
    assert rec["collude_deviation"] == pytest.approx(st["dev2"] ** 0.5, rel=1e-9)
    assert ("collude_z" in rec) == (mode == "alie")
    a.close(); b.close()


def test_quiet_rounds_and_none_craft_nothing(monkeypatch):
    from rlr_b200.parallel.fused_agg import FusedAggregator
    calls = []
    real = FusedAggregator.collude
    monkeypatch.setattr(FusedAggregator, "collude", lambda self, *a, **k: calls.append(a) or real(self, *a, **k))
    plain, none = _engine(), _engine(attack_collude="none")
    for r in (1, 2):
        plain.run_round(r); none.run_round(r)
    assert torch.equal(plain.w_global, none.w_global) and calls == [] and none.last_collude is None
    sched = _engine(attack_collude="minmax", attack_start=2, attack_force=True)
    sched.run_round(1)
    assert calls == [] and sched.last_collude is None
    sched.run_round(2)
    assert len(calls) == 1 and sched.last_collude["collude_honest"] > 0
    for e in (plain, none, sched):
        e.close()


def test_no_corrupt_and_no_honest_participants():
    eng = _engine(attack_collude="minsum")
    assert eng._collude([2, 3, 4], 1) is None                              # C = 0: nothing launched
    eng.run_round(1)
    before = [s.clone() for s in eng.fused.slots]
    assert eng._collude([0, 1], 1) == {"collude_honest": 0}                # H = 0: nothing crafted
    assert all(torch.equal(x, y) for x, y in zip(before, eng.fused.slots))
    eng.close()


def test_composes_with_selection_and_defenses():
    for kw in (dict(select="multikrum", num_agents=8), dict(select="dnc", num_agents=8, dnc_dim=200), dict(aggr="rfa"),
               dict(aggr="flame", robustLR_threshold=0), dict(aggr="foolsgold")):
        eng = _engine(attack_collude="minmax", rounds=1, **kw)
        h = eng.fit()
        assert h[0]["collude_honest"] > 0 and np.isfinite(eng.w_global.numpy()).all()
        eng.close()


# ---- 2 ranks over gloo ------------------------------------------------------------------------------------------------------
def _gloo_worker(rank, world, port, outdir, transport):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args as mk
    eng = FLEngine(mk(data="fmnist", synthetic=800, synthetic_val=200, num_agents=4, local_ep=1, bs=64, device="cpu", num_corrupt=1,
                      poison_frac=0.5, log_dir="", seed=3, attack_collude="minmax", collude_dir="std", trainer="torch",
                      agg_transport=transport), verbose=False)
    devs = []
    for r in range(1, 3):
        eng.run_round(r)
        devs.append(eng.last_collude["collude_deviation"])
    torch.save({"w": eng.w_global.clone(), "devs": devs}, os.path.join(outdir, f"r{rank}.pt"))
    eng.close()
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("transport", ["gather", "reduce"])
def test_gloo_ranks_agree_with_one_process(tmp_path, transport):
    mp.spawn(_gloo_worker, args=(2, _free_port(), str(tmp_path), transport), nprocs=2, join=True)
    outs = [torch.load(os.path.join(tmp_path, f"r{r}.pt")) for r in range(2)]
    assert torch.equal(outs[0]["w"], outs[1]["w"]) and outs[0]["devs"] == outs[1]["devs"]
    from rlr_b200.engine import FLEngine
    one = FLEngine(make_args(data="fmnist", synthetic=800, synthetic_val=200, num_agents=4, local_ep=1, bs=64, device="cpu",
                             num_corrupt=1, poison_frac=0.5, log_dir="", seed=3, attack_collude="minmax", collude_dir="std",
                             trainer="torch"), verbose=False)
    devs = []
    for r in range(1, 3):
        one.run_round(r)
        devs.append(one.last_collude["collude_deviation"])
    np.testing.assert_allclose(devs, outs[0]["devs"], rtol=1e-6)
    torch.testing.assert_close(one.w_global, outs[0]["w"], rtol=1e-4, atol=1e-5)
    one.close()


def test_federated_py_logs_the_collude_fields(tmp_path):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "federated.py", "--data=fmnist", "--local_ep=1", "--bs=64", "--num_agents=10", "--rounds=2",
                        "--num_corrupt=2", "--poison_frac=0.5", "--synthetic=400", "--synthetic_val=80", "--attack_collude=alie",
                        "--select=multikrum", f"--log_dir={tmp_path}", "--device=cpu"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "Attack (collude / dir / z): alie / backdoor / per round" in r.stdout
    run_dirs = os.listdir(tmp_path)
    recs = [json.loads(l) for l in open(tmp_path / run_dirs[0] / "metrics.jsonl")]
    assert [rec["round"] for rec in recs] == [1, 2]
    for rec in recs:
        if "collude_honest" in rec:
            assert rec["collude_honest"] > 0 and rec["collude_deviation"] >= 0 and rec["collude_z"] >= 0
    assert any("collude_honest" in rec for rec in recs)
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    acc = EventAccumulator(str(tmp_path / run_dirs[0]))
    acc.Reload()
    tags = set(acc.Tags()["scalars"])
    assert {"Attack/Collude_Honest", "Attack/Collude_Deviation", "Attack/Collude_Z"} <= tags
