"""Local objectives (``--prox_mu``, FedProx; ``--attack_constrain``, constrain-and-scale) on CPU: option validation and the banner, the
optimizer step's CPU statement against autograd and ``torch.optim.SGD`` in fp64 (clipped and not, PGD off / inside / projected, masked,
the first step of a fused hand-off, the ``||d|| = 0`` rule), the default objective bit for bit, and engine runs (constrained corrupt
agents against alpha = 1, a quiet round of a schedule, Neurotoxin's mask, FedProx with the FLTrust root job, reproducibility)."""
import math

import numpy as np
import pytest
import torch

from rlr_b200 import ops
from rlr_b200.options import local_objective, make_args, print_exp_details


# ---- options ------------------------------------------------------------------------------------------------------------
def test_defaults_are_off_and_the_banner(capsys):
    a = make_args()
    assert a.prox_mu == 0.0 and a.attack_constrain == 1.0
    assert local_objective(a, True) is None and local_objective(a, False) is None
    print_exp_details(a)
    assert "Local objective" not in capsys.readouterr().out
    print_exp_details(make_args(prox_mu=0.01))
    assert "Local objective (prox mu / constrain alpha): 0.01 / 1.0" in capsys.readouterr().out
    print_exp_details(make_args(num_corrupt=1, attack_constrain=0.7))
    assert "Local objective (prox mu / constrain alpha): 0.0 / 0.7" in capsys.readouterr().out


def test_local_objective_per_agent():
    a = make_args(num_corrupt=1, attack_constrain=0.75, prox_mu=0.5)
    assert local_objective(a, True) == (0.75, 0.25, 0.5)
    assert local_objective(a, False) == (1.0, 0.0, 0.5)              # honest agents, the root job, quiet rounds
    b = make_args(num_corrupt=1, attack_constrain=0.75)
    assert local_objective(b, True) == (0.75, 0.25, 0.0) and local_objective(b, False) is None


@pytest.mark.parametrize("kw", [
    dict(prox_mu=-0.1), dict(prox_mu=float("inf")), dict(prox_mu=float("nan")),
    dict(attack_constrain=0.0), dict(attack_constrain=-0.5), dict(attack_constrain=1.5), dict(attack_constrain=float("nan")),
    dict(attack_constrain=float("inf")),
])
def test_rejects_out_of_range_values(kw):
    with pytest.raises(ValueError):
        make_args(num_corrupt=1, **kw)


def test_constrain_needs_corrupt_agents_and_prox_does_not():
    with pytest.raises(ValueError, match="num_corrupt"):
        make_args(num_corrupt=0, attack_constrain=0.5)
    make_args(num_corrupt=1, attack_constrain=0.5)
    make_args(num_corrupt=0, attack_constrain=1.0, prox_mu=0.1)


# ---- the step's CPU statement against autograd ----------------------------------------------------------------------------
N, K, LR, MOM, MAX_NORM = 600, 544, 0.1, 0.9, 10.0


def _autograd_steps(w_start, w0, gs, obj, pgd, masked=None, w_in=None):
    """The reference: per step, the autograd gradient of a <g_t, w> + b ||w - w0|| + (mu/2) ||w - w0||^2 over the model parameters
    [0, K) (g_t over every coordinate), Neurotoxin's mask, clip_grad_norm_(10), torch.optim.SGD(momentum), then PGD onto the ball of
    radius pgd around w0 (masked coordinates left alone).  ``w_in``: the first step starts from w_in on [0, K) and keeps w[K:]."""
    a, b, mu = obj
    p = torch.nn.Parameter((w_start if w_in is None else torch.cat([w_in[:K], w_start[K:]])).clone())
    sgd = torch.optim.SGD([p], lr=LR, momentum=MOM)
    for g in gs:
        sgd.zero_grad()
        d = p[:K] - w0[:K]
        loss = a * (g * p).sum() + b * torch.linalg.vector_norm(d) + mu / 2 * (d * d).sum()
        loss.backward()
        if masked is not None:
            p.grad[:K][masked] = 0
        torch.nn.utils.clip_grad_norm_([p], MAX_NORM)
        if w_in is not None:
            p.grad[K:] = 0                                           # the first step keeps the BatchNorm tail
        sgd.step()
        with torch.no_grad():
            if pgd > 0:
                d = p[:K] - w0[:K]
                denom = max(1.0, float(d.norm()) / pgd)
                if denom > 1.0:
                    proj = w0[:K] + d / denom
                    p[:K] = proj if masked is None else torch.where(masked, p[:K], proj)
    return p.detach()


def _mask(gen):
    bits = torch.rand(K, generator=gen) < 0.2
    words = torch.from_numpy(np.packbits(np.concatenate([bits.numpy(), np.zeros(ops.mask_words(K) * 32 - K, bool)]),
                                         bitorder="little").view(np.int32).copy())
    assert torch.equal(ops.mask_bits(words, K), bits)
    return bits, words


OBJECTIVES = {"prox": (1.0, 0.0, 0.5), "constrain": (0.7, 0.3, 0.0), "both": (0.6, 0.4, 0.25)}


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("pgd", ["off", "inside", "projected"])
@pytest.mark.parametrize("clipped", [True, False])
@pytest.mark.parametrize("obj", list(OBJECTIVES))
def test_cpu_statement_matches_autograd(obj, clipped, pgd, masked):
    """Three steps from w = w0: the first has d = 0 (b / ||d|| := 0, torch's subgradient there), the later ones a d that grows."""
    gen = torch.Generator().manual_seed(7 + len(obj) + 2 * clipped + len(pgd) + 5 * masked)
    w0 = torch.randn(N, generator=gen, dtype=torch.float64)
    scale = 2.0 if clipped else 0.01                                 # ||g|| ~ 49 (clipped) or ~ 0.25 (not clipped)
    gs = [torch.randn(N, generator=gen, dtype=torch.float64) * scale for _ in range(3)]
    bits, words = _mask(gen) if masked else (None, None)
    clip = {"off": 0.0, "inside": 100.0, "projected": 0.05}[pgd]
    opt = ops.FlatSGD(N, "cpu", LR, MOM, MAX_NORM, clip, n_pgd=K)
    w, m = w0.clone(), torch.zeros(N, dtype=torch.float64)
    for g in gs:
        opt.step(w, g, m, w0=w0, grad_mask=words, objective=OBJECTIVES[obj])
    ref = _autograd_steps(w0, w0, gs, OBJECTIVES[obj], clip, masked=bits)
    torch.testing.assert_close(w, ref, rtol=1e-12, atol=1e-13)
    assert not torch.equal(w, w0)
    if masked:
        assert torch.equal(w[:K][bits], w0[:K][bits])


@pytest.mark.parametrize("pgd", ["off", "projected"])
@pytest.mark.parametrize("obj", list(OBJECTIVES))
def test_cpu_first_step_reads_w_in(obj, pgd):
    """The first step of a fused hand-off: parameters and d come from w_in (here not w0, so d != 0), w's own values on [0, K) and the
    momentum are never read (NaN), w[K:] (BatchNorm statistics) is kept bit for bit."""
    gen = torch.Generator().manual_seed(31 + len(obj) + len(pgd))
    w0 = torch.randn(N, generator=gen, dtype=torch.float64)
    w_in = w0 + 0.05 * torch.randn(N, generator=gen, dtype=torch.float64)
    g = torch.randn(N, generator=gen, dtype=torch.float64) * 2.0
    w = torch.full((N,), float("nan"), dtype=torch.float64)
    w[K:] = 3.0 + torch.arange(N - K, dtype=torch.float64)
    tail = w[K:].clone()
    m = torch.full((N,), float("nan"), dtype=torch.float64)
    clip = {"off": 0.0, "projected": 0.05}[pgd]
    opt = ops.FlatSGD(N, "cpu", LR, MOM, MAX_NORM, clip, n_pgd=K)
    opt.step(w, g, m, w0=w0, w_in=w_in, objective=OBJECTIVES[obj])
    ref = _autograd_steps(w, w0, [g], OBJECTIVES[obj], clip, w_in=w_in)
    torch.testing.assert_close(w[:K], ref[:K], rtol=1e-12, atol=1e-13)
    assert torch.equal(w[K:], tail) and bool((m[K:] == 0).all())


def test_zero_distance_rule_and_the_statement():
    """At d = 0 the constrain term contributes nothing, so (alpha, 1 - alpha, 0) is alpha * CE there; past it beta = b / ||d|| + mu."""
    gen = torch.Generator().manual_seed(2)
    w0, g = torch.randn(N, generator=gen), torch.randn(N, generator=gen)
    G, gn, sums = ops.objective_gradient(g, w0.clone(), w0, (0.5, 0.5, 0.0), K)
    assert torch.equal(G, g * 0.5) and sums[1] == 0.0 and sums[2] == 0.0 and gn == pytest.approx(0.5 * float(g.double().norm()))
    w = w0 + 0.01 * torch.randn(N, generator=gen)
    G, gn, (s_gg, s_gd, s_dd) = ops.objective_gradient(g, w, w0, (0.5, 0.5, 0.25), K)
    d = (w[:K] - w0[:K]).double()
    beta = float(np.float32(0.5)) / math.sqrt(s_dd) + 0.25
    ref = 0.5 * g.double()
    ref[:K] += beta * d
    torch.testing.assert_close(G.double(), ref, rtol=1e-6, atol=1e-7)
    assert gn == pytest.approx(float(ref.norm()), rel=1e-12)


def test_default_objective_is_the_plain_step_bit_for_bit():
    gen = torch.Generator().manual_seed(4)
    w0, g = torch.randn(N, generator=gen), torch.randn(N, generator=gen)
    opt = ops.FlatSGD(N, "cpu", LR, MOM, MAX_NORM, 0.01, n_pgd=K)
    a, ma, b, mb = w0.clone(), torch.zeros(N), w0.clone(), torch.zeros(N)
    opt.step(a, g, ma, w0=w0)
    opt.step(b, g, mb, w0=w0, objective=(1.0, 0.0, 0.0))
    assert torch.equal(a, b) and torch.equal(ma, mb)
    with pytest.raises(ValueError, match="w0"):
        opt.step(b, g, mb, objective=(1.0, 0.0, 0.1))


# ---- engine runs ----------------------------------------------------------------------------------------------------------
def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="fmnist", synthetic=800, synthetic_val=200, num_agents=5, local_ep=1, bs=64, device="cpu", num_corrupt=1,
                poison_frac=0.5, robustLR_threshold=0, log_dir="", seed=5, trainer="torch", diagnostics=True)
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def _slots(eng, n_jobs):
    return [eng.fused.slots[eng.fused.slot_owner(j)[1]].clone() for j in range(n_jobs)]


def _update_norm(slot, w_g, nv):
    return float((slot[:nv].double() - w_g[:nv].double()).norm())


def test_defaults_given_explicitly_are_the_plain_run_bit_for_bit():
    a, b = _engine(), _engine(prox_mu=0.0, attack_constrain=1.0)
    for r in (1, 2):
        a.run_round(r); b.run_round(r)
    assert torch.equal(a.w_global, b.w_global)
    a.close(); b.close()


def test_constrained_corrupt_agent_against_alpha_one():
    a, b = _engine(), _engine(attack_constrain=0.5)
    nv = a.layout.n_vote
    w_g = a.w_global.clone()
    ca, cb = a.run_round(1)["chosen"], b.run_round(1)["chosen"]
    assert ca == cb and 0 in ca
    sa, sb = _slots(a, len(ca)), _slots(b, len(cb))
    for j, agent in enumerate(ca):
        if agent < 1:
            assert _update_norm(sb[j], w_g, nv) < _update_norm(sa[j], w_g, nv)
        else:
            assert torch.equal(sb[j], sa[j])                         # honest agents train on plain cross-entropy
    assert b.aggregator.last_norms["Norms/Avg_Corrupt_L2"] < a.aggregator.last_norms["Norms/Avg_Corrupt_L2"]
    assert b.aggregator.last_norms["Norms/Avg_Honest_L2"] == a.aggregator.last_norms["Norms/Avg_Honest_L2"]
    a.close(); b.close()


def test_a_quiet_round_trains_the_corrupt_agent_like_alpha_one():
    kw = dict(attack_start=2, attack_force=True)
    a, b = _engine(**kw), _engine(attack_constrain=0.5, **kw)
    ca, cb = a.run_round(1)["chosen"], b.run_round(1)["chosen"]
    assert ca == cb and 0 in ca and not b.last_attack_active
    assert all(torch.equal(x, y) for x, y in zip(_slots(a, len(ca)), _slots(b, len(cb))))
    assert torch.equal(a.w_global, b.w_global)
    ca, cb = a.run_round(2)["chosen"], b.run_round(2)["chosen"]     # the attack round
    j = ca.index(0)
    assert b.last_attack_active and not torch.equal(_slots(a, len(ca))[j], _slots(b, len(cb))[j])
    a.close(); b.close()


def test_constrained_neurotoxin_agent_keeps_the_mask():
    eng = _engine(attack_neurotoxin=0.02, attack_constrain=0.5, attack_force=True)
    nv = eng.layout.n_vote
    eng.run_round(1)
    w2 = eng.w_global.clone()
    chosen = eng.run_round(2)["chosen"]
    bits = ops.mask_bits(eng.attack_mask, nv)
    assert int(bits.sum()) > 0
    corrupt = _slots(eng, len(chosen))[chosen.index(0)]
    assert torch.equal(corrupt[:nv][bits].view(torch.int32), w2[:nv][bits].view(torch.int32))
    assert not torch.equal(corrupt[:nv], w2[:nv])
    eng.close()


def test_prox_shrinks_every_update_including_the_root_job():
    kw = dict(aggr="fltrust", root_size=100)
    a, b = _engine(**kw), _engine(prox_mu=2.0, **kw)
    nv = a.layout.n_vote
    w_g = a.w_global.clone()
    ca, cb = a.run_round(1)["chosen"], b.run_round(1)["chosen"]
    assert ca == cb
    sa, sb = _slots(a, len(ca) + 1), _slots(b, len(cb) + 1)          # position len(chosen): the FLTrust root job
    for x, y in zip(sa, sb):
        assert _update_norm(y, w_g, nv) < _update_norm(x, w_g, nv)
    a.close(); b.close()


def test_runs_are_reproducible():
    kw = dict(prox_mu=0.1, attack_constrain=0.6, attack_boost=3.0, clip=1.0)
    a, b = _engine(**kw), _engine(**kw)
    for r in (1, 2):
        a.run_round(r); b.run_round(r)
    assert torch.equal(a.w_global, b.w_global)
    a.close(); b.close()
