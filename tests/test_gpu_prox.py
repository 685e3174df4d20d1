"""GPU: the local objectives (``--prox_mu``, ``--attack_constrain``) on the sm_90a optimizer kernels.

* the objective's norm pass and step (``sqnorm_kernel<., true>`` / ``sgd_step_kernel<., true>``, flat_sgd.cuh) against the fp64 statement of
  ``ops.objective_gradient`` over several grid sweeps: clipped and not, PGD off / inside / projected, masked, the ``||d|| = 0`` first step,
  the first step of a fused hand-off (NaN in w and m never read, the BatchNorm tail kept bit for bit), and bitwise repeats;
* the default objective: the same launches per step, and a native run bit for bit like one without the flags;
* engine runs on the native trainer: constrained corrupt agents against alpha = 1, a quiet round of a schedule, Neurotoxin's mask, FedProx
  with the FLTrust root job, reproducibility, captured graphs against eager steps, and learning like the torch trainer."""
import math

import numpy as np
import pytest
import torch

import rlr_b200  # noqa: F401
from rlr_b200 import ops
from rlr_b200.options import make_args

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24                 # unit roundoff of fp32


def _f32(x):
    return float(np.float32(x))


LR, MOM, MAX_NORM = _f32(0.1), _f32(0.9), 10.0
PGD_CLIP = {"off": 0.0, "inside": 64.0, "projected": 0.0625}
OBJECTIVES = {"prox": (1.0, 0.0, 0.5), "constrain": (0.7, 0.3, 0.0), "both": (0.6, 0.4, 0.25)}


def _sizes():
    """Two full sweeps of the optimizer kernels' capped grid (4 CTAs / SM x 256 threads x 4 coordinates) plus a remainder that is a
    multiple of 4 but not of 32, and n_pgd a multiple of 4 inside the second sweep and inside a 32-coordinate group."""
    S = torch.cuda.get_device_properties(0).multi_processor_count * 4 * 256 * 4
    n = 2 * S + (S // 2) // 8 * 8 + 4
    k = S + (S // 3) // 32 * 32 + 12
    assert n % 4 == 0 and n % 32 and k % 4 == 0 and k % 32
    return n, k


def _statement(w, g, m, w0, obj, clip, k, w_in=None, masked=None):
    """One objective step in fp64 from the kernel's own previous state, and per-coordinate bounds on the fp32 kernels' error.  Returns
    ``(w', m', (S_gg, S_gd, S_dd), ||w' - w0||^2 or None, bound_w, bound_m, rho)``.

    The objective's d and sums are those of ``ops.objective_gradient``: d = fp32(src - w0) is formed here exactly as the kernel forms it,
    so G = a g + beta d is exact in fp64.  The kernel rounds a g, beta, beta d and the sum (<= 3U (|a g| + |beta d|)), and its clip
    coefficient carries <= 5U relative (S_gg from fp32 squares, sqrt, + 1e-6f, the division), so with B = coef (|a g| + |beta d|):
      m' = mu m + coef G:  |dm| <= 8U |mu m| + 12U B = Em;   w' = w - lr m':  Ew = lr Em + U (lr |m'| + |w'|)
    and PGD as in test_gpu_flat_kernels.py.  The first-step variant reads w_in and zero momentum on [0, k) and leaves w[k:] alone."""
    src = w_in if w_in is not None else w
    a, b, mu = (_f32(x) for x in obj)
    g = g.clone()
    if masked is not None:
        g[:k][masked] = 0
    d32 = src[:k] - w0[:k]                                           # fp32, as the kernel
    if masked is not None:
        d32[masked] = 0
    g64, d = g.double(), d32.double()
    s_gg, s_gd, s_dd = float((g64 * g64).sum()), float((g64[:k] * d).sum()), float((d * d).sum())
    beta = (b / math.sqrt(s_dd) if s_dd > 0 else 0.0) + mu
    G = a * g64
    G[:k] += beta * d
    mag = (a * g64).abs()
    mag[:k] += (beta * d).abs()
    gn = math.sqrt(max(0.0, a * a * s_gg + 2 * a * beta * s_gd + beta * beta * s_dd))
    coef = min(1.0, MAX_NORM / (gn + 1e-6))
    assert coef == 1.0 and gn < MAX_NORM / 1.1 or gn > 1.1 * MAX_NORM, "keep the clip decision far from its edge"
    w64, m64 = w.double(), m.double()
    if w_in is None:
        am = MOM * m64
        m1 = am + coef * G
        w1 = w64 - LR * m1
    else:
        am = torch.zeros_like(m64)
        m1 = coef * G
        m1[k:] = 0
        w1 = w64.clone()
        w1[:k] = w_in[:k].double() - LR * m1[:k]
    em = 8 * U * am.abs() + 12 * U * coef * mag
    ew = LR * em + U * (LR * m1.abs() + w1.abs())
    if w_in is not None:
        em[k:] = 0
        ew[k:] = 0
    dsq, rho = None, 0.0
    if clip > 0:
        dd = w1[:k] - w0[:k].double()
        dsq = float((dd * dd).sum())
        r = math.sqrt(dsq)
        rho = float(ew[:k].norm()) / r + 3 * U
        assert r > 1.1 * clip or r < clip / 1.1, "keep the projection decision far from its edge"
        denom = max(1.0, r / clip)
        if denom > 1.0:
            inv = 1.0 / denom
            proj = w0[:k].double() + dd * inv
            ep = inv * (ew[:k] + U * dd.abs()) + (rho + 2 * U) * inv * dd.abs() + U * (inv * dd.abs() + proj.abs())
            if masked is not None:
                proj = torch.where(masked, w1[:k], proj)
                ep = torch.where(masked, ew[:k], ep)
            w1[:k] = proj
            ew[:k] = ep
    return w1, m1, (s_gg, s_gd, s_dd), dsq, ew, em, rho


def _check(opt, w, m, shadow, ref, n, shadow_upto=None):
    w1, m1, (s_gg, s_gd, s_dd), dsq, ew, em, rho = ref
    err_w = (w.cpu().double() - w1).abs()
    err_m = (m.cpu().double() - m1).abs()
    assert bool((err_w <= ew).all()), f"w: worst excess {float((err_w - ew).max()):.3e} at {int((err_w - ew).argmax())}"
    assert bool((err_m <= em).all()), f"m: worst excess {float((err_m - em).max()):.3e} at {int((err_m - em).argmax())}"
    sums = [float(x) for x in opt.norms[2:5]]
    # S_gg: fp32 squares and pair sums (2U relative); S_gd, S_dd: exact products; fp64 accumulation over n / 4 terms per thread + tree
    assert abs(sums[0] - s_gg) <= (2 * U + n * 2.0 ** -52) * s_gg, (sums[0], s_gg)
    assert abs(sums[2] - s_dd) <= n * 2.0 ** -52 * s_dd, (sums[2], s_dd)
    assert abs(sums[1] - s_gd) <= n * 2.0 ** -52 * math.sqrt(s_gg * s_dd), (sums[1], s_gd)
    if dsq is not None:
        n1 = float(opt.norms[1])
        assert abs(n1 - dsq) <= (2 * rho + rho * rho) * dsq, (n1, dsq)
    s = n if shadow_upto is None else shadow_upto
    assert torch.equal(shadow[:s], w[:s].bfloat16())


def _mask(k, gen):
    bits = torch.rand(k, generator=gen, device=DEV) < 0.2
    words = torch.from_numpy(np.packbits(np.concatenate([bits.cpu().numpy(), np.zeros(ops.mask_words(k) * 32 - k, bool)]),
                                         bitorder="little").view(np.int32).copy()).to(DEV)
    assert torch.equal(ops.mask_bits(words, k), bits)
    return bits, words


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("pgd", ["off", "inside", "projected"])
@pytest.mark.parametrize("clipped", [True, False])
@pytest.mark.parametrize("obj", list(OBJECTIVES))
def test_objective_step_over_several_sweeps_matches_fp64_statement(obj, clipped, pgd, masked):
    """Three steps from w = w0: the first has d = 0 (b / ||d|| := 0), the later ones the d the earlier steps made.  ||g|| ~ 30 sqrt(n)
    >> 10 (clipped) or ~ 3e-3 sqrt(n) ~ 3.5 << 10 (not clipped), and each unclipped step moves w[:n_pgd] by more than 1.1 x the
    projected case's radius."""
    n, k = _sizes()
    gen = torch.Generator(device=DEV).manual_seed(17 + len(obj) + 2 * clipped + len(pgd) + 5 * masked)
    w0 = torch.randn(n, generator=gen, device=DEV)
    w, m = w0.clone(), torch.zeros(n, device=DEV)
    shadow = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
    bits, words = _mask(k, gen) if masked else (None, None)
    opt = ops.FlatSGD(n, DEV, LR, MOM, MAX_NORM, PGD_CLIP[pgd], n_pgd=k)
    for step in range(3):
        g = torch.randn(n, generator=gen, device=DEV) * (30.0 if clipped else 3e-3)
        ref = _statement(w.cpu(), g.cpu(), m.cpu(), w0.cpu(), OBJECTIVES[obj], PGD_CLIP[pgd], k,
                         masked=bits.cpu() if masked else None)
        assert (ref[2][2] == 0.0) == (step == 0)
        opt.step(w, g, m, w0=w0, w_bf16=shadow, grad_mask=words, objective=OBJECTIVES[obj])
        _check(opt, w, m, shadow, ref, n)
    if masked:
        assert torch.equal(w[:k][bits].view(torch.int32), w0[:k][bits].view(torch.int32))


@pytest.mark.parametrize("same", [True, False])
@pytest.mark.parametrize("pgd", ["off", "projected"])
@pytest.mark.parametrize("obj", ["prox", "constrain"])
def test_first_step_reads_w_in_and_keeps_the_tail(obj, pgd, same):
    """``w_in``: parameters and d come from w_in -- the round's global parameters (``same``: w0 itself, so d = 0, as in every run) or
    a vector near it -- while w and m hold NaN on [0, n_pgd), which must never be read, and w[n_pgd:] is kept bit for bit."""
    n, k = _sizes()
    gen = torch.Generator(device=DEV).manual_seed(5 + len(obj) + len(pgd) + same)
    w0 = torch.randn(n, generator=gen, device=DEV)
    w_in = w0 if same else w0 + 1e-3 * torch.randn(n, generator=gen, device=DEV)
    w = torch.full((n,), float("nan"), device=DEV)
    w[k:] = 7.0 + torch.arange(n - k, device=DEV, dtype=torch.float32) * 1e-3
    tail = w[k:].clone()
    m = torch.full((n,), float("nan"), device=DEV)
    shadow = torch.full((n,), float("nan"), dtype=torch.bfloat16, device=DEV)
    g = torch.randn(n, generator=gen, device=DEV) * 30.0
    opt = ops.FlatSGD(n, DEV, LR, MOM, MAX_NORM, PGD_CLIP[pgd], n_pgd=k)
    ref = _statement(w.cpu(), g.cpu(), torch.zeros(n), w0.cpu(), OBJECTIVES[obj], PGD_CLIP[pgd], k, w_in=w_in.cpu())
    opt.step(w, g, m, w0=w0, w_bf16=shadow, w_in=w_in, objective=OBJECTIVES[obj])
    assert torch.equal(w[k:], tail) and bool((m[k:] == 0).all())
    _check(opt, w, m, shadow, ref, n, shadow_upto=None if pgd != "off" else k)


def test_objective_step_is_bitwise_reproducible():
    n, k = _sizes()
    gen = torch.Generator(device=DEV).manual_seed(3)
    w0 = torch.randn(n, generator=gen, device=DEV)
    w_start = w0 + 1e-3 * torch.randn(n, generator=gen, device=DEV)
    m_start = 1e-3 * torch.randn(n, generator=gen, device=DEV)
    g = torch.randn(n, generator=gen, device=DEV) * 30.0
    _, words = _mask(k, gen)
    runs = []
    for _ in range(4):
        w, m = w_start.clone(), m_start.clone()
        shadow = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
        opt = ops.FlatSGD(n, DEV, LR, MOM, MAX_NORM, PGD_CLIP["projected"], n_pgd=k)
        opt.step(w, g, m, w0=w0, w_bf16=shadow, grad_mask=words, objective=OBJECTIVES["both"])
        runs.append((w, m, shadow, opt.norms.clone()))
    assert float(runs[0][3][1]) > PGD_CLIP["projected"] ** 2 and float(runs[0][3][4]) > 0
    for r in runs[1:]:
        for x, y in zip(runs[0], r):
            assert torch.equal(x, y)


def test_objective_takes_the_launches_of_the_plain_step():
    n, k = _sizes()
    w0 = torch.randn(n, device=DEV)
    counts = []
    for obj in (None, OBJECTIVES["both"]):
        for pgd in ("off", "projected"):
            opt = ops.FlatSGD(n, DEV, LR, MOM, MAX_NORM, PGD_CLIP[pgd], n_pgd=k)
            w, m, g = w0.clone(), torch.zeros(n, device=DEV), torch.randn(n, device=DEV)
            c0 = ops.launch_calls()
            opt.step(w, g, m, w0=w0, objective=obj)
            counts.append(ops.launch_calls() - c0)
    assert counts[0:2] == counts[2:4]


# ---- engine runs on the native trainer ------------------------------------------------------------------------------------
def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="cifar10", model="cnn_cifar", synthetic=512, synthetic_val=128, num_agents=4, local_ep=1, bs=64, device=DEV,
                num_corrupt=1, poison_frac=0.5, robustLR_threshold=0, log_dir="", seed=5, diagnostics=True)
    base.update(kw)
    eng = FLEngine(make_args(**base), verbose=False)
    assert eng.trainer.name == "native"
    return eng


def _slots(eng, n_jobs):
    return [eng.fused.slots[eng.fused.slot_owner(j)[1]].clone() for j in range(n_jobs)]


def _update_norm(slot, w_g, nv):
    return float((slot[:nv].double() - w_g[:nv].double()).norm())


def test_defaults_given_explicitly_are_the_plain_run_bit_for_bit():
    a, b = _engine(), _engine(prox_mu=0.0, attack_constrain=1.0)
    for r in (1, 2):
        a.run_round(r); b.run_round(r)
    assert torch.equal(a.global_params(), b.global_params())
    assert a.trainer.launches_per_step() == b.trainer.launches_per_step() > 0
    a.close(); b.close()


def test_constrained_corrupt_agent_against_alpha_one():
    a, b = _engine(), _engine(attack_constrain=0.5, prox_mu=0.0)
    nv = a.layout.n_vote
    w_g = a.global_params().clone()
    ca, cb = a.run_round(1)["chosen"], b.run_round(1)["chosen"]
    assert ca == cb and 0 in ca
    sa, sb = _slots(a, len(ca)), _slots(b, len(cb))
    for j, agent in enumerate(ca):
        if agent < 1:
            assert _update_norm(sb[j], w_g, nv) < _update_norm(sa[j], w_g, nv)
        else:
            assert torch.equal(sb[j], sa[j])
    assert b.aggregator.last_norms["Norms/Avg_Corrupt_L2"] < a.aggregator.last_norms["Norms/Avg_Corrupt_L2"]
    assert a.trainer.launches_per_step() == b.trainer.launches_per_step()
    a.close(); b.close()


def test_a_quiet_round_trains_the_corrupt_agent_like_alpha_one():
    kw = dict(attack_start=2, attack_force=True)
    a, b = _engine(**kw), _engine(attack_constrain=0.5, **kw)
    ca, cb = a.run_round(1)["chosen"], b.run_round(1)["chosen"]
    assert ca == cb and 0 in ca
    assert all(torch.equal(x, y) for x, y in zip(_slots(a, len(ca)), _slots(b, len(cb))))
    ca, cb = a.run_round(2)["chosen"], b.run_round(2)["chosen"]
    assert not torch.equal(_slots(a, len(ca))[ca.index(0)], _slots(b, len(cb))[cb.index(0)])
    a.close(); b.close()


def test_constrained_neurotoxin_agent_keeps_the_mask():
    eng = _engine(attack_neurotoxin=0.02, attack_constrain=0.5, attack_boost=4.0, attack_force=True)
    nv = eng.layout.n_vote
    eng.run_round(1)
    w2 = eng.global_params().clone()
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
    w_g = a.global_params().clone()
    ca, cb = a.run_round(1)["chosen"], b.run_round(1)["chosen"]
    assert ca == cb
    for x, y in zip(_slots(a, len(ca) + 1), _slots(b, len(cb) + 1)):
        assert _update_norm(y, w_g, nv) < _update_norm(x, w_g, nv)
    a.close(); b.close()


def test_runs_are_reproducible():
    kw = dict(prox_mu=0.1, attack_constrain=0.6, attack_boost=3.0, clip=1.0)
    a, b = _engine(**kw), _engine(**kw)
    for r in (1, 2, 3):
        a.run_round(r); b.run_round(r)
    assert torch.equal(a.global_params(), b.global_params())
    a.close(); b.close()


def _resnet_run(**kw):
    from rlr_b200.engine import FLEngine
    ops.reset_fallbacks()
    args = make_args(data="cifar10", model="resnet18", num_agents=4, num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, synthetic=512,
                     synthetic_val=128, log_dir="", seed=3, robustLR_threshold=2, device=DEV, attack_constrain=0.5, prox_mu=0.01, **kw)
    eng = FLEngine(args, verbose=False)
    assert eng.trainer.name == "native"
    out = []
    for r in range(1, 3):
        chosen = eng.run_round(r)["chosen"]
        out.append((chosen, _slots(eng, len(chosen)), eng.global_params().clone()))
    torch.cuda.synchronize()
    assert ops.fallback_calls() == {}
    eng.close()
    return out


def test_native_graphs_equal_eager_steps_for_honest_and_constrained_agents():
    graphs = _resnet_run()
    eager = _resnet_run(no_graphs=True)
    for (ca, sa, wa), (cb, sb, wb) in zip(graphs, eager):
        assert ca == cb and 0 in ca and len(ca) > 1                   # one constrained corrupt agent, honest ones beside it
        for x, y in zip(sa, sb):
            assert torch.equal(x, y)
        assert torch.equal(wa, wb)


@pytest.mark.parametrize("model", ["resnet18", "cnn_cifar"])
def test_native_trainer_with_objectives_learns_like_torch_trainer(model):
    from rlr_b200.engine import FLEngine
    accs = {}
    for trainer in ("native", "torch"):
        args = make_args(data="cifar10", model=model, num_agents=2, local_ep=2, bs=64, synthetic=1000, synthetic_val=200, log_dir="",
                         device=DEV, trainer=trainer, seed=2, num_corrupt=1, poison_frac=0.1, prox_mu=0.01, attack_constrain=0.7)
        eng = FLEngine(args, verbose=False)
        for r in range(1, 11):
            eng.run_round(r)
        accs[trainer] = eng.evaluate(10)["val_acc"]
        assert eng.trainer.name == trainer
        eng.close()
    print(model, accs)
    assert accs["native"] > 0.85 and accs["torch"] > 0.85
