"""CRFL (``--param_clip`` / ``--param_noise`` / ``--certify``) on CPU: option validation, refusals and the banner; the Clopper-Pearson bound
against scipy; the abstain rule and the radius; ``ops.crfl_statement`` (the clip bound, the identity bit for bit, the padding and the
BatchNorm tail untouched, the noise on the real coordinates only); the Philox stream words kept apart from the aggregate, dropout and
augmentation streams; the in-process aggregation; engine runs with the torch trainer (two runs identical, resume bit for bit, ``certify()``
deterministic, tiny sigma giving the plain predictions); and 2 gloo ranks against one process for the training pass and the counts."""
import math
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.models import get_layout
from rlr_b200.options import make_args, print_exp_details

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- options ------------------------------------------------------------------------------------------------------------
def test_defaults_are_off_and_the_banner(capsys):
    a = make_args()
    assert a.param_clip == 0.0 and a.param_noise == 0.0 and not a.certify
    assert a.certify_n0 is None and a.certify_n is None and a.certify_alpha is None
    print_exp_details(a)
    out = capsys.readouterr().out
    assert "CRFL" not in out and "Certify" not in out
    b = make_args(param_clip=15, param_noise=0.01, certify=True)
    assert (b.certify_n0, b.certify_n, b.certify_alpha) == (100, 1000, 1e-3)
    print_exp_details(b)
    out = capsys.readouterr().out
    assert "CRFL (param clip rho / noise sigma): 15.0 / 0.01" in out and "Certify (n0 / n / alpha): 100 / 1000 / 0.001" in out
    c = make_args(param_noise=0.5, certify=True, certify_n0=3, certify_n=7, certify_alpha=0.05)
    assert (c.certify_n0, c.certify_n, c.certify_alpha) == (3, 7, 0.05)
    assert make_args(param_clip=2.0).param_noise == 0.0                      # either flag alone
    assert make_args(param_noise=2.0).param_clip == 0.0


@pytest.mark.parametrize("kw, match", [
    (dict(param_clip=-1.0), "--param_clip"), (dict(param_clip=float("inf")), "--param_clip"), (dict(param_clip=float("nan")), "--param_clip"),
    (dict(param_noise=-0.1), "--param_noise"), (dict(param_noise=float("inf")), "--param_noise"),
    (dict(certify=True), "needs --param_noise > 0"), (dict(certify=True, param_clip=3.0), "needs --param_noise > 0"),
    (dict(certify_n0=5), "need --certify"), (dict(certify_n=5, param_noise=0.1), "need --certify"),
    (dict(certify_alpha=0.1, param_noise=0.1), "need --certify"),
    (dict(certify=True, param_noise=0.1, certify_n0=0), "--certify_n0"), (dict(certify=True, param_noise=0.1, certify_n=0), "--certify_n "),
    (dict(certify=True, param_noise=0.1, certify_alpha=0.0), "--certify_alpha"),
    (dict(certify=True, param_noise=0.1, certify_alpha=1.0), "--certify_alpha"),
])
def test_refusals(kw, match):
    with pytest.raises(ValueError, match=match):
        make_args(**kw)


# ---- the certificate --------------------------------------------------------------------------------------------------------
def test_clopper_pearson_against_scipy():
    stats = pytest.importorskip("scipy.stats")
    for n in (1, 2, 7, 100, 1000):
        ks = sorted(set([0, 1, 2, n // 2, n - 1, n] + list(range(0, n + 1, max(1, n // 37)))))
        ks = [k for k in ks if 0 <= k <= n]
        for alpha in (1e-3, 0.05, 0.3):
            got = ops.clopper_pearson_lower(ks, n, alpha)
            for k, g in zip(ks, got):
                want = 0.0 if k == 0 else float(stats.beta.ppf(alpha, k, n - k + 1))
                assert abs(g - want) <= 1e-9, (n, k, alpha, g, want)
    assert ops.clopper_pearson_lower(5, 5, 0.01)[0] == pytest.approx(0.01 ** (1 / 5), abs=1e-12)
    with pytest.raises(ValueError):
        ops.clopper_pearson_lower([6], 5, 0.01)


def test_abstain_rule_and_radius():
    norm = pytest.importorskip("scipy.stats").norm
    n, alpha, sigma = 100, 0.01, 0.25
    sel = np.array([[3, 5, 0], [4, 4, 2], [0, 0, 0], [1, 0, 9], [10, 0, 0]])
    est = np.array([[0, 100, 0], [55, 45, 0], [0, 0, 0], [2, 1, 97], [40, 60, 0]])
    pred, radius, pa = ops.certify_decision(sel, est, n, alpha, sigma)
    want_pa = ops.clopper_pearson_lower([100, 55, 0, 97, 40], n, alpha)
    assert np.array_equal(pa, want_pa)
    # row 0: certain; row 1: tie in the selection goes to class 0, p_A(55) < 1/2 abstains; row 2: no votes abstains; row 3: class 2;
    # row 4: the selection picked class 0, whose estimate is 40 -> abstain even though class 1 has 60
    assert pred.tolist() == [1, -1, -1, 2, -1]
    for i in (0, 3):
        assert pa[i] > 0.5 and radius[i] == pytest.approx(sigma * norm.ppf(pa[i]), rel=1e-12)
    assert radius[[1, 2, 4]].tolist() == [0.0, 0.0, 0.0]
    labels = np.array([1, 0, 0, 0, 0])
    cert = ops.certified_accuracy(pred, radius, labels, sigma)
    assert cert[0] == 0.2 and cert == sorted(cert, reverse=True)
    big = radius[0] / sigma
    assert ops.certified_accuracy(pred, radius, labels, sigma, (big, big + 1e-6)) == [0.2, 0.0]


def test_vote_count_statement():
    logits = torch.tensor([[0.0, 2.0, 2.0], [5.0, 1.0, 5.0], [float("nan"), 1.0, 0.0], [1.0, float("inf"), 0.0], [-1.0, -2.0, -3.0]])
    counts = torch.zeros((7, 3), dtype=torch.int32)
    ops.vote_count(logits, counts, 2)
    ops.vote_count(logits[:2], counts, 0)
    want = torch.zeros((7, 3), dtype=torch.int32)
    want[0, 1] = want[1, 0] = want[2, 1] = want[3, 0] = want[6, 0] = 1
    assert torch.equal(counts, want)


# ---- the clip / noise statement ------------------------------------------------------------------------------------------------
def _vectors(model="cnn_cifar", seed=0, scale=1.0):
    lay = get_layout(model)
    rs = np.random.RandomState(seed)
    w = (scale * rs.randn(lay.n_total)).astype(np.float32)
    return lay, w, ops.real_mask(lay)


def test_real_mask_covers_exactly_the_parameters():
    for model in ("cnn_mnist", "resnet18"):
        lay = get_layout(model)
        m = ops.real_mask(lay)
        bits = ops.mask_bits(m, lay.n_vote)
        assert m.dtype == torch.int32 and m.numel() == ops.mask_words(lay.n_vote)
        assert int(bits.sum()) == lay.n_params
        for p in lay.params:
            assert bits[p.offset:p.offset + p.numel].all()


def test_clip_bounds_the_norm_and_rho_above_is_the_identity():
    lay, w, mask = _vectors("resnet18", scale=0.05)
    real = ops.mask_bits(mask, lay.n_vote).numpy()
    norm = float(np.sqrt(np.sum(w[:lay.n_vote][real].astype(np.float64) ** 2)))
    for rho in (1.0, 0.5 * norm, norm * (1 - 1e-6)):
        out, n_pre, s = ops.crfl_statement(w, mask, lay.n_vote, rho, 0.0, 7, ops.crfl_stream(1))
        assert n_pre == pytest.approx(norm, rel=1e-12) and s < 1.0
        after = float(np.sqrt(np.sum(out[:lay.n_vote][real].astype(np.float64) ** 2)))
        assert after <= rho * (1 + 4e-7)
        assert out[lay.n_vote:].tobytes() == w[lay.n_vote:].tobytes()
    for rho in (norm * (1 + 1e-6), 2 * norm, 0.0):
        out, _, s = ops.crfl_statement(w, mask, lay.n_vote, rho, 0.0, 7, ops.crfl_stream(1))
        assert s == 1.0 and out.tobytes() == w.tobytes()
    wz = w.copy()
    wz[:8] = -0.0                                                              # signed zeros survive s = 1, sigma = 0
    out, _, _ = ops.crfl_statement(wz, mask, lay.n_vote, 0.0, 0.0, 7, 1)
    assert out.tobytes() == wz.tobytes()


def test_norm_exactly_at_rho_is_not_scaled_and_nan_propagates():
    lay = get_layout("cnn_mnist")
    mask = ops.real_mask(lay)
    w = np.zeros(lay.n_total, dtype=np.float32)
    w[0], w[1] = 3.0, 4.0
    out, n_pre, s = ops.crfl_statement(w, mask, lay.n_vote, 5.0, 0.0, 1, 1)
    assert n_pre == 5.0 and s == 1.0 and out.tobytes() == w.tobytes()
    w[2] = np.nan
    out, n_pre, s = ops.crfl_statement(w, mask, lay.n_vote, 1.0, 0.1, 1, ops.crfl_stream(3))
    assert math.isnan(n_pre) and s == 1.0 and np.isnan(out[2]) and np.isfinite(np.delete(out, 2)).all()


def test_noise_touches_only_real_coordinates():
    lay, w, mask = _vectors("resnet18", seed=2)
    w[lay.n_vote:] = 1.25                                                      # the BatchNorm running statistics
    real = ops.mask_bits(mask, lay.n_vote).numpy()
    assert (~real).any()                                                       # resnet18 has alignment padding below n_vote
    sigma, seed, stream = 0.1, 11, ops.crfl_stream(4)
    out, _, s = ops.crfl_statement(w, mask, lay.n_vote, 0.0, sigma, seed, stream)
    assert s == 1.0
    v = w[:lay.n_vote]
    o = out[:lay.n_vote]
    assert o[~real].tobytes() == v[~real].tobytes() and out[lay.n_vote:].tobytes() == w[lay.n_vote:].tobytes()
    z = ops.philox_normals(seed, stream, lay.n_vote).astype(np.float32)
    want = (v + np.float32(sigma) * z).astype(np.float32)
    assert o[real].tobytes() == want[real].tobytes()
    d = (o[real].astype(np.float64) - v[real]) / sigma
    assert abs(d.mean()) < 5e-3 and abs(d.std() - 1.0) < 5e-3                # N(0, 1) noise
    # clip then noise: the scaled value plus the noise
    out2, _, s2 = ops.crfl_statement(w, mask, lay.n_vote, 1.0, sigma, seed, stream)
    assert s2 < 1.0
    want2 = ((v * np.float32(s2)).astype(np.float32) + np.float32(sigma) * z).astype(np.float32)
    assert out2[:lay.n_vote][real].tobytes() == want2[real].tobytes()


def test_box_muller_lanes_follow_the_philox_words():
    seed, stream = 3, ops.crfl_stream(2)
    z = ops.philox_normals(seed, stream, 8).reshape(2, 4)
    for q in range(2):
        u = [((int(x[0]) >> 8) + 1) / 2 ** 24 for x in ops.philox4x32([q], stream, seed)]
        r0, r1 = math.sqrt(-2 * math.log(u[0])), math.sqrt(-2 * math.log(u[2]))
        want = [r0 * math.cos(2 * math.pi * u[1]), r0 * math.sin(2 * math.pi * u[1]), r1 * math.cos(2 * math.pi * u[3]),
                r1 * math.sin(2 * math.pi * u[3])]
        assert np.allclose(z[q], want, rtol=1e-14, atol=1e-15)


def test_stream_words_stay_apart_from_every_other_stream():
    from rlr_b200.models.native import dropout_stream_base
    train = {ops.crfl_stream(r) for r in range(0, 2000)}
    cert = {ops.crfl_stream(m, certify=True) for m in range(0, 20000)}
    assert len(train) == 2000 and len(cert) == 20000 and not train & cert
    assert all(w >> 63 for w in train | cert)                                 # above every augmentation word and round number
    assert all((w >> 62) & 1 for w in cert) and not any((w >> 62) & 1 for w in train)
    aggregate = set(range(0, 1 << 20))                                          # the aggregate noise stream is the bare round number
    augment = {ops.augment_stream(s, a, r, e) for s in (0, 1, 5) for a in range(10) for r in range(1, 30) for e in range(3)}
    dropout = set()
    for s in (0, 1, 5):
        for a in range(10):
            for r in range(1, 30):
                base = dropout_stream_base(s, a, r)
                dropout.update((((base + k) << 20) ^ node) & (2 ** 64 - 1) for k in range(4) for node in range(8))
    for other in (aggregate, augment, dropout):
        assert not (train | cert) & other


def test_cpu_step_and_smooth_write_in_place():
    lay, w, mask = _vectors("cnn_mnist", seed=3)
    t = torch.from_numpy(w.copy())
    stats, wb = torch.zeros(2, dtype=torch.float64), torch.zeros(lay.n_total, dtype=torch.bfloat16)
    ref, norm, s = ops.crfl_statement(w, mask, lay.n_vote, 2.0, 0.01, 5, ops.crfl_stream(9))
    ops.crfl_step(t, t, mask, lay.n_vote, 2.0, 0.01, 5, 9, stats, wb)
    assert t.numpy().tobytes() == ref.tobytes() and torch.equal(wb, t.to(torch.bfloat16)) and stats.tolist() == [norm, s]
    out = torch.empty(lay.n_total)
    ops.crfl_smooth(torch.from_numpy(w), mask, lay.n_vote, 0.3, 5, 12, out)
    ref2, _, _ = ops.crfl_statement(w, mask, lay.n_vote, 0.0, 0.3, 5, ops.crfl_stream(12, certify=True))
    assert out.numpy().tobytes() == ref2.tobytes()


# ---- in-process aggregation ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("topk", [0.0, 0.05])
def test_in_process_aggregation_applies_the_pass_after_the_step(topk):
    from rlr_b200.aggregation import Aggregation
    lay = get_layout("cnn_mnist")
    n, nv = lay.n_total, lay.n_vote
    args = make_args(param_clip=3.0, param_noise=1e-3, robustLR_threshold=2, aggr="avg", server_topk=topk, seed=4)
    sizes = {i: 10 + i for i in range(4)}
    agg = Aggregation(sizes, lay.n_params, None, args, layout=lay)
    g = torch.Generator().manual_seed(9)
    w = 0.05 * torch.randn(n, generator=g)
    ref_w, ref_e = w.clone(), torch.zeros(nv)
    mask = ops.real_mask(lay)
    for rnd in (1, 2, 3):
        ws = {i: w + 0.01 * torch.randn(n, generator=g) for i in sizes}
        plain = ops.fused_aggregate(ref_w, [x - w + ref_w for x in ws.values()], [float(s) for s in sizes.values()], "avg", 2, 1.0,
                                    n_vote=nv, out=torch.empty(n))
        if topk:
            plain, e2, *_ = ops.sparsefed_statement(ref_w, plain, ref_e, nv, ops.sparsefed_k(topk, lay.n_params))
            ref_e = torch.from_numpy(e2)
        out, norm, s = ops.crfl_statement(plain, mask, nv, 3.0, 1e-3, 4, ops.crfl_stream(rnd))
        ref_w = torch.from_numpy(out)
        agg.aggregate_updates(w, {i: x - w + w for i, x in ws.items()}, rnd, n_vote=nv)
        assert torch.equal(w, ref_w)
        assert agg.last_crfl == {"param_norm": norm, "param_scale": s}


# ---- engine runs ----------------------------------------------------------------------------------------------------------
def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="fmnist", synthetic=800, synthetic_val=200, num_agents=4, local_ep=1, bs=64, device="cpu", num_corrupt=1,
                poison_frac=0.5, robustLR_threshold=2, log_dir="", seed=5, trainer="torch")
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


CRFL = dict(param_clip=9.0, param_noise=1e-3, rounds=3, certify=True, certify_n0=4, certify_n=12)


def test_engine_runs_are_identical_log_and_resume_bit_for_bit(tmp_path):
    a, b = _engine(**CRFL), _engine(**CRFL)
    ha, hb = a.fit(), b.fit()
    assert torch.equal(a.w_global, b.w_global)
    assert [h["param_norm"] for h in ha] == [h["param_norm"] for h in hb]
    assert any(h["param_scale"] < 1.0 for h in ha)                            # rho = 9 is below the model's norm
    last = ha[-1]
    for name in ("val", "poison"):
        assert len(last[f"certify_{name}_certified"]) == 5
        assert last[f"certify_{name}_acc"] == last[f"certify_{name}_certified"][0]
        assert last[f"certify_{name}_acc"] + last[f"certify_{name}_abstain"] <= 1.0
        assert last[f"certify_{name}_acc"] == hb[-1][f"certify_{name}_acc"]
        assert np.array_equal(a.last_certify[name]["estimation"], b.last_certify[name]["estimation"])
    assert "certify_val_acc" not in ha[0]
    ck = str(tmp_path / "ck.pt")
    first = _engine(checkpoint=ck, **{**CRFL, "rounds": 2, "certify": False, "certify_n0": None, "certify_n": None})
    first.fit()
    second = _engine(resume=ck, **CRFL)
    assert second.start_round == 3
    h2 = second.fit()
    assert torch.equal(second.w_global, a.w_global)
    assert h2[-1]["param_norm"] == ha[-1]["param_norm"] and h2[-1]["certify_val_acc"] == ha[-1]["certify_val_acc"]
    for e in (a, b, first, second):
        e.close()


def test_off_allocates_nothing():
    e = _engine(rounds=1)
    e.fit()
    assert e.fused.scratch is None and e.fused.crfl_mask is None and e.fused.crfl_stats is None and e.last_crfl is None
    e.close()


def test_certify_is_deterministic_and_tiny_sigma_gives_the_plain_predictions():
    e = _engine(rounds=2, param_noise=1e-7)
    e.fit()
    e.args.certify_n0, e.args.certify_n = 3, 10
    r1, r2 = e.certify(), e.certify()
    fwd = e.trainer.eval_forward(e.global_params())
    for name, ds in (("val", e.val_dataset), ("poison", e.poisoned_val)):
        for key in ("pred", "radius", "selection", "estimation"):
            assert np.array_equal(r1[name][key], r2[name][key])
        x, y = ds.batch(torch.arange(len(ds)))
        plain = fwd(x).argmax(1).numpy()
        assert np.array_equal(r1[name]["labels"], y.numpy())
        # every draw votes for the plain prediction: n_A = n, p_A = alpha^(1/n) > 1/2, so nothing abstains
        assert (r1[name]["estimation"].max(1) == 10).all() and np.array_equal(r1[name]["pred"], plain)
        assert r1[name]["abstain"] == 0.0
        assert r1[name]["acc"] == pytest.approx(float(np.mean(plain == y.numpy())))
    e.close()


# ---- 2 gloo ranks against one process ---------------------------------------------------------------------------------------
PASS_CASES = [("gather", "avg", 0), ("reduce", "sign", 0), ("gather", "avg", 40)]   # (transport, mode, SparseFed k)


def _run_pass(fa, rank, seed, n_part, mode):
    g = torch.Generator().manual_seed(seed)
    fa.w_global.copy_(0.05 * torch.randn(fa.n, generator=g))
    stats = []
    for rnd in (1, 2, 3):
        for j in range(n_part):
            a = fa.w_global + 0.01 * torch.randn(fa.n, generator=g)
            r, s = fa.slot_owner(j)
            if r == rank:
                fa.slots[s].copy_(a)
        fa.aggregate([float(10 + 3 * j) for j in range(n_part)], mode, 2, 0.25, 0.0, seed=5, rnd=rnd)
        stats.append(fa.crfl_stats.tolist())
    return fa.w_global.clone(), stats


CERT_KW = dict(data="fmnist", synthetic=400, synthetic_val=150, num_agents=2, local_ep=1, bs=64, device="cpu", num_corrupt=1,
               poison_frac=0.5, log_dir="", seed=6, trainer="torch", rounds=1, param_noise=0.05, certify=True, certify_n0=3, certify_n=8)


def _gloo_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed("cpu")
    lay = get_layout("cnn_mnist")
    out = {}
    for ci, (transport, mode, k) in enumerate(PASS_CASES):
        fa = FusedAggregator(ctx, lay.n_total, lay.n_vote, 2, "gloo", transport=transport, topk_k=k,
                             crfl=(2.0, 1e-3, ops.real_mask(lay)))
        out[ci] = _run_pass(fa, rank, ci, 4, mode)
        fa.close()
    eng = FLEngine(make_args(**CERT_KW), ctx=ctx, verbose=False)
    res = eng.certify()
    out["cert"] = {name: (res[name]["selection"], res[name]["estimation"]) for name in res}
    eng.close()
    torch.save(out, os.path.join(outdir, f"r{rank}.pt"))
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_ranks_equal_one_process(tmp_path):
    from rlr_b200.parallel import FusedAggregator
    from rlr_b200.parallel.comm import DistContext
    world = 2
    mp.spawn(_gloo_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"r{r}.pt", weights_only=False) for r in range(world)]
    lay = get_layout("cnn_mnist")
    for ci, (transport, mode, k) in enumerate(PASS_CASES):
        solo = FusedAggregator(DistContext(), lay.n_total, lay.n_vote, 4, "local", topk_k=k, crfl=(2.0, 1e-3, ops.real_mask(lay)))
        ref = _run_pass(solo, 0, ci, 4, mode)
        assert all(s[1] < 1.0 for s in ref[1])
        for o in outs:
            assert torch.equal(o[ci][0], ref[0]), transport
            assert o[ci][1] == ref[1]
    solo = _engine(**CERT_KW)
    res = solo.certify()
    for name in ("val", "poison"):
        assert res[name]["estimation"].sum() == 8 * len(res[name]["labels"])          # every row voted in every estimation draw
        for o in outs:
            assert np.array_equal(o["cert"][name][0], res[name]["selection"]) and np.array_equal(o["cert"][name][1], res[name]["estimation"])
    solo.close()
