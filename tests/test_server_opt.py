"""Server optimizers (``--server_opt`` momentum / adagrad / adam / yogi) on CPU: the fp64 statement against an independent
per-coordinate loop of the update equations, sgd equivalences, option validation, checkpoint / resume, and the gloo transports."""
import math
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.engine import FLEngine
from rlr_b200.options import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ["sgd", "momentum", "adagrad", "adam", "yogi"]


def _loop_round(g, ws, wt, mode, theta, lr, noise, n_vote, kind, b1, b2, tau, m, v):
    """One round, coordinate by coordinate, in Python floats (fp64); m / v are float32 numpy arrays updated in place."""
    n, K = len(g), len(ws)
    out = np.zeros(n, dtype=np.float32)
    tot = sum(wt)
    for i in range(n):
        gi = float(g[i])
        u = [float(w[i]) - gi for w in ws]
        mean = sum(wk * uk for wk, uk in zip(wt, u)) / tot
        if i >= n_vote:
            out[i] = gi + mean
            continue
        s = sum((uk > 0) - (uk < 0) for uk in u)
        agg = mean if mode == "avg" else sorted(u)[(K - 1) // 2] if mode == "comed" else float((s > 0) - (s < 0))
        a = agg + float(noise[i])
        d = a if (theta <= 0 or abs(s) >= theta) else -a
        if kind == "sgd":
            out[i] = gi + lr * d
            continue
        if kind == "momentum":
            m1 = b1 * float(m[i]) + d
            step = m1
        else:
            m1 = b1 * float(m[i]) + (1 - b1) * d
            v0 = float(v[i])
            if kind == "adagrad":
                v1 = v0 + d * d
            elif kind == "adam":
                v1 = b2 * v0 + (1 - b2) * d * d
            else:
                v1 = v0 - (1 - b2) * d * d * ((v0 > d * d) - (v0 < d * d))
            v[i] = v1
            step = m1 / (math.sqrt(v1) + tau)
        m[i] = m1
        out[i] = gi + lr * step
    return out


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mode", ["avg", "comed", "sign"])
@pytest.mark.parametrize("theta", [0, 3])
@pytest.mark.parametrize("noisy", [False, True])
def test_oracle_matches_per_coordinate_loop(kind, mode, theta, noisy):
    n, n_vote, K, lr, b1, b2, tau = 96, 80, 5, 0.3, 0.9, 0.99, 1e-3
    gen = torch.Generator().manual_seed(KINDS.index(kind) * 100 + len(mode) * 10 + theta + noisy)
    g = torch.randn(n, generator=gen)
    opt = ops.ServerOptState(kind, n, b1, b2, tau)
    m = np.zeros(n, dtype=np.float32)
    v = np.full(n, np.float32(tau * tau), dtype=np.float32)
    wt = [float(10 + 7 * k) for k in range(K)]
    for rnd in range(5):
        ws = [g + 0.05 * torch.randn(n, generator=gen) * (torch.rand(n, generator=gen) > 0.2) for _ in range(K)]
        noise = torch.zeros(n, dtype=torch.float64)
        if noisy:
            noise[:n_vote] = 0.01 * torch.randn(n_vote, generator=gen, dtype=torch.float64)
        ref = _loop_round(g.numpy(), [w.numpy() for w in ws], wt, mode, theta, lr, noise.numpy(), n_vote, kind, b1, b2, tau, m, v)
        got, _ = ops.aggregate_oracle(g, ws, wt, mode, theta, lr, noise if noisy else None, n_vote, opt=opt)
        torch.testing.assert_close(got, torch.from_numpy(ref), atol=1e-6, rtol=1e-6)
        if kind != "sgd":
            torch.testing.assert_close(opt.m, torch.from_numpy(m), atol=1e-6, rtol=1e-6)
            assert torch.all(opt.m[n_vote:] == 0), "BatchNorm-style tail coordinates carry no state"
        if opt.v is not None:
            torch.testing.assert_close(opt.v, torch.from_numpy(v), atol=1e-6, rtol=1e-6)
        g = got


@pytest.mark.parametrize("mode", ["avg", "comed", "sign"])
def test_momentum_with_zero_beta_is_sgd_bitwise(mode):
    n, n_vote, K = 4096, 4000, 6
    gen = torch.Generator().manual_seed(3)
    g = torch.randn(n, generator=gen)
    ws = [g + 0.1 * torch.randn(n, generator=gen) for _ in range(K)]
    wt = [1.0 + k for k in range(K)]
    noise = 0.02 * torch.randn(n, generator=gen, dtype=torch.float64)
    noise[n_vote:] = 0
    for theta, nz in ((0, None), (3, None), (3, noise)):
        opt = ops.ServerOptState("momentum", n, beta1=0.0)
        a, fa = ops.aggregate_oracle(g, ws, wt, mode, theta, 0.7, nz, n_vote)
        b, fb = ops.aggregate_oracle(g, ws, wt, mode, theta, 0.7, nz, n_vote, opt=opt)
        assert torch.equal(a, b) and fa == fb
        # the partials form (reduce transport) shares the same step
        if mode != "comed":
            vote, wsum = ops.aggregate_partials(g, ws, wt, n_vote)
            c, _ = ops.aggregate_from_partials(g, vote, wsum, sum(wt), mode, theta, 0.7, nz, n_vote,
                                               ops.ServerOptState("momentum", n, beta1=0.0))
            d, _ = ops.aggregate_from_partials(g, vote, wsum, sum(wt), mode, theta, 0.7, nz, n_vote)
            assert torch.equal(c, d)


def test_cpu_fused_aggregate_carries_state():
    n = 512
    g = torch.randn(n)
    ws = [g + 0.1 * torch.randn(n) for _ in range(3)]
    opt_a, opt_b = ops.ServerOptState("adam", n), ops.ServerOptState("adam", n)
    ref, _ = ops.aggregate_oracle(g, ws, [1, 2, 3], "avg", 0, 0.1, None, n, opt=opt_a)
    out = ops.fused_aggregate(g.clone(), ws, [1, 2, 3], "avg", 0, 0.1, opt=opt_b)
    assert torch.equal(out, ref) and torch.equal(opt_a.m, opt_b.m) and torch.equal(opt_a.v, opt_b.v)
    assert ops.ServerOptState("sgd", n).m is None and ops.ServerOptState("momentum", n).v is None


def test_options_validation_and_server_lr():
    assert make_args(aggr="avg", server_lr=0.5).server_lr == 1.0                       # reference rule kept for sgd
    assert make_args(aggr="sign", server_lr=0.5).server_lr == 0.5
    for aggr in ("avg", "comed", "sign"):
        assert make_args(aggr=aggr, server_lr=0.05, server_opt="adam").server_lr == 0.05
    for bad in (dict(server_opt="nesterov"), dict(server_opt="adam", server_beta1=1.0), dict(server_opt="yogi", server_beta2=-0.1),
                dict(server_opt="adagrad", server_tau=0.0), dict(server_opt="momentum", server_beta1=1.5)):
        with pytest.raises(ValueError):
            make_args(**bad)
    with pytest.raises(SystemExit):
        from rlr_b200.options import args_parser
        args_parser(["--server_opt", "lamb"])


def _engine(**kw):
    base = dict(data="fmnist", synthetic=1200, synthetic_val=300, num_agents=3, local_ep=1, bs=64, log_dir="", device="cpu",
                robustLR_threshold=2, server_opt="adam", server_lr=0.01, seed=4)
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def test_checkpoint_resume_is_bitwise_and_mismatch_raises(tmp_path, capsys):
    full = _engine(rounds=4)
    full.fit()
    ck = str(tmp_path / "ck.pt")
    first = _engine(rounds=2, checkpoint=ck)
    first.fit()
    saved = torch.load(ck, weights_only=False)["server_opt"]
    assert saved["server_opt"] == "adam" and saved["m"].shape == saved["v"].shape == (first.layout.n_total,)
    second = _engine(rounds=4, resume=ck)
    assert second.start_round == 3 and torch.equal(second.fused.opt.m, first.fused.opt.m)
    second.fit()
    assert torch.equal(second.w_global, full.w_global)
    assert torch.equal(second.fused.opt.m, full.fused.opt.m) and torch.equal(second.fused.opt.v, full.fused.opt.v)
    assert not torch.equal(full.fused.opt.m, torch.zeros_like(full.fused.opt.m))
    with pytest.raises(ValueError, match="server_opt"):
        _engine(resume=ck, server_opt="yogi")
    with pytest.raises(ValueError, match="beta1"):
        _engine(resume=ck, server_beta1=0.5)
    plain = str(tmp_path / "sgd.pt")
    _engine(rounds=1, checkpoint=plain, server_opt="sgd").fit()
    assert "server_opt" not in torch.load(plain, weights_only=False)
    with pytest.raises(ValueError, match="no server optimizer state"):
        _engine(resume=plain)
    # the banner names the optimizer only when it is not sgd
    capsys.readouterr()
    FLEngine(make_args(data="fmnist", synthetic=256, synthetic_val=64, num_agents=2, log_dir="", device="cpu"), verbose=True)
    assert "Server optimizer" not in capsys.readouterr().out
    FLEngine(make_args(data="fmnist", synthetic=256, synthetic_val=64, num_agents=2, log_dir="", device="cpu", server_opt="yogi"),
             verbose=True)
    assert "Server optimizer (beta1 / beta2 / tau): yogi" in capsys.readouterr().out


def test_in_process_aggregation_keeps_its_own_state():
    eng = _engine(rounds=1)
    n = eng.layout.n_total
    g = eng.w_global.clone()
    ws = {a: g + 0.01 * torch.randn(n) for a in range(3)}
    ref_opt = ops.ServerOptState("adam", n, 0.9, 0.99, 1e-3)
    for rnd in (1, 2):
        want, _ = ops.aggregate_oracle(g, list(ws.values()), [float(eng.agent_data_sizes[a]) for a in ws], "avg", 2, 0.01, None,
                                       eng.layout.n_vote, opt=ref_opt)
        eng.aggregator.aggregate_updates(g, ws, rnd)
        assert torch.equal(g, want)
    assert torch.equal(eng.aggregator.opt.m, ref_opt.m) and eng.fused.opt.m.abs().sum() == 0


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _transport_worker(rank, world, port, outdir, cases):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed("cpu")
    out = {}
    for ci, (n, n_vote, n_part, mode, theta, noise, kind) in enumerate(cases):
        max_slots = (n_part + world - 1) // world
        res = {}
        for transport in ("gather", "reduce"):
            fa = FusedAggregator(ctx, n, n_vote, max_slots, "gloo", transport=transport,
                                 server_opt=dict(kind=kind, beta1=0.8, beta2=0.95, tau=1e-2))
            g = torch.Generator().manual_seed(100 + ci)
            fa.w_global.copy_(torch.randn(n, generator=g))
            for rnd in (1, 2, 3):
                for j in range(n_part):
                    a = fa.w_global + 0.1 * torch.randn(n, generator=g)
                    r, s = fa.slot_owner(j)
                    if r == rank:
                        fa.slots[s].copy_(a)
                weights = [float(10 + 3 * j) for j in range(n_part)]
                fa.aggregate(weights, mode, theta, 0.05, noise, seed=5, rnd=rnd)
            m, v = fa.server_opt_state()
            res[transport] = (fa.w_global.clone(), m, v)
            fa.close()
        out[ci] = res
    torch.save(out, os.path.join(outdir, f"t{rank}.pt"))
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_transports_agree_with_server_optimizer_state(tmp_path):
    """gather and reduce transports (3 CPU ranks) give the same parameters and optimizer state, identical on every rank."""
    world = 3
    cases = [(4096, 4000, 5, "avg", 0, 0.0, "adam"), (4096, 4096, 4, "sign", 2, 0.0, "yogi"), (4096, 4032, 6, "avg", 3, 0.05, "momentum"),
             (4096, 4096, 5, "avg", 2, 0.0, "adagrad")]
    mp.spawn(_transport_worker, args=(world, _free_port(), str(tmp_path), cases), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"t{r}.pt") for r in range(world)]
    for ci in range(len(cases)):
        wg, mg, vg = outs[0][ci]["gather"]
        wr, mr, vr = outs[0][ci]["reduce"]
        torch.testing.assert_close(wr, wg, rtol=1e-6, atol=1e-6)
        torch.testing.assert_close(mr, mg, rtol=1e-6, atol=1e-6)
        if vg is not None:
            torch.testing.assert_close(vr, vg, rtol=1e-6, atol=1e-6)
        assert not torch.equal(mg, torch.zeros_like(mg))
        for o in outs[1:]:
            for t in ("gather", "reduce"):
                for x, y in zip(o[ci][t], outs[0][ci][t]):
                    assert (x is None and y is None) or torch.equal(x, y)
