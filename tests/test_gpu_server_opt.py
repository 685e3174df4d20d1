"""GPU: the server optimizers (momentum / adagrad / adam / yogi) in the fused aggregation kernel against the fp64 statement, on every
kernel path, with carried state; sgd equivalence; the sharded state layout; native ResNet-18 rounds; and (>= 2 GPUs) the fused P2P
path with per-rank state slices."""
import os
import socket
import sys

import pytest
import torch
import torch.multiprocessing as mp

import rlr_b200  # noqa: F401
from rlr_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ["momentum", "adagrad", "adam", "yogi"]
# vector kernels (avg / sign, median K <= 8), sorting networks (8 < K <= 64), shared-memory bisection (64 < K <= 320), L2 bisection
PATHS = ([(m, K, t) for m in ("avg", "sign") for K, t in ((1, 0), (5, 3), (64, 16), (1024, 300))] +
         [("comed", K, t) for K, t in ((1, 0), (2, 2), (5, 3), (8, 4), (9, 3), (12, 5), (16, 0), (17, 6), (24, 9), (32, 8), (40, 12),
                                       (48, 20), (64, 16), (65, 20), (200, 50), (321, 100), (1024, 300))])


def _agents(g, K, gen):
    n = g.numel()
    return [g + 0.1 * torch.randn(n, generator=gen) * (torch.rand(n, generator=gen) > 0.2) for _ in range(K)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mode,K,theta", PATHS)
def test_kernel_server_opt_matches_oracle(kind, mode, K, theta):
    n, n_vote = 8192, 6144
    gen = torch.Generator().manual_seed(K * 31 + theta + KINDS.index(kind))
    lr = 0.01 if mode == "sign" else 0.5
    ref_opt = ops.ServerOptState(kind, n, 0.9, 0.99, 1e-3)
    dev_opt = ops.ServerOptState(kind, n, 0.9, 0.99, 1e-3, device=DEV)
    g = torch.randn(n)
    wt = [float(100 + 13 * k) for k in range(K)]
    for rnd in range(3):
        ws = _agents(g, K, gen)
        ref, nflip = ops.aggregate_oracle(g, ws, wt, mode, theta, lr, None, n_vote, opt=ref_opt)
        flipped = torch.zeros(1, dtype=torch.int64, device=DEV)
        out = torch.empty(n, device=DEV)
        ops.fused_aggregate(g.to(DEV), [w.to(DEV) for w in ws], wt, mode, theta, lr, n_vote=n_vote, out=out, flipped=flipped,
                            opt=dev_opt)
        torch.testing.assert_close(out.cpu(), ref, atol=1e-6, rtol=1e-6)
        torch.testing.assert_close(dev_opt.m.cpu(), ref_opt.m, atol=1e-6, rtol=1e-6)
        if ref_opt.v is not None:
            torch.testing.assert_close(dev_opt.v.cpu(), ref_opt.v, atol=1e-6, rtol=1e-6)
        assert int(flipped.item()) == nflip
        assert torch.all(dev_opt.m[n_vote:] == 0)
        g = ref


@pytest.mark.parametrize("mode,K", [("avg", 5), ("sign", 5), ("comed", 5), ("comed", 12), ("comed", 100), ("comed", 400)])
def test_momentum_with_zero_beta_is_sgd_bitwise_on_device(mode, K):
    n, n_vote = 8192, 8000
    gen = torch.Generator().manual_seed(K)
    g = torch.randn(n).to(DEV)
    ws = [w.to(DEV) for w in _agents(g.cpu(), K, gen)]
    wt = [1.0 + k for k in range(K)]
    for theta, noise in ((0, 0.0), (3, 0.0), (3, 0.01)):
        a, b = torch.empty_like(g), torch.empty_like(g)
        fa, fb = torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
        ops.fused_aggregate(g, ws, wt, mode, theta, 0.3, noise, 7, 2, n_vote, out=a, flipped=fa)
        ops.fused_aggregate(g, ws, wt, mode, theta, 0.3, noise, 7, 2, n_vote, out=b, flipped=fb,
                            opt=ops.ServerOptState("momentum", n, beta1=0.0, device=DEV))
        assert torch.equal(a, b) and torch.equal(fa, fb)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mode,K", [("avg", 6), ("comed", 6), ("comed", 30), ("comed", 150), ("sign", 6)])
def test_sharded_state_launches_equal_one_full_launch(kind, mode, K):
    """Two launches over [0, per) and [per, n), each with its own state slice (state_base = begin), equal one launch over [0, n)."""
    n, n_vote, per = 8192, 7000, 4096
    gen = torch.Generator().manual_seed(K + 3)
    g = torch.randn(n).to(DEV)
    wt = [float(5 + k) for k in range(K)]
    full = ops.ServerOptState(kind, n, 0.8, 0.9, 1e-2, device=DEV)
    parts = [ops.ServerOptState(kind, per, 0.8, 0.9, 1e-2, device=DEV, base=0),
             ops.ServerOptState(kind, n - per, 0.8, 0.9, 1e-2, device=DEV, base=per)]
    for rnd in range(2):
        ws = [w.to(DEV) for w in _agents(g.cpu(), K, gen)]
        agents = ops.PtrTable([w.data_ptr() for w in ws], DEV, ws)
        wtt = torch.tensor(wt, dtype=torch.float64, device=DEV)
        a, b = torch.empty_like(g), torch.empty_like(g)
        fa, fb = torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
        for out, flipped, opt, lo, hi in ((a, fa, full, 0, n), (b, fb, parts[0], 0, per), (b, fb, parts[1], per, n)):
            outs = ops.PtrTable([out.data_ptr()], DEV)
            ops.ext().fused_aggregate(agents.tensor, wtt, None, float(sum(wt)), g.data_ptr(), outs.tensor, None, False, lo, hi, n_vote,
                                      ops.MODE_IDS[mode], 3, 0.2, 0.01, 1, rnd, flipped, None, None, 0, 1, 0, False,
                                      *ops.opt_launch_args(opt))
        assert torch.equal(a, b) and torch.equal(fa, fb)
        assert torch.equal(full.m, torch.cat([parts[0].m, parts[1].m]))
        if full.v is not None:
            assert torch.equal(full.v, torch.cat([parts[0].v, parts[1].v]))
        g = a.clone()


def test_native_resnet18_adam_rlr_rounds_are_bitwise_reproducible():
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args

    def run():
        ops.reset_fallbacks()
        eng = FLEngine(make_args(data="cifar10", model="resnet18", num_agents=3, local_ep=1, bs=64, synthetic=384, synthetic_val=64,
                                 log_dir="", device=DEV, seed=2, robustLR_threshold=2, server_opt="adam", server_lr=0.01), verbose=False)
        assert eng.trainer.name == "native"
        w0 = eng.global_params().clone()
        for r in (1, 2):
            eng.run_round(r)
        w = eng.global_params().clone()
        torch.cuda.synchronize()
        assert ops.fallback_calls() == {}, ops.fallback_calls()
        m, v = eng.fused.opt.m.clone(), eng.fused.opt.v.clone()
        eng.close()
        return w0, w, m, v
    a, b = run(), run()
    assert not torch.equal(a[0], a[1]) and a[2].abs().sum() > 0
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ---- >= 2 GPUs -------------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _p2p_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed()
    n, n_vote, n_part = 1 << 18, (1 << 18) - 1024, 2 * world + 1
    fa = FusedAggregator(ctx, n, n_vote, (n_part + world - 1) // world, "fused", server_opt=dict(kind="adam", beta1=0.9, beta2=0.99, tau=1e-3))
    assert fa.sharded and fa.opt.m.numel() == fa.end - fa.begin
    gen = torch.Generator().manual_seed(0)
    w = torch.randn(n, generator=gen)
    ref_opt = ops.ServerOptState("adam", n)
    errs = []
    fa.w_global.copy_(w.to(ctx.device))
    for rnd in range(3):
        parts = [w + 0.05 * torch.randn(n, generator=gen) for _ in range(n_part)]
        for j in range(n_part):
            r, s = fa.slot_owner(j)
            if r == ctx.rank:
                fa.slots[s].copy_(parts[j].to(ctx.device))
        torch.cuda.synchronize(); dist.barrier()
        weights = [float(50 + 7 * j) for j in range(n_part)]
        fa.aggregate(weights, "comed" if rnd == 1 else "avg", 3, 0.05, 0.0, 0, rnd)
        torch.cuda.synchronize()
        w, _ = ops.aggregate_oracle(w, parts, weights, "comed" if rnd == 1 else "avg", 3, 0.05, None, n_vote, opt=ref_opt)
        errs.append(float((fa.w_global.cpu() - w).abs().max()))
    m, v = fa.server_opt_state()
    allw = ctx.all_gather(fa.w_global)
    res = {"errs": errs, "m_err": float((m.cpu() - ref_opt.m).abs().max()), "v_err": float((v.cpu() - ref_opt.v).abs().max()),
           "same": bool((allw == allw[0:1]).all().item())}
    fa.close()
    # engine checkpoint at this world size, resumed at world 1 in the parent process
    args = make_args(data="fmnist", synthetic=1024, synthetic_val=128, num_agents=world, local_ep=1, bs=64, log_dir="", seed=5,
                     robustLR_threshold=2, server_opt="yogi", server_lr=0.01, rounds=2, checkpoint=os.path.join(outdir, "ck.pt"))
    eng = FLEngine(args, verbose=False)
    assert eng.fused.sharded
    eng.fit()
    res["ck_m"] = eng.fused.server_opt_state()[0].cpu()
    eng.close()
    torch.save(res, os.path.join(outdir, f"p2p{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


def test_fused_p2p_sharded_state_matches_oracle_and_resumes_at_world_1(tmp_path):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_p2p_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"p2p{r}.pt") for r in range(world)]
    for r in res:
        assert max(r["errs"]) < 2e-6 and r["m_err"] < 1e-6 and r["v_err"] < 1e-6 and r["same"], r
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    eng = FLEngine(make_args(data="fmnist", synthetic=1024, synthetic_val=128, num_agents=world, local_ep=1, bs=64, log_dir="", seed=5,
                             robustLR_threshold=2, server_opt="yogi", server_lr=0.01, rounds=3, resume=str(tmp_path / "ck.pt"),
                             device=DEV), verbose=False)
    assert eng.start_round == 3 and not eng.fused.sharded
    assert torch.equal(eng.fused.opt.m.cpu(), res[0]["ck_m"])
    eng.fit()
    assert torch.isfinite(eng.w_global).all()
    eng.close()
