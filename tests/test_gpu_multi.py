"""Multi-GPU: the fused P2P aggregate+broadcast kernel (peer reads over NVLink, multicast / per-peer stores, in-kernel
flag barriers) against the fp64 oracle and against the NCCL all_gather baseline.  Needs >= 2 GPUs
(``python -m pytest tests/test_gpu_multi.py -m gpu`` on a multi-GPU machine); skips on one GPU."""
import os
import socket
import sys

import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _agg_worker(rank, world, port, outdir, provider):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200 import ops
    from rlr_b200.parallel import FusedAggregator, init_distributed
    from rlr_b200.parallel import symm as symm_mod
    ctx = init_distributed()
    if provider != "auto":  # force the CUDA-IPC provider (per-peer stores, no multicast)
        orig = symm_mod.SymmetricBuffer.__init__
        symm_mod.SymmetricBuffer.__init__ = lambda self, c, n, p="auto": orig(self, c, n, provider)
    n, n_vote, n_part = 1 << 20, (1 << 20) - 4096, 2 * world + 1   # uneven: rank 0 hosts one extra participant
    slots = (n_part + world - 1) // world
    fa = FusedAggregator(ctx, n, n_vote, slots, "fused")
    results = {"provider": fa.buf.provider, "multimem": fa.use_multimem}
    gen = torch.Generator().manual_seed(0)
    w0 = torch.randn(n, generator=gen)
    parts = [w0 + 0.05 * torch.randn(n, generator=gen) * (torch.rand(n, generator=gen) > 0.3) for _ in range(n_part)]
    weights = [float(50 + 7 * j) for j in range(n_part)]
    for case, (mode, theta, lr) in enumerate([("avg", 0, 1.0), ("avg", 3, 1.0), ("comed", 2, 1.0), ("sign", 3, 0.01)]):
        fa.w_global.copy_(w0.to(ctx.device))
        for j in range(n_part):
            r, s = fa.slot_owner(j)
            if r == ctx.rank:
                fa.slots[s].copy_(parts[j].to(ctx.device))
        torch.cuda.synchronize()
        for rep in range(3):   # repeated launches exercise the epoch-counted flag reuse; result is idempotent only for rep 0
            if rep > 0:
                fa.w_global.copy_(w0.to(ctx.device))
                torch.cuda.synchronize(); dist.barrier()
            fa.aggregate(weights, mode, theta, lr, 0.0, 0, case)
        torch.cuda.synchronize()
        ref, nflip = ops.aggregate_oracle(w0, parts, weights, mode, theta, lr, None, n_vote)
        got = fa.w_global.cpu()
        tot = fa.flipped.clone()
        dist.all_reduce(tot)
        results[f"{mode}-{theta}"] = dict(err=float((got - ref).abs().max()), flipped=int(tot.item()), flipped_ref=nflip,
                                          shadow_err=float((fa.w_bf16.float().cpu() - got.bfloat16().float()).abs().max()))
        dist.barrier()
    torch.save(results, os.path.join(outdir, f"agg{rank}.pt"))
    fa.close()
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("provider", ["auto", "ipc"])
def test_fused_p2p_aggregate_matches_oracle(tmp_path, provider):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_agg_worker, args=(world, _free_port(), str(tmp_path), provider), nprocs=world, join=True)
    for r in range(world):
        res = torch.load(tmp_path / f"agg{r}.pt")
        print(r, res["provider"], res["multimem"])
        for k, v in res.items():
            if isinstance(v, dict):
                assert v["err"] < 2e-6, (r, k, v)
                assert v["flipped"] == v["flipped_ref"], (r, k, v)
                assert v["shadow_err"] == 0.0, (r, k, v)


def _engine_worker(rank, world, port, outdir, backend):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    args = make_args(data="fmnist", synthetic=2048, synthetic_val=256, num_agents=world + 1, local_ep=1, bs=64, log_dir="",
                     robustLR_threshold=2, num_corrupt=1, poison_frac=0.5, backend=backend, trainer="torch", dtype="fp32", seed=5)
    eng = FLEngine(args, verbose=False)
    for r in range(1, 3):
        eng.run_round(r)
    ev = eng.evaluate(2)
    torch.save({"w": eng.w_global.cpu(), "acc": ev["val_acc"], "backend": eng.fused.backend, "provider": eng.fused.buf.provider},
               os.path.join(outdir, f"eng_{backend}_{rank}.pt"))
    eng.close()
    dist.barrier(); dist.destroy_process_group()


def test_engine_fused_equals_nccl_baseline(tmp_path):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    for backend in ("fused", "nccl"):
        mp.spawn(_engine_worker, args=(world, _free_port(), str(tmp_path), backend), nprocs=world, join=True)
    f = [torch.load(tmp_path / f"eng_fused_{r}.pt") for r in range(world)]
    n = [torch.load(tmp_path / f"eng_nccl_{r}.pt") for r in range(world)]
    for r in range(1, world):
        assert torch.equal(f[r]["w"], f[0]["w"]), "all ranks hold the same global params after the fused broadcast"
    # fused vs NCCL transport: identical participants/shards/seeds => same training up to nondeterministic cuDNN/atomics
    assert abs(f[0]["acc"] - n[0]["acc"]) < 0.2 and f[0]["backend"] == "fused" and n[0]["backend"] == "nccl"


def _handoff_worker(rank, world, port, outdir, fused, tag):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    # FedAvg without the (discontinuous) sign vote, ONE local step per agent and round: every step is a first step of the hand-off path
    args = make_args(data="cifar10", model="cnn_cifar", synthetic=64 * 2 * world, synthetic_val=128, num_agents=2 * world, local_ep=1, bs=64,
                     log_dir="", seed=7, no_fused_handoff=not fused)
    eng = FLEngine(args, verbose=False)
    assert eng.handoff == fused and eng.fused.backend == "fused"
    snaps = []
    for r in range(1, 4):
        eng.run_round(r)
        snaps.append(eng.global_params().clone())
    torch.cuda.synchronize()
    allw = eng.ctx.all_gather(snaps[-1])
    torch.save({"w": [s_.cpu() for s_ in snaps], "same": bool((allw == allw[0:1]).all().item())}, os.path.join(outdir, f"handoff_{tag}_{rank}.pt"))
    eng.close()
    dist.barrier(); dist.destroy_process_group()


def test_fused_handoff_across_gpus_equals_barrier_path(tmp_path):
    """Broadcast (+) first-GEMM fusion on >= 2 GPUs: the aggregation kernel publishes per-slice ready words instead of running its
    barrier-out, and the next round's stem GEMM reads the multicast bf16 shadow behind them.  Global parameters must be bit-identical
    across ranks, and equal to the barrier path up to the run-to-run noise of that path itself (split-K atomics order; dropout masks
    are a pure function of (seed, agent, round, step) in both)."""
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    for fused, tag in ((False, "a"), (False, "b"), (True, "f")):
        mp.spawn(_handoff_worker, args=(world, _free_port(), str(tmp_path), fused, tag), nprocs=world, join=True)
    res = {t: [torch.load(tmp_path / f"handoff_{t}_{r}.pt") for r in range(world)] for t in "abf"}
    for t in "abf":
        for r in range(world):
            assert res[t][r]["same"], "all ranks hold identical global parameters"
    rel = lambda x, y: float((x.double() - y.double()).norm() / (y.double().norm() + 1e-12))
    for i in (0, 2):
        noise, diff = rel(res["b"][0]["w"][i], res["a"][0]["w"][i]), rel(res["f"][0]["w"][i], res["a"][0]["w"][i])
        print(f"round {i + 1}: barrier-vs-barrier {noise:.2e}  fused-vs-barrier {diff:.2e}")
        assert diff <= 3 * noise + (1e-5 if i == 0 else 1e-4), (i, diff, noise)


def _stress_worker(rank, world, port, outdir, handoff, iters):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200 import ops
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed()
    n = 1 << 16
    fa = FusedAggregator(ctx, n, n, 1, "fused")
    if handoff:
        fa.enable_handoff()
    bad = 0
    # every iteration: each rank's slot := its rank + iteration (a constant vector), FedAvg of K = world participants, so the new
    # global parameters are known in closed form; any missed flag / stale read / torn broadcast shows up as a wrong value
    expect = torch.zeros((), dtype=torch.float64)
    fa.w_global.zero_()
    torch.cuda.synchronize(); dist.barrier()
    for it in range(iters):
        fa.slots[0].copy_(fa.w_global + float(rank + 1))          # reads w_global: must see the complete broadcast of iteration it-1
        if handoff:
            pass                                                  # (the copy above is stream-ordered after acquire() below)
        fa.aggregate([1.0] * world, "avg", 0, 1.0, 0.0, 0, it)
        fa.acquire()
        expect = expect + (world + 1) / 2.0
        if it % 97 == 0 or it == iters - 1:
            got = fa.w_global.double()
            bad += int((got - expect).abs().max().item() > 1e-3 * max(1.0, float(expect)))
    torch.cuda.synchronize()
    torch.save({"bad": bad, "final": float(fa.w_global[0]), "expect": float(expect)}, os.path.join(outdir, f"stress_{int(handoff)}_{rank}.pt"))
    fa.close()
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("handoff", [False, True])
def test_flag_protocol_stress_1000_epochs(tmp_path, handoff):
    """1000 back-to-back aggregations without host synchronisation: epoch-counted release/acquire flags (barrier-in, barrier-out or
    ready words) are reused every launch; a protocol error would corrupt the closed-form result."""
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_stress_worker, args=(world, _free_port(), str(tmp_path), handoff, 1000), nprocs=world, join=True)
    for r in range(world):
        res = torch.load(tmp_path / f"stress_{int(handoff)}_{r}.pt")
        assert res["bad"] == 0 and abs(res["final"] - res["expect"]) < 1e-3 * res["expect"], (r, res)
