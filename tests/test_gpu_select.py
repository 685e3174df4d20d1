"""Krum / Multi-Krum on the H100: ``pairwise_sqdist_kernel`` (ops/csrc/select.cu) against the fp64 statement for participant counts
from 3 to the 1024 of the kernel's tables, exact zeros between identical participants, run-to-run bitwise equality, multikrum with
M = K against no selection bit for bit, no library fall-throughs, and -- with two or more GPUs -- the fused multi-GPU distance pass
on both symmetric-memory providers."""
import os
import socket
import sys

import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.aggregation import Aggregation
from rlr_b200.options import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# fp32 differences and fp32 partial sums over <= 256 coordinates, folded into fp64.  Measured on an H100 80GB HBM3 (700 W): largest
# relative error 1.3e-7 and largest error relative to max(D) 1.0e-7 over the cases below (both at K = 1024; <= 3.2e-8 for K <= 200).
RTOL, ATOL_REL = 1e-5, 1e-7


def _participants(K, n, seed, sybils=True):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randn(n, generator=gen, device=DEV)
    ws = [g + torch.randn(n, generator=gen, device=DEV) * (0.01 * (1 + k % 7)) for k in range(K)]
    if sybils and K >= 3:
        ws[1] = ws[0].clone()                                          # bitwise-identical participants
        ws[2] = ws[0] + 1e-6 * torch.randn(n, generator=gen, device=DEV)   # a near-duplicate
    return g, ws


def _check(D, ref):
    err = (D - ref).abs()
    bound = RTOL * ref.abs() + ATOL_REL * float(ref.max())
    ok = bool((err <= bound).all())
    rel = float((err / ref.clamp_min(1e-300)).max())
    return ok, rel, float(err.max()) / max(float(ref.max()), 1e-300)


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("K", [3, 8, 10, 33, 40, 64, 65, 200, 1024])
def test_kernel_matches_fp64_statement(K, scaled):
    ops.reset_fallbacks()
    n = 1 << 20 if K <= 64 else (1 << 18 if K <= 200 else 1 << 14)
    n_vote = n - 1024 if K <= 200 else n - 64                        # BatchNorm-style tail coordinates do not count
    g, ws = _participants(K, n, K + 17 * scaled)
    for w in ws:
        w[n_vote:] += 100.0
    scales = (0.25 + torch.rand(K, device=DEV)).float() if scaled else None
    D = ops.pairwise_sqdist(ws, n_vote, g if scaled else None, scales)
    ref = ops.sqdist_statement(ws, 0, n_vote, g if scaled else None, scales)
    ok, rel, rel_max = _check(D, ref)
    print(f"K={K} scaled={scaled}: max rel err {rel:.2e}, max err / max D {rel_max:.2e}")
    assert ok, (rel, rel_max)
    assert torch.equal(D, D.T) and bool((D.diagonal() == 0).all())
    if not scaled:
        assert float(D[0, 1]) == 0.0
    assert ops.fallback_calls() == {}


def test_identical_participants_are_exactly_zero_apart():
    n = 1 << 18
    g, ws = _participants(12, n, 3, sybils=False)
    for j in (4, 7, 11):
        ws[j] = ws[2].clone()
    D = ops.pairwise_sqdist(ws, n)
    for a in (2, 4, 7, 11):
        for b in (2, 4, 7, 11):
            assert float(D[a, b]) == 0.0
    Ds = ops.pairwise_sqdist(ws, n, g, torch.full((12,), 0.5, device=DEV))     # equal clipping scales keep them identical
    assert float(Ds[2, 7]) == 0.0 and float(Ds[2, 3]) > 0.0


@pytest.mark.parametrize("K", [8, 40, 200])
def test_two_launches_are_bitwise_equal(K):
    n = 1 << 20 if K <= 40 else 1 << 18
    g, ws = _participants(K, n, 5)
    a = ops.pairwise_sqdist(ws, n - 256)
    b = ops.pairwise_sqdist(ws, n - 256)
    s = torch.rand(K, device=DEV) + 0.5
    c, d = ops.pairwise_sqdist(ws, n, g, s), ops.pairwise_sqdist(ws, n, g, s)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(c, d)


def test_more_than_1024_participants_fall_through_to_the_statement():
    ops.reset_fallbacks()
    g, ws = _participants(1025, 256, 9)
    D = ops.pairwise_sqdist(ws, 256)
    assert torch.equal(D, ops.sqdist_statement(ws, 0, 256))
    assert list(ops.fallback_calls()) == ["pairwise_sqdist"]
    ops.reset_fallbacks()


@pytest.mark.parametrize("aggr,theta,clip", [("avg", 0, 0.0), ("avg", 3, 0.0), ("comed", 2, 0.0), ("sign", 3, 0.0), ("avg", 2, 0.5)])
def test_multikrum_all_admitted_equals_no_selection_on_device(aggr, theta, clip):
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ops.reset_fallbacks()
    K, n, nv = 10, 1 << 20, (1 << 20) - 4096
    g, ws = _participants(K, n, 21)
    sizes = {i: 100 + 13 * i for i in range(K)}
    base = dict(num_agents=K, aggr=aggr, robustLR_threshold=theta, server_lr=0.01, clip=clip, server_clip=clip > 0, device=DEV)
    dict_form, slots_form = {}, {}
    for sel in ("none", "multikrum"):
        a = make_args(**base, **(dict(select=sel, select_m=K) if sel != "none" else {}))
        wg = g.clone()
        Aggregation(sizes, n, None, a).aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
        dict_form[sel] = wg
        fa = FusedAggregator(init_distributed(DEV), n, nv, K, "local")
        fa.w_global.copy_(g)
        for j in range(K):
            fa.slots[j].copy_(ws[j])
        agg = Aggregation(sizes, n, None, a, fused=fa)
        agg.aggregate_slots(list(range(K)), 1)
        slots_form[sel] = fa.w_global.clone()
        fa.close()
    torch.cuda.synchronize()
    assert torch.equal(dict_form["none"], dict_form["multikrum"])
    assert torch.equal(slots_form["none"], slots_form["multikrum"])
    assert ops.fallback_calls() == {}


def test_selected_round_matches_the_oracle_on_the_admitted_set():
    K, n, nv = 8, 1 << 20, (1 << 20) - 4096
    g, ws = _participants(K, n, 33, sybils=False)
    ws[0] = ws[0] + 0.5                                                   # far away: rejected
    sizes = {i: 100 + 13 * i for i in range(K)}
    a = make_args(num_agents=K, num_corrupt=1, aggr="avg", robustLR_threshold=2, device=DEV, select="multikrum")
    agg = Aggregation(sizes, n, None, a)
    wg = g.clone()
    agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
    assert agg.last_admitted == list(range(1, K))
    ref, _ = ops.aggregate_oracle(g, ws[1:], [sizes[i] for i in range(1, K)], "avg", 2, a.server_lr, None, nv)
    assert float((wg - ref).abs().max()) < 2e-6


# ---- two or more GPUs ------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# fused path: round 0 with the barrier-out, hand-off from round 1 on, so the distance passes of rounds 2 (clipped), 3 (unclipped) and
# 4 (clipped) each follow an aggregate that published ready words instead of running a barrier-out
N_ROUNDS, HANDOFF_FROM, SCALED_ROUNDS = 5, 1, (2, 4)


def _multi_worker(rank, world, port, outdir, provider):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200 import ops as ops_
    from rlr_b200.parallel import FusedAggregator, init_distributed
    from rlr_b200.parallel import symm as symm_mod
    ctx = init_distributed()
    if provider != "auto":  # force the CUDA-IPC provider (per-peer stores, no multicast)
        orig = symm_mod.SymmetricBuffer.__init__
        symm_mod.SymmetricBuffer.__init__ = lambda self, c, n, p="auto": orig(self, c, n, provider)
    n, nv, n_part = 1 << 20, (1 << 20) - 4096, 2 * world + 3
    slots = (n_part + world - 1) // world
    gen = torch.Generator().manual_seed(0)
    w0 = torch.randn(n, generator=gen)
    parts = [w0 + 0.02 * (1 + j % 3) * torch.randn(n, generator=gen) for j in range(n_part)]
    parts[0] = w0 + 0.5                                                   # far away: rejected
    parts[2] = parts[1].clone()                                           # a Sybil pair
    weights = [float(50 + 7 * j) for j in range(n_part)]
    f, m = 1, n_part - 1
    res = {"fused": [], "nccl": [], "handoff": []}
    for backend in ("fused", "nccl"):
        fa = FusedAggregator(ctx, n, nv, slots, backend, transport="gather")
        for rnd in range(N_ROUNDS):
            if backend == "fused" and rnd == HANDOFF_FROM:
                fa.enable_handoff()          # the aggregations publish ready words from here on; no barrier-out
            if backend == "fused":
                res["handoff"].append(fa.handoff)
            w_in = w0 + 0.01 * rnd
            fa.w_global.copy_(w_in.to(ctx.device))       # the previous round ended with acquire() + synchronize + barrier
            for j in range(n_part):
                r, s = fa.slot_owner(j)
                if r == ctx.rank:
                    fa.slots[s].copy_((parts[j] + 0.01 * rnd).to(ctx.device))
            torch.cuda.synchronize(); dist.barrier()
            scales = torch.linspace(0.6, 1.0, n_part, device=ctx.device) if rnd in SCALED_ROUNDS else None
            copies = fa.gather_participants(n_part) if fa.gathers(n_part) else None
            D = fa.pairwise_sqdist(n_part, scales, copies)                 # fused: its barrier-in right after a hand-off aggregate
            keep = ops_.krum_select(D, list(range(n_part)), f, m)
            fa.aggregate(weights, "avg", 2, 1.0, 0.0, 0, rnd, scales, members=keep, participants=copies)
            fa.acquire()
            torch.cuda.synchronize()
            ref, _ = ops_.aggregate_oracle(w_in, [parts[j] + 0.01 * rnd for j in keep], [weights[j] for j in keep], "avg", 2, 1.0,
                                           None, nv, scales[keep].cpu() if scales is not None else None)
            res[backend].append(dict(D=D.cpu(), keep=keep, err=float((fa.w_global.cpu() - ref).abs().max())))
            dist.barrier()
        fa.close()
    res["provider"] = provider
    torch.save(res, os.path.join(outdir, f"sel_{provider}_{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("provider", ["auto", "ipc"])
def test_fused_multi_gpu_distances_and_selection(tmp_path, provider):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_multi_worker, args=(world, _free_port(), str(tmp_path), provider), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"sel_{provider}_{r}.pt") for r in range(world)]
    assert res[0]["handoff"] == [rnd >= HANDOFF_FROM for rnd in range(N_ROUNDS)]
    for rnd in range(N_ROUNDS):
        f0 = res[0]["fused"][rnd]
        for r in range(world):
            fr, nr = res[r]["fused"][rnd], res[r]["nccl"][rnd]
            assert torch.equal(fr["D"], f0["D"]) and fr["keep"] == f0["keep"], (r, rnd)
            assert fr["err"] < 2e-6 and nr["err"] < 2e-6, (r, rnd, fr["err"], nr["err"])
        g0 = res[0]["nccl"][rnd]["D"]
        ok, rel, rel_max = _check(f0["D"], g0)
        assert ok, (rnd, rel, rel_max)
        assert f0["keep"] == res[0]["nccl"][rnd]["keep"] and 0 not in f0["keep"]
        assert float(f0["D"][1, 2]) == 0.0


# ---- the engine: --select with the fused hand-off (the default) against --no_fused_handoff -----------------------------------------------
def _engine_select_run(world, handoff):
    from rlr_b200.engine import FLEngine
    args = make_args(data="cifar10", model="cnn_cifar", synthetic=128 * max(5, 2 * world), synthetic_val=128, num_agents=max(5, 2 * world),
                     num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, log_dir="", seed=7, select="multikrum",
                     no_fused_handoff=not handoff, **({} if world > 1 else {"device": DEV}))
    eng = FLEngine(args, verbose=False)
    assert eng.handoff == handoff
    snaps, admitted = [], []
    for r in range(1, 5):
        eng.run_round(r)                    # rounds 2-4: the distance pass follows a round whose aggregate ran the hand-off
        snaps.append(eng.global_params().clone().cpu())
        admitted.append(list(eng.aggregator.last_admitted))
    torch.cuda.synchronize()
    same = True
    if world > 1:
        allw = eng.ctx.all_gather(eng.global_params().clone())
        same = bool((allw == allw[0:1]).all().item())
    out = {"w": snaps, "admitted": admitted, "same": same, "m": eng.args.select_m, "backend": eng.fused.backend}
    eng.close()
    return out


def _engine_select_worker(rank, world, port, outdir, handoff, tag):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    torch.save(_engine_select_run(world, handoff), os.path.join(outdir, f"eng_{tag}_{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("multi", [False, True])
def test_engine_select_with_fused_handoff_equals_barrier_path(tmp_path, multi):
    """Two barrier-path runs (a, b) measure the run-to-run noise of the native trainer; the hand-off run (f) must admit the same
    participants every round and stay within that noise.  multi: every GPU, one rank each, on the fused multi-GPU path."""
    world = min(torch.cuda.device_count(), 8) if multi else 1
    if multi and world < 2:
        pytest.skip("needs >= 2 GPUs")
    res = {}
    for tag, handoff in (("a", False), ("b", False), ("f", True)):
        if multi:
            mp.spawn(_engine_select_worker, args=(world, _free_port(), str(tmp_path), handoff, tag), nprocs=world, join=True)
            res[tag] = [torch.load(tmp_path / f"eng_{tag}_{r}.pt") for r in range(world)]
        else:
            res[tag] = [_engine_select_run(1, handoff)]
    if multi:
        assert res["f"][0]["backend"] == "fused"
    for t in "abf":
        for r in range(world):
            assert res[t][r]["same"] and res[t][r]["admitted"] == res["a"][0]["admitted"], (t, r)
            assert all(len(a) == res[t][r]["m"] for a in res[t][r]["admitted"])
    rel = lambda x, y: float((x.double() - y.double()).norm() / (y.double().norm() + 1e-12))
    for i in range(4):
        noise, diff = rel(res["b"][0]["w"][i], res["a"][0]["w"][i]), rel(res["f"][0]["w"][i], res["a"][0]["w"][i])
        print(f"world {world} round {i + 1}: barrier-vs-barrier {noise:.2e}  handoff-vs-barrier {diff:.2e}")
        assert diff <= 3 * noise + (1e-5 if i == 0 else 1e-4), (i, diff, noise)
