"""RFA on the H100: ``rfa_sqdist_kernel`` (ops/csrc/rfa.cu) against the fp64 statement for participant counts from 1 to the 1024 of the
kernel's tables, with and without clip scales, run-to-run bitwise equality, the fall-through above 1024 participants, the dict and slots
forms of the server step against the oracle with the same weights, a ResNet-18 engine run twice, and -- with two or more GPUs -- the
fused multi-GPU distance pass on both symmetric-memory providers and the engine with the fused hand-off against the barrier path."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.aggregation import Aggregation
from rlr_b200.options import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# fp32 values (one rounding more with clip scales), z in fp64 kept as an fp32 pair, fp32 squares summed over <= 128 coordinates per
# thread and folded into fp64.  Relative error of d_k^2 against the fp64 statement.  Measured on an H100 80GB HBM3 (700 W) over the
# cases below: at most 5.6e-9 without clip scales and 2.0e-8 with them (K = 200 and 1024; 0 at K = 1, where z = x exactly).
TOL = 1e-7


def _participants(K, n, seed, boost=True):
    """w_global and K participants around a common update, spread 1x..5x; with ``boost`` participant 0's update is scaled x100."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randn(n, generator=gen, device=DEV)
    mean = 0.01 * torch.randn(n, generator=gen, device=DEV)
    ws = [g + mean + 0.01 * (1 + k % 5) * torch.randn(n, generator=gen, device=DEV) for k in range(K)]
    if boost:
        ws[0] = g + 100.0 * (ws[0] - g)
    return g, ws


def _b(K, seed):
    b = np.random.default_rng(seed).uniform(0.1, 1.0, K)
    return b / b.sum()


def _rel(a, ref):
    a, ref = a.double().cpu(), ref.double().cpu()
    zero = ref == 0
    assert torch.equal(a[zero], ref[zero])
    return float(((a - ref).abs()[~zero] / ref[~zero]).max()) if (~zero).any() else 0.0


@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("K", [1, 2, 8, 33, 64, 65, 200, 1024])
def test_kernel_matches_fp64_statement(K, clip):
    ops.reset_fallbacks()
    n = 1 << 20 if K <= 65 else (1 << 18 if K <= 200 else 1 << 14)
    n_vote = n - 1024 if K <= 200 else n - 64                        # BatchNorm-style tail coordinates do not count
    g, ws = _participants(K, n, K + 3)
    for k, w in enumerate(ws):
        w[n_vote:] += 100.0 * (k + 1)                                # a leak past n_vote would dominate every distance
    b = _b(K, K)
    sc = torch.linspace(0.2, 1.0, K, device=DEV) if clip else None
    d2 = ops.rfa_sqdist(ws, b, n_vote, g if clip else None, sc)
    ref = ops.rfa_statement(ws, b, 0, n_vote, g if clip else None, sc)
    err = _rel(d2, ref)
    print(f"K={K} clip={clip}: max rel err of d^2 {err:.2e}")
    assert err <= TOL, err
    assert ops.fallback_calls() == {}


@pytest.mark.parametrize("K", [8, 40, 200])
def test_two_launches_are_bitwise_equal(K):
    ops.reset_fallbacks()
    n = 1 << 20 if K <= 40 else 1 << 18
    g, ws = _participants(K, n, 5)
    sc = torch.linspace(0.5, 1.0, K, device=DEV)
    for scales in (None, sc):
        a = ops.rfa_sqdist(ws, _b(K, 1), n - 256, g, scales)
        b = ops.rfa_sqdist(ws, _b(K, 1), n - 256, g, scales)
        torch.cuda.synchronize()
        assert torch.equal(a, b)
    assert ops.fallback_calls() == {}


def test_more_than_1024_participants_fall_through_to_the_statement():
    ops.reset_fallbacks()
    g, ws = _participants(1025, 256, 9)
    b = _b(1025, 2)
    d2 = ops.rfa_sqdist(ws, b, 256)
    assert torch.equal(d2, ops.rfa_statement(ws, b, 0, 256))
    assert list(ops.fallback_calls()) == ["rfa_sqdist"]
    ops.reset_fallbacks()


@pytest.mark.parametrize("theta,server_opt,select,clip", [(0, "sgd", "none", 0.0), (2, "sgd", "none", 0.0), (2, "adam", "none", 0.0),
                                                          (2, "sgd", "multikrum", 0.0), (2, "sgd", "none", 0.05),
                                                          (2, "sgd", "multikrum", 0.05)])
def test_dict_and_slots_forms_match_each_other_and_the_oracle(theta, server_opt, select, clip):
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ops.reset_fallbacks()
    K, n, nv = 10, 1 << 20, (1 << 20) - 4096
    g, ws = _participants(K, n, 21)
    sizes = {i: 100 + 13 * i for i in range(K)}
    a = make_args(num_agents=K, num_corrupt=1, aggr="rfa", robustLR_threshold=theta, server_opt=server_opt, server_lr=0.05, select=select,
                  clip=clip, server_clip=clip > 0, device=DEV)
    wg = g.clone()
    dict_form = Aggregation(sizes, n, None, a)
    dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
    fa = FusedAggregator(init_distributed(DEV), n, nv, K, "local", server_opt=dict(kind=server_opt, beta1=a.server_beta1,
                                                                                   beta2=a.server_beta2, tau=a.server_tau))
    fa.w_global.copy_(g)
    for j, w in enumerate(ws):
        fa.slots[j].copy_(w)
    slots_form = Aggregation(sizes, n, None, a, fused=fa)
    slots_form.aggregate_slots(list(range(K)), 1)
    torch.cuda.synchronize()
    assert torch.equal(fa.w_global, wg) and slots_form.last_rfa == dict_form.last_rfa
    assert slots_form.last_admitted == dict_form.last_admitted
    keep = list(dict_form.last_admitted) if select != "none" else list(range(K))
    if select != "none" and clip == 0:
        assert keep == list(range(1, K))                                   # the boosted participant 0 is what multikrum rejects
    norms = ops.update_norms(g, ws, nv)
    sc = (1.0 / torch.clamp(norms / clip, min=1.0)).float()[keep] if clip > 0 else None
    members = [ws[j] for j in keep]
    alpha = [float(sizes[j]) for j in keep]
    beta, F = ops.rfa(alpha, lambda b: ops.rfa_sqdist(members, b, nv, g if sc is not None else None, sc), 3, 1e-6)
    beta_ref, F_ref = ops.rfa(alpha, lambda b: ops.rfa_statement(members, b, 0, nv, g if sc is not None else None, sc), 3, 1e-6)
    np.testing.assert_allclose(beta, beta_ref, rtol=1e-6)
    np.testing.assert_allclose(F, F_ref, rtol=1e-6)
    assert F[1] <= F[0] and F[2] <= F[1]
    opt = ops.ServerOptState(server_opt, n, beta1=a.server_beta1, beta2=a.server_beta2, tau=a.server_tau, device=DEV)
    ref, _ = ops.aggregate_oracle(g, members, beta, "avg", theta, a.server_lr, None, nv, sc, opt)
    err = float((wg - ref).abs().max())
    print(f"theta={theta} {server_opt} {select} clip={clip}: max |w - oracle| {err:.2e}, F per pass {F}")
    assert err < 2e-6
    if select == "none" and clip == 0:
        assert dict_form.last_rfa["RFA/Corrupt_Weight"] < 0.02            # the boosted participant holds almost no weight
    assert ops.fallback_calls() == {}
    fa.close()


def test_engine_resnet18_rfa_is_reproducible():
    from rlr_b200.engine import FLEngine

    def run():
        ops.reset_fallbacks()
        args = make_args(data="cifar10", model="resnet18", num_agents=4, num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, synthetic=512,
                         synthetic_val=128, log_dir="", seed=3, aggr="rfa", robustLR_threshold=2, device=DEV)
        eng = FLEngine(args, verbose=False)
        out = []
        for r in range(1, 3):
            eng.run_round(r)
            out.append((eng.global_params().clone(), dict(eng.aggregator.last_rfa)))
        torch.cuda.synchronize()
        assert ops.fallback_calls() == {}
        eng.close()
        return out

    a, b = run(), run()
    for (wa, ra), (wb, rb) in zip(a, b):
        assert torch.equal(wa, wb) and ra == rb and ra["RFA/Passes"] == 3
    print("RFA/Corrupt_Weight per round:", [r["RFA/Corrupt_Weight"] for _, r in a])


# ---- two or more GPUs ------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# fused path: round 0 with the barrier-out, hand-off from round 1 on, so the passes of rounds 1-3 each follow an aggregate that published
# ready words instead of running a barrier-out; the clipped rounds (odd) read w_global and have to acquire it first
N_ROUNDS, HANDOFF_FROM = 4, 1


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
    n, nv, n_part = 1 << 20, (1 << 20) - 4096, 2 * world + 1
    slots = (n_part + world - 1) // world
    gen = torch.Generator().manual_seed(0)
    w0 = torch.randn(n, generator=gen)
    mean = 0.01 * torch.randn(n, generator=gen)
    parts = [w0 + mean + 0.01 * (1 + j % 3) * torch.randn(n, generator=gen) for j in range(n_part)]
    parts[0] = w0 + 100.0 * (parts[0] - w0)
    alpha = [float(100 + 7 * j) for j in range(n_part)]
    members = [j for j in range(n_part) if j != 1]                  # a member table that is not the round's full table
    res = {"fused": [], "nccl": [], "handoff": []}
    for backend in ("fused", "nccl"):
        fa = FusedAggregator(ctx, n, nv, slots, backend, transport="gather")
        for rnd in range(N_ROUNDS):
            if backend == "fused" and rnd == HANDOFF_FROM:
                fa.enable_handoff()
            if backend == "fused":
                res["handoff"].append(fa.handoff)
            w_in = w0 + 0.01 * rnd
            fa.w_global.copy_(w_in.to(ctx.device))
            jobs = [p + 0.01 * rnd for p in parts]
            for j, w in enumerate(jobs):
                r, s = fa.slot_owner(j)
                if r == ctx.rank:
                    fa.slots[s].copy_(w.to(ctx.device))
            torch.cuda.synchronize(); dist.barrier()
            copies = fa.gather_participants(n_part) if fa.gathers(n_part) else None
            scales = torch.linspace(0.5, 1.0, n_part, device=ctx.device) if rnd % 2 else None
            mem = members if rnd >= 2 else None
            idx = mem if mem is not None else list(range(n_part))
            beta, F = ops_.rfa([alpha[j] for j in idx], lambda b: fa.rfa_sqdist(n_part, b, scales, mem, copies), 3, 1e-6)
            weights = list(alpha)
            for j, bj in zip(idx, beta):
                weights[j] = bj
            fa.aggregate(weights, "avg", 2, 1.0, 0.0, 0, rnd, scales, members=mem, participants=copies, total_weight=sum(beta))
            fa.acquire()
            torch.cuda.synchronize()
            ref, _ = ops_.aggregate_oracle(w_in, [jobs[j] for j in idx], beta, "avg", 2, 1.0, None, nv,
                                           scales[idx].cpu() if scales is not None else None)
            res[backend].append(dict(beta=beta, F=F, err=float((fa.w_global.cpu() - ref).abs().max())))
            dist.barrier()
        fa.close()
    torch.save(res, os.path.join(outdir, f"rfa_{provider}_{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("provider", ["auto", "ipc"])
def test_fused_multi_gpu_rfa_passes(tmp_path, provider):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_multi_worker, args=(world, _free_port(), str(tmp_path), provider), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"rfa_{provider}_{r}.pt") for r in range(world)]
    assert res[0]["handoff"] == [rnd >= HANDOFF_FROM for rnd in range(N_ROUNDS)]
    for rnd in range(N_ROUNDS):
        f0 = res[0]["fused"][rnd]
        for r in range(world):
            fr, nr = res[r]["fused"][rnd], res[r]["nccl"][rnd]
            assert fr["beta"] == f0["beta"] and fr["F"] == f0["F"], (r, rnd)          # the same doubles on every rank
            assert fr["err"] < 2e-6 and nr["err"] < 2e-6, (r, rnd, fr["err"], nr["err"])
        np.testing.assert_allclose(f0["beta"], res[0]["nccl"][rnd]["beta"], rtol=1e-6)


# ---- the engine: rfa with the fused hand-off (the default) against --no_fused_handoff ---------------------------------------------------
def _engine_run(world, handoff):
    from rlr_b200.engine import FLEngine
    args = make_args(data="cifar10", model="cnn_cifar", synthetic=128 * max(5, 2 * world), synthetic_val=128, num_agents=max(5, 2 * world),
                     num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, log_dir="", seed=7, aggr="rfa", robustLR_threshold=2,
                     no_fused_handoff=not handoff, **({} if world > 1 else {"device": DEV}))
    eng = FLEngine(args, verbose=False)
    assert eng.handoff == handoff
    snaps, weights = [], []
    for r in range(1, 5):
        eng.run_round(r)                    # rounds 2-4: the passes follow a round whose aggregate ran the hand-off
        snaps.append(eng.global_params().clone().cpu())
        weights.append(eng.aggregator.last_rfa["RFA/Corrupt_Weight"])
    torch.cuda.synchronize()
    same = True
    if world > 1:
        allw = eng.ctx.all_gather(eng.global_params().clone())
        same = bool((allw == allw[0:1]).all().item())
    out = {"w": snaps, "corrupt_weight": weights, "same": same, "backend": eng.fused.backend}
    eng.close()
    return out


def _engine_worker(rank, world, port, outdir, handoff, tag):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    torch.save(_engine_run(world, handoff), os.path.join(outdir, f"eng_{tag}_{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("multi", [False, True])
def test_engine_rfa_with_fused_handoff_equals_barrier_path(tmp_path, multi):
    """Two barrier-path runs (a, b) measure the run-to-run noise of the native trainer; the hand-off run (f) must stay within that noise.
    multi: every GPU, one rank each, on the fused multi-GPU path."""
    world = min(torch.cuda.device_count(), 8) if multi else 1
    if multi and world < 2:
        pytest.skip("needs >= 2 GPUs")
    res = {}
    for tag, handoff in (("a", False), ("b", False), ("f", True)):
        if multi:
            mp.spawn(_engine_worker, args=(world, _free_port(), str(tmp_path), handoff, tag), nprocs=world, join=True)
            res[tag] = [torch.load(tmp_path / f"eng_{tag}_{r}.pt") for r in range(world)]
        else:
            res[tag] = [_engine_run(1, handoff)]
    if multi:
        assert res["f"][0]["backend"] == "fused"
    for t in "abf":
        for r in range(world):
            assert res[t][r]["same"] and res[t][r]["corrupt_weight"] == res[t][0]["corrupt_weight"], (t, r)
    print("corrupt weight per round:", res["a"][0]["corrupt_weight"])
    rel = lambda x, y: float((x.double() - y.double()).norm() / (y.double().norm() + 1e-12))
    for i in range(4):
        noise, diff = rel(res["b"][0]["w"][i], res["a"][0]["w"][i]), rel(res["f"][0]["w"][i], res["a"][0]["w"][i])
        print(f"world {world} round {i + 1}: barrier-vs-barrier {noise:.2e}  handoff-vs-barrier {diff:.2e}")
        assert diff <= 3 * noise + (1e-5 if i == 0 else 1e-4), (i, diff, noise)
