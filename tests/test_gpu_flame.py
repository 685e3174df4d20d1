"""FLAME on the H100: the Gram pass (``pairwise_sqdist_kernel<true>``, ops/csrc/select.cu) against the fp64 statement for participant counts
from 1 to the 1024 of the kernel's tables, run-to-run bitwise equality, the fall-through above 1024 participants, the dict and slots forms
of the server step against each other and the oracle, a ResNet-18 engine run twice, and -- with two or more GPUs -- the fused multi-GPU
Gram pass on both symmetric-memory providers and the engine with the fused hand-off against the barrier path."""
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
# Δ = w - w_global rounded once to fp32, fp32 products summed over <= 256 coordinates per thread and folded into fp64.  The bound is on
# the cosine: |G_ij - statement_ij| <= TOL * sqrt(G_ii G_jj), and the relative error of the diagonal (the squared norms) <= TOL.
# Measured on an H100 80GB HBM3 (700 W) over the cases below: at most 2.1e-8 up to K = 200 and 8.5e-8 at K = 1024.
TOL = 1e-6


def _participants(K, n, seed, boost=True):
    """w_global and K participants around a common update, spread 1x..5x; with ``boost`` participant 0's update is scaled x100."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randn(n, generator=gen, device=DEV)
    mean = 0.01 * torch.randn(n, generator=gen, device=DEV)
    ws = [g + mean + 0.01 * (1 + k % 5) * torch.randn(n, generator=gen, device=DEV) for k in range(K)]
    if boost:
        ws[0] = g + 100.0 * (ws[0] - g)
    return g, ws


def _errors(G, ref):
    G, ref = G.double().cpu(), ref.double().cpu()
    q = torch.diagonal(ref)
    cos_err = float(((G - ref).abs() / torch.sqrt(torch.outer(q, q))).max())
    diag_err = float(((torch.diagonal(G) - q).abs() / q).max())
    return cos_err, diag_err


@pytest.mark.parametrize("K", [1, 2, 8, 33, 64, 65, 200, 1024])
def test_kernel_matches_fp64_statement(K):
    ops.reset_fallbacks()
    n = 1 << 20 if K <= 65 else (1 << 18 if K <= 200 else 1 << 14)
    n_vote = n - 1024 if K <= 200 else n - 64                        # BatchNorm-style tail coordinates do not count
    g, ws = _participants(K, n, K + 3)
    for k, w in enumerate(ws):
        w[n_vote:] += 100.0 * (k + 1)                                # a leak past n_vote would dominate every entry
    G = ops.pairwise_gram(ws, g, n_vote)
    ref = ops.gram_statement(ws, g, 0, n_vote)
    assert G.shape == (K, K) and G.dtype == torch.float64
    assert torch.equal(G, G.T)
    cos_err, diag_err = _errors(G, ref)
    print(f"K={K}: max |dG| / sqrt(G_ii G_jj) {cos_err:.2e}, max rel err of the diagonal {diag_err:.2e}")
    assert cos_err <= TOL and diag_err <= TOL, (cos_err, diag_err)
    assert ops.fallback_calls() == {}


@pytest.mark.parametrize("K", [8, 40, 200])
def test_two_launches_are_bitwise_equal(K):
    ops.reset_fallbacks()
    n = 1 << 20 if K <= 40 else 1 << 18
    g, ws = _participants(K, n, 5)
    a = ops.pairwise_gram(ws, g, n - 256)
    b = ops.pairwise_gram(ws, g, n - 256)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    assert ops.fallback_calls() == {}


def test_more_than_1024_participants_fall_through_to_the_statement():
    ops.reset_fallbacks()
    g, ws = _participants(1025, 256, 9)
    G = ops.pairwise_gram(ws, g, 256)
    assert torch.equal(G, ops.gram_statement(ws, g, 0, 256))
    assert list(ops.fallback_calls()) == ["pairwise_gram"]
    ops.reset_fallbacks()


def _colluding_round(K, n, seed):
    """Participants 0..2 push one direction, the rest another; participant 3's honest update is boosted x100."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randn(n, generator=gen, device=DEV)
    honest, evil = torch.randn(n, generator=gen, device=DEV), torch.randn(n, generator=gen, device=DEV)
    ws = []
    for k in range(K):
        u = (evil if k < 3 else honest) + 0.3 * torch.randn(n, generator=gen, device=DEV)
        ws.append(g + 0.01 * (1 + 0.2 * k) * (100.0 if k == 3 else 1.0) * u)
    return g, ws


@pytest.mark.parametrize("theta,server_opt,select,lam", [(0, "sgd", "none", 0.0), (2, "sgd", "none", 0.0), (2, "adam", "none", 0.0),
                                                         (2, "sgd", "multikrum", 0.0), (2, "sgd", "none", 1e-3),
                                                         (2, "sgd", "multikrum", 1e-3)])
def test_dict_and_slots_forms_match_each_other_and_the_oracle(theta, server_opt, select, lam):
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ops.reset_fallbacks()
    K, n, nv = 10, 1 << 20, (1 << 20) - 4096
    g, ws = _colluding_round(K, n, 21)
    sizes = {i: 100 + 13 * i for i in range(K)}
    a = make_args(num_agents=K, num_corrupt=3, aggr="flame", robustLR_threshold=theta, server_opt=server_opt, server_lr=0.05, select=select,
                  select_f=1 if select != "none" else -1, flame_lambda=lam, device=DEV)
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
    assert torch.equal(fa.w_global, wg) and slots_form.last_flame == dict_form.last_flame
    assert slots_form.last_admitted == dict_form.last_admitted
    adm = dict_form.last_admitted
    cand = list(range(K))
    if select != "none":
        cand = ops.krum_select(ops.sqdist_statement(ws, 0, nv), list(range(K)), a.select_f, a.select_m)
    assert not {0, 1, 2} & set(adm) and len(adm) >= len(cand) // 2 + 1
    assert (3 in adm) == (3 in cand)                                      # the boosted honest update is clipped, not rejected
    members, sc, S, noise_std = ops.flame_admit(ops.gram_statement([ws[j] for j in cand], g, 0, nv), cand, lam)
    assert [cand[j] for j in members] == adm
    np.testing.assert_allclose(dict_form.last_flame["FLAME/Clip_Bound"], S, rtol=1e-6)
    assert dict_form.last_flame["FLAME/Noise_Std"] == lam * dict_form.last_flame["FLAME/Clip_Bound"]
    opt = ops.ServerOptState(server_opt, n, beta1=a.server_beta1, beta2=a.server_beta2, tau=a.server_tau, device=DEV)
    ref, _ = ops.aggregate_oracle(g, [ws[j] for j in adm], [1.0] * len(adm), "avg", theta, a.server_lr, None, nv,
                                  [float(sc[j]) for j in members], opt, float(len(adm)))
    diff = (wg - ref).double()
    err = float(diff.abs().max())
    print(f"theta={theta} {server_opt} {select} lambda={lam}: admitted {adm}, S {S:.4f}, max |w - noiseless oracle| {err:.2e}")
    if lam == 0:
        assert err < 2e-6
    else:                                                                 # the kernel's Philox noise of std lambda * S, times lr = +-1
        std = float(diff[:nv].std())
        assert abs(std / noise_std - 1.0) < 0.02 and float(diff[nv:].abs().max()) < 2e-6, (std, noise_std)
    assert ops.fallback_calls() == {}
    fa.close()


def test_engine_resnet18_flame_is_reproducible():
    from rlr_b200.engine import FLEngine

    def run():
        ops.reset_fallbacks()
        args = make_args(data="cifar10", model="resnet18", num_agents=4, num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, synthetic=512,
                         synthetic_val=128, log_dir="", seed=3, aggr="flame", robustLR_threshold=2, device=DEV)
        eng = FLEngine(args, verbose=False)
        out = []
        for r in range(1, 3):
            eng.run_round(r)
            out.append((eng.global_params().clone(), dict(eng.aggregator.last_flame), list(eng.aggregator.last_admitted)))
        torch.cuda.synchronize()
        assert ops.fallback_calls() == {}
        eng.close()
        return out

    a, b = run(), run()
    for (wa, fa, aa), (wb, fb, ab) in zip(a, b):
        assert torch.equal(wa, wb) and fa == fb and aa == ab and fa["FLAME/Admitted"] >= 3
    print("FLAME per round:", [f for _, f, _ in a])


# ---- two or more GPUs ------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# fused path: round 0 with the barrier-out, hand-off from round 1 on, so the passes of rounds 1-3 each follow an aggregate that published
# ready words instead of running a barrier-out; the pass reads w_global and has to acquire it first
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
    n, nv, n_part = 1 << 20, (1 << 20) - 4096, 2 * world + 3
    slots = (n_part + world - 1) // world
    gen = torch.Generator().manual_seed(0)
    w0 = torch.randn(n, generator=gen)
    honest, evil = torch.randn(n, generator=gen), torch.randn(n, generator=gen)
    parts = [w0 + 0.01 * (1 + 0.2 * j) * ((evil if j < 2 else honest) + 0.3 * torch.randn(n, generator=gen)) for j in range(n_part)]
    parts[2] = w0 + 100.0 * (parts[2] - w0)
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
            mem = members if rnd >= 2 else None
            cand = mem if mem is not None else list(range(n_part))
            G = fa.pairwise_gram(n_part, mem, copies)
            adm, sc, S, _ = ops_.flame_admit(G, cand, 0.0)
            keep = [cand[j] for j in adm]
            scales = torch.ones(n_part)
            scales[torch.as_tensor(cand)] = sc
            fa.aggregate([1.0] * n_part, "avg", 2, 1.0, 0.0, 0, rnd, scales, members=keep, participants=copies, total_weight=len(keep))
            fa.acquire()
            torch.cuda.synchronize()
            ref, _ = ops_.aggregate_oracle(w_in, [jobs[j] for j in keep], [1.0] * len(keep), "avg", 2, 1.0, None, nv,
                                           [float(scales[j]) for j in keep], None, float(len(keep)))
            res[backend].append(dict(G=G.cpu(), keep=keep, S=S, err=float((fa.w_global.cpu() - ref).abs().max())))
            dist.barrier()
        fa.close()
    single = []
    if rank == 0:                                                    # the same passes in one process, on this GPU
        for rnd in range(N_ROUNDS):
            jobs = [(p + 0.01 * rnd).to(ctx.device) for p in parts]
            cand = members if rnd >= 2 else list(range(n_part))
            single.append(ops_.pairwise_gram([jobs[j] for j in cand], (w0 + 0.01 * rnd).to(ctx.device), nv).cpu())
    torch.save(dict(res, single=single), os.path.join(outdir, f"flame_{provider}_{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("provider", ["auto", "ipc"])
def test_fused_multi_gpu_gram_pass(tmp_path, provider):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_multi_worker, args=(world, _free_port(), str(tmp_path), provider), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"flame_{provider}_{r}.pt") for r in range(world)]
    assert res[0]["handoff"] == [rnd >= HANDOFF_FROM for rnd in range(N_ROUNDS)]
    for rnd in range(N_ROUNDS):
        f0 = res[0]["fused"][rnd]
        single = res[0]["single"][rnd]
        cos_err, diag_err = _errors(f0["G"], single)                # rank-ordered partials: another order of adds than one launch
        assert cos_err <= TOL and diag_err <= TOL, (rnd, cos_err, diag_err)
        for r in range(world):
            fr, nr = res[r]["fused"][rnd], res[r]["nccl"][rnd]
            assert torch.equal(fr["G"], f0["G"]) and fr["keep"] == f0["keep"] and fr["S"] == f0["S"], (r, rnd)   # the same doubles
            assert fr["keep"] == nr["keep"], (r, rnd)
            assert fr["err"] < 2e-6 and nr["err"] < 2e-6, (r, rnd, fr["err"], nr["err"])
            assert torch.equal(nr["G"], single), (r, rnd)            # the gather transport runs the single-process launch


# ---- the engine: flame with the fused hand-off (the default) against --no_fused_handoff -------------------------------------------------
def _engine_run(world, handoff):
    from rlr_b200.engine import FLEngine
    args = make_args(data="cifar10", model="cnn_cifar", synthetic=128 * max(5, 2 * world), synthetic_val=128, num_agents=max(5, 2 * world),
                     num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, log_dir="", seed=7, aggr="flame", robustLR_threshold=2,
                     no_fused_handoff=not handoff, **({} if world > 1 else {"device": DEV}))
    eng = FLEngine(args, verbose=False)
    assert eng.handoff == handoff
    snaps, admitted = [], []
    for r in range(1, 5):
        eng.run_round(r)                    # rounds 2-4: the Gram pass follows a round whose aggregate ran the hand-off
        snaps.append(eng.global_params().clone().cpu())
        admitted.append(list(eng.aggregator.last_admitted))
    torch.cuda.synchronize()
    same = True
    if world > 1:
        allw = eng.ctx.all_gather(eng.global_params().clone())
        same = bool((allw == allw[0:1]).all().item())
    out = {"w": snaps, "admitted": admitted, "same": same, "backend": eng.fused.backend}
    eng.close()
    return out


def _engine_worker(rank, world, port, outdir, handoff, tag):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    torch.save(_engine_run(world, handoff), os.path.join(outdir, f"eng_{tag}_{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("multi", [False, True])
def test_engine_flame_with_fused_handoff_equals_barrier_path(tmp_path, multi):
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
            assert res[t][r]["same"] and res[t][r]["admitted"] == res[t][0]["admitted"], (t, r)
    print("admitted per round:", res["a"][0]["admitted"])
    rel = lambda x, y: float((x.double() - y.double()).norm() / (y.double().norm() + 1e-12))
    for i in range(4):
        noise, diff = rel(res["b"][0]["w"][i], res["a"][0]["w"][i]), rel(res["f"][0]["w"][i], res["a"][0]["w"][i])
        print(f"world {world} round {i + 1}: barrier-vs-barrier {noise:.2e}  handoff-vs-barrier {diff:.2e}")
        assert diff <= 3 * noise + (1e-5 if i == 0 else 1e-4), (i, diff, noise)
