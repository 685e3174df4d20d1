"""DnC selection on the H100: ``dnc_gather_kernel`` bit for bit against ``ops.dnc_gather_statement`` and the gather + Gram launches
against the fp64 statement for K from 2 to 65 and samples below, at and above n_vote, run-to-run bitwise equality, the fall-through past
1024 participants, engine runs (reproducible, the no-removal case equal to ``--select none``, both step forms admitting the same set,
the fused hand-off against the barrier path) and -- with two or more GPUs -- the fused multi-GPU pass against the gather transport."""
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
# The Gram kernel adds fp32 products over <= 256 coordinates and folds them into fp64 (the FoolsGold / FLAME Gram pass): relative error
# a few 1e-7 of the larger entries.
RTOL, ATOL_REL = 1e-5, 1e-6


def _participants(K, n, seed, scale=0.01):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randn(n, generator=gen, device=DEV)
    ws = [g + torch.randn(n, generator=gen, device=DEV) * (scale * (1 + k % 5)) for k in range(K)]
    return g, ws


def _close(G, ref):
    err = (G - ref).abs()
    bound = RTOL * ref.abs() + ATOL_REL * float(ref.diagonal(dim1=-2, dim2=-1).abs().max())
    return bool((err <= bound).all()), float(err.max())


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("case", ["below", "at", "above"])
@pytest.mark.parametrize("K", [2, 10, 64, 65])
def test_gather_and_gram_match_the_statement(K, case, scaled):
    ops.reset_fallbacks()
    n, nv = 200_004, 199_999                                            # n_vote not a multiple of 4
    b = {"below": 10_001, "at": nv, "above": nv + 5}[case]              # nor b
    g, ws = _participants(K, n, K + 3 * scaled)
    scales = (0.25 + torch.rand(K, device=DEV)).float() if scaled else None
    T = 2
    samples = np.stack([ops.dnc_sample(1, 2, t, b, nv) for t in range(T)])
    G = ops.dnc_grams(ws, g, samples, nv, scales)
    # the gather alone, bit for bit the statement
    S = samples.shape[1]
    pad = (S + 3) // 4 * 4
    y = torch.empty((T, K, pad), dtype=torch.float32, device=DEV)
    tab = ops.PtrTable([w.data_ptr() for w in ws], DEV)
    rng = torch.tensor([[0, S]] * T, dtype=torch.int32, device=DEV)
    ops.ext().dnc_gather(tab.tensor, g.data_ptr(), scales, torch.from_numpy(samples.astype(np.int32)).to(DEV), rng, y, None, None, 0, 1, 0)
    torch.cuda.synchronize()
    for t in range(T):
        assert torch.equal(y[t, :, :S], ops.dnc_gather_statement(ws, g, samples[t], scales)), t
        assert not y[t, :, S:].any()
    ref = ops.dnc_gram_statement(ws, g, samples, scales)
    ok, err = _close(G, ref)
    print(f"K={K} b={b} scaled={scaled}: max abs err {err:.2e}")
    assert ok, err
    assert ops.fallback_calls() == {}


@pytest.mark.parametrize("K", [8, 64])
def test_two_launches_are_bitwise_equal(K):
    n, nv = 1 << 20, (1 << 20) - 4096
    g, ws = _participants(K, n, 5)
    samples = np.stack([ops.dnc_sample(0, 1, t, 10_000, nv) for t in range(3)])
    s = torch.rand(K, device=DEV) + 0.5
    a, b = ops.dnc_grams(ws, g, samples, nv), ops.dnc_grams(ws, g, samples, nv)
    c, d = ops.dnc_grams(ws, g, samples, nv, s), ops.dnc_grams(ws, g, samples, nv, s)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(c, d)


def test_more_than_1024_participants_fall_through_to_the_statement():
    ops.reset_fallbacks()
    g, ws = _participants(1025, 256, 9)
    samples = ops.dnc_sample(0, 1, 0, 100, 250)[None]
    G = ops.dnc_grams(ws, g, samples, 250)
    assert torch.equal(G, ops.dnc_gram_statement(ws, g, samples))
    assert list(ops.fallback_calls()) == ["dnc_grams"]
    ops.reset_fallbacks()


# ---- the engine on one GPU --------------------------------------------------------------------------------------------------------
def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="cifar10", model="cnn_cifar", synthetic=128 * 6, synthetic_val=128, num_agents=6, num_corrupt=1, poison_frac=0.5,
                local_ep=1, bs=64, log_dir="", seed=5, rounds=3, snap=100, device=DEV)
    base.update(kw)
    eng = FLEngine(make_args(**base), verbose=False)
    admitted = []
    for r in range(1, 4):
        eng.run_round(r)
        admitted.append(list(eng.aggregator.last_admitted) if eng.aggregator.last_admitted is not None else None)
    torch.cuda.synchronize()
    out = dict(w=eng.global_params().clone(), admitted=admitted, trainer=eng.trainer.name)
    eng.close()
    return out


def test_engine_run_is_reproducible_and_no_removal_equals_no_selection():
    ops.reset_fallbacks()
    a, b = _engine(select="dnc", dnc_dim=5000), _engine(select="dnc", dnc_dim=5000)
    assert a["trainer"] == "native"
    print("DnC admitted per round:", a["admitted"])
    assert torch.equal(a["w"], b["w"]) and a["admitted"] == b["admitted"]
    assert all(len(x) == 5 for x in a["admitted"])
    none, zero = _engine(), _engine(select="dnc", dnc_frac=0.0)
    assert torch.equal(none["w"], zero["w"])
    assert all(sorted(x) == list(range(6)) for x in zero["admitted"])
    assert ops.fallback_calls() == {}


def test_resnet18_round_admits_the_same_set_in_both_step_forms():
    from rlr_b200.engine import FLEngine
    ops.reset_fallbacks()
    args = make_args(data="cifar10", model="resnet18", num_agents=6, num_corrupt=2, poison_frac=0.5, local_ep=1, bs=64, synthetic=768,
                     synthetic_val=128, log_dir="", seed=3, select="dnc", dnc_iters=2, robustLR_threshold=2, device=DEV)
    eng = FLEngine(args, verbose=False)
    nv = eng.layout.n_vote
    dict_form = Aggregation(eng.agent_data_sizes, eng.layout.n_params, None, args, layout=eng.layout)
    orig = eng.aggregator.aggregate_slots
    seen = []

    def aggregate_slots(participants, rnd):
        eng.fused.acquire()
        wg = eng.fused.w_global.clone()
        ws = {a: eng.fused.slots[j].clone() for j, a in enumerate(participants)}
        orig(participants, rnd)
        dict_form.aggregate_updates(wg, ws, rnd, n_vote=nv)
        torch.cuda.synchronize()
        seen.append((eng.aggregator.last_admitted, dict_form.last_admitted, torch.equal(eng.fused.w_global, wg)))
    eng.aggregator.aggregate_slots = aggregate_slots
    for r in range(1, 3):
        eng.run_round(r)
    torch.cuda.synchronize()
    print("ResNet-18 DnC admitted (slots form, dict form, same step):", seen)
    assert seen and all(s == d and len(s) >= 2 and same for s, d, same in seen), seen
    assert ops.fallback_calls() == {}
    eng.close()


# ---- two or more GPUs ------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


N_ROUNDS, HANDOFF_FROM, SCALED_ROUNDS = 4, 1, (2,)


def _multi_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200 import ops as ops_
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed()
    n, nv, n_part = 1 << 20, (1 << 20) - 4093, 2 * world + 3
    slots = (n_part + world - 1) // world
    gen = torch.Generator().manual_seed(0)
    w0 = torch.randn(n, generator=gen)
    d = torch.randn(n, generator=gen)
    parts = [w0 + 0.02 * torch.randn(n, generator=gen) for j in range(n_part)]
    for j in (0, 1):
        parts[j] = parts[j] + 0.04 * d                                     # a shared direction: removed
    res = {"fused": [], "nccl": []}
    for backend in ("fused", "nccl"):
        fa = FusedAggregator(ctx, n, nv, slots, backend, transport="gather")
        for rnd in range(N_ROUNDS):
            if backend == "fused" and rnd == HANDOFF_FROM:
                fa.enable_handoff()
            w_in = w0 + 0.01 * rnd
            fa.w_global.copy_(w_in.to(ctx.device))
            for j in range(n_part):
                r, s = fa.slot_owner(j)
                if r == ctx.rank:
                    fa.slots[s].copy_((parts[j] + 0.01 * rnd).to(ctx.device))
            torch.cuda.synchronize(); dist.barrier()
            scales = torch.linspace(0.6, 1.0, n_part, device=ctx.device) if rnd in SCALED_ROUNDS else None
            samples = np.stack([ops_.dnc_sample(0, rnd, t, 50_001 if rnd < 3 else nv, nv) for t in range(2)])
            copies = fa.gather_participants(n_part) if fa.gathers(n_part) else None
            G = fa.dnc_grams(n_part, samples, scales, None, copies)
            keep = ops_.dnc_select(G, list(range(n_part)), 2, 1.0)
            fa.aggregate([float(50 + 7 * j) for j in range(n_part)], "avg", 2, 1.0, 0.0, 0, rnd, scales, members=keep, participants=copies)
            fa.acquire()
            torch.cuda.synchronize()
            res[backend].append(dict(G=G.cpu(), keep=keep))
            dist.barrier()
        fa.close()
    torch.save(res, os.path.join(outdir, f"dnc_{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


def test_fused_multi_gpu_grams_and_selection(tmp_path):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_multi_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"dnc_{r}.pt") for r in range(world)]
    for rnd in range(N_ROUNDS):
        f0, g0 = res[0]["fused"][rnd], res[0]["nccl"][rnd]
        for r in range(world):
            assert torch.equal(res[r]["fused"][rnd]["G"], f0["G"]) and res[r]["fused"][rnd]["keep"] == f0["keep"], (r, rnd)
        ok, err = _close(f0["G"], g0["G"])
        assert ok, (rnd, err)
        assert f0["keep"] == g0["keep"] and 0 not in f0["keep"] and 1 not in f0["keep"], (rnd, f0["keep"])


# ---- the engine: --select dnc with the fused hand-off (the default) against --no_fused_handoff -------------------------------------------
def _engine_select_run(world, handoff):
    from rlr_b200.engine import FLEngine
    args = make_args(data="cifar10", model="cnn_cifar", synthetic=128 * max(5, 2 * world), synthetic_val=128, num_agents=max(5, 2 * world),
                     num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, log_dir="", seed=7, select="dnc", dnc_dim=20_000,
                     no_fused_handoff=not handoff, **({} if world > 1 else {"device": DEV}))
    eng = FLEngine(args, verbose=False)
    assert eng.handoff == handoff
    snaps, admitted = [], []
    for r in range(1, 5):
        eng.run_round(r)
        snaps.append(eng.global_params().clone().cpu())
        admitted.append(list(eng.aggregator.last_admitted))
    torch.cuda.synchronize()
    same = True
    if world > 1:
        allw = eng.ctx.all_gather(eng.global_params().clone())
        same = bool((allw == allw[0:1]).all().item())
    out = {"w": snaps, "admitted": admitted, "same": same, "K": eng.args.num_agents, "backend": eng.fused.backend}
    eng.close()
    return out


def _engine_select_worker(rank, world, port, outdir, handoff, tag):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    torch.save(_engine_select_run(world, handoff), os.path.join(outdir, f"eng_{tag}_{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("multi", [False, True])
def test_engine_dnc_with_fused_handoff_equals_barrier_path(tmp_path, multi):
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
            assert all(len(a) == res[t][r]["K"] - 1 for a in res[t][r]["admitted"])
    rel = lambda x, y: float((x.double() - y.double()).norm() / (y.double().norm() + 1e-12))
    for i in range(4):
        noise, diff = rel(res["b"][0]["w"][i], res["a"][0]["w"][i]), rel(res["f"][0]["w"][i], res["a"][0]["w"][i])
        print(f"world {world} round {i + 1}: barrier-vs-barrier {noise:.2e}  handoff-vs-barrier {diff:.2e}")
        assert diff <= 3 * noise + (1e-5 if i == 0 else 1e-4), (i, diff, noise)
