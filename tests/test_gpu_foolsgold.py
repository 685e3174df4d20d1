"""FoolsGold on the H100: the history accumulate (``history_accumulate_kernel``, ops/csrc/foolsgold.cu) bitwise against the fp32 statement at
the ResNet-18 size on a coordinate range that does not start at 0, also through offset row pointers of a sliced table; the history Gram
(``pairwise_sqdist_kernel<true, true>``, ops/csrc/select.cu) against the fp64 statement and bitwise from launch to launch; a one-GPU engine
run against the in-process dict form; and -- with two or more GPUs -- the fused sharded history against the gather path, the same decisions on
every rank, and a checkpoint taken at world size 2 resumed at 1."""
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
# the Gram pass is FLAME's kernel on other rows: the same bound on the cosine and on the relative error of the diagonal (tests/test_gpu_flame.py)
TOL = 1e-6


def _nv():
    from rlr_b200.models import get_layout
    return get_layout("resnet18").n_vote


def _errors(G, ref):
    G, ref = G.double().cpu(), ref.double().cpu()
    q = torch.diagonal(ref)
    cos_err = float(((G - ref).abs() / torch.sqrt(torch.outer(q, q))).max())
    diag_err = float(((torch.diagonal(G) - q).abs() / q).max())
    return cos_err, diag_err


@pytest.mark.parametrize("K", [1, 8, 40, 64, 65, 200])
def test_accumulate_kernel_equals_the_statement_at_resnet18_size(K):
    nv = _nv()
    lo, hi = 4100, nv - 8                                           # a range that does not start at 0 (and stops short of n_vote)
    gen = torch.Generator(device=DEV).manual_seed(K)
    g = torch.randn(nv, generator=gen, device=DEV)
    pool = [g + 0.01 * torch.randn(nv, generator=gen, device=DEV) for _ in range(min(K, 8))]
    ws = [pool[k % len(pool)] for k in range(K)]                    # slots may repeat; history rows may not
    H = torch.randn((K, nv), generator=gen, device=DEV)
    before = H.clone()
    want = ops.history_statement([before[k] for k in range(K)], ws, g, lo, hi)
    ops.history_accumulate([H[k] for k in range(K)], ws, g, lo, hi)
    torch.cuda.synchronize()
    for k in range(K):
        assert torch.equal(H[k, lo:hi], want[k]), k
    assert torch.equal(H[:, :lo], before[:, :lo]) and torch.equal(H[:, hi:], before[:, hi:])   # nothing outside [lo, hi)
    if K <= 65:                                                     # the sharded layout: rows hold [lo, hi) only, pointers offset by lo
        S = before[:, lo:hi].contiguous()
        tab = ops.PtrTable([w.data_ptr() for w in ws], g.device)
        rows = ops.PtrTable([S.data_ptr() + 4 * ((hi - lo) * k - lo) for k in range(K)], g.device)
        ops.ext().history_accumulate(tab.tensor, rows.tensor, g.data_ptr(), lo, hi, None, None, 0, 1, 0)
        torch.cuda.synchronize()
        assert torch.equal(S, H[:, lo:hi])


@pytest.mark.parametrize("K", [1, 8, 65, 200])
def test_history_gram_matches_the_fp64_statement_and_repeats_bitwise(K):
    ops.reset_fallbacks()
    n = 1 << 20 if K <= 65 else 1 << 18
    gen = torch.Generator(device=DEV).manual_seed(K + 1)
    common = torch.randn(n, generator=gen, device=DEV)
    H = torch.stack([(0.5 if k % 3 == 0 else 0.0) * common + (1 + k % 5) * torch.randn(n, generator=gen, device=DEV) for k in range(K)])
    nv = n - 1024
    H[:, nv:] += 1e3                                                # coordinates past n_vote do not count
    rows = [H[k] for k in range(K)]
    G = ops.history_gram(rows, nv)
    G2 = ops.history_gram(rows, nv)
    torch.cuda.synchronize()
    assert G.shape == (K, K) and G.dtype == torch.float64 and torch.equal(G, G.T)
    assert torch.equal(G, G2)
    cos_err, diag_err = _errors(G, ops.history_gram_statement(rows, 0, nv))
    print(f"K={K}: max |dG| / sqrt(G_ii G_jj) {cos_err:.2e}, max rel err of the diagonal {diag_err:.2e}")
    assert cos_err <= TOL and diag_err <= TOL, (cos_err, diag_err)
    assert ops.fallback_calls() == {}


@pytest.mark.parametrize("K", [8, 65])
def test_sliced_rows_through_offset_pointers(K):
    """The fused path's addressing on one GPU: a table that holds only the columns [lo, hi) of each row, its pointers offset by lo, read by
    the Gram pass over [lo, hi); and an empty slice (a rank whose coordinates lie past n_vote), which touches nothing and sums to 0."""
    n = 1 << 20
    lo, hi = 4096 * 3 + 4, n - 4096
    gen = torch.Generator(device=DEV).manual_seed(K + 7)
    full = torch.randn((K, n), generator=gen, device=DEV)
    S = full[:, lo:hi].contiguous()
    rows = ops.PtrTable([S.data_ptr() + 4 * ((hi - lo) * k - lo) for k in range(K)], full.device)
    G = torch.empty(K, K, dtype=torch.float64, device=DEV)
    ops.ext().history_gram(rows.tensor, lo, hi, G)
    cos_err, diag_err = _errors(G, ops.history_gram_statement([full[k] for k in range(K)], lo, hi))
    assert cos_err <= TOL and diag_err <= TOL, (cos_err, diag_err)
    E = S[:, :0]                                                     # width 0
    erows = ops.PtrTable([E.data_ptr() - 4 * hi for _ in range(K)], full.device)
    g = torch.randn(n, generator=gen, device=DEV)
    tab = ops.PtrTable([full[k].data_ptr() for k in range(K)], full.device)
    before = S.clone()
    ops.ext().history_accumulate(tab.tensor, erows.tensor, g.data_ptr(), hi, hi, None, None, 0, 1, 0)
    ops.ext().history_gram(erows.tensor, hi, hi, G)
    torch.cuda.synchronize()
    assert torch.equal(S, before) and not G.any()


def test_one_gpu_engine_rounds_equal_the_dict_form():
    """The engine's rounds (slots form, half the agents per round) against the dict form fed the same slots: history and w_global bitwise."""
    from rlr_b200.engine import FLEngine
    ops.reset_fallbacks()
    args = make_args(data="cifar10", model="resnet18", num_agents=6, agent_frac=0.5, num_corrupt=2, poison_frac=0.5, local_ep=1, bs=64,
                     synthetic=768, synthetic_val=128, log_dir="", seed=3, aggr="foolsgold", robustLR_threshold=2, device=DEV)
    eng = FLEngine(args, verbose=False)
    nv = eng.layout.n_vote
    dict_form = Aggregation(eng.agent_data_sizes, eng.layout.n_params, None, args, layout=eng.layout)
    orig = eng.aggregator.aggregate_slots
    same = []

    def aggregate_slots(participants, rnd):
        eng.fused.acquire()
        wg = eng.fused.w_global.clone()
        ws = {a: eng.fused.slots[j].clone() for j, a in enumerate(participants)}
        orig(participants, rnd)
        dict_form.aggregate_updates(wg, ws, rnd, n_vote=nv)
        torch.cuda.synchronize()
        same.append((torch.equal(eng.fused.w_global, wg), torch.equal(eng.fused.history, dict_form.history),
                     eng.aggregator.last_foolsgold == dict_form.last_foolsgold, eng.aggregator.last_admitted == dict_form.last_admitted))
    eng.aggregator.aggregate_slots = aggregate_slots
    for r in range(1, 4):
        eng.run_round(r)
    torch.cuda.synchronize()
    print("FoolsGold per round:", eng.aggregator.last_foolsgold, "history rows touched:", int((eng.fused.history != 0).any(1).sum()))
    assert same and all(all(s) for s in same), same
    assert ops.fallback_calls() == {}
    eng.close()


# ---- two or more GPUs ------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _multi_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200 import ops as ops_
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed()
    n, nv, n_part, agents = 1 << 20, (1 << 20) - 4096, 2 * world + 3, 4 * world + 4
    slots = (n_part + world - 1) // world
    gen = torch.Generator().manual_seed(0)
    w0 = torch.randn(n, generator=gen)
    evil = torch.randn(n, generator=gen)
    res = {}
    for backend in ("fused", "nccl"):
        fa = FusedAggregator(ctx, n, nv, slots, backend, transport="gather", n_part=n_part, history_agents=agents)
        out = []
        for rnd in range(4):
            if backend == "fused" and rnd == 1:
                fa.enable_handoff()
            ids = [int(a) for a in torch.randperm(agents, generator=torch.Generator().manual_seed(rnd))[:n_part]]
            w_in = w0 + 0.01 * rnd
            fa.w_global.copy_(w_in.to(ctx.device))
            for j, a in enumerate(ids):
                r, s = fa.slot_owner(j)
                if r == ctx.rank:
                    u = evil if a < 3 else torch.randn(n, generator=torch.Generator().manual_seed(1000 * rnd + a))
                    fa.slots[s].copy_((w_in + 0.01 * u).to(ctx.device))
            torch.cuda.synchronize(); dist.barrier()
            copies = fa.gather_participants(n_part) if fa.gathers(n_part) else None
            members = [j for j in range(n_part) if j != 1] if rnd >= 2 else None
            G = fa.foolsgold_gram(n_part, ids, members, copies)
            alpha = ops_.foolsgold_weights(G)
            out.append(dict(G=G.cpu(), alpha=alpha.tolist()))
        out.append(dict(history=fa.foolsgold_history()))
        res[backend] = out
        fa.close()
    torch.save(res, os.path.join(outdir, f"fg_{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


def test_fused_sharded_history_equals_the_gather_path(tmp_path):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_multi_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"fg_{r}.pt") for r in range(world)]
    f0, g0 = res[0]["fused"], res[0]["nccl"]
    assert torch.equal(f0[-1]["history"], g0[-1]["history"])       # exact fp32: the same bits whichever rank holds a column
    for rnd in range(4):
        cos_err, diag_err = _errors(f0[rnd]["G"], g0[rnd]["G"])     # rank-ordered partials: another order of adds than one launch
        assert cos_err <= TOL and diag_err <= TOL, (rnd, cos_err, diag_err)
        for r in range(world):
            assert torch.equal(res[r]["fused"][rnd]["G"], f0[rnd]["G"]) and res[r]["fused"][rnd]["alpha"] == f0[rnd]["alpha"], (r, rnd)
            assert torch.equal(res[r]["nccl"][rnd]["G"], g0[rnd]["G"]) and res[r]["nccl"][rnd]["alpha"] == g0[rnd]["alpha"], (r, rnd)
    for r in range(1, world):                                       # the host table is built on the main rank only
        assert res[r]["fused"][-1]["history"] is None and res[r]["nccl"][-1]["history"] is None


def _engine_args(world, **kw):
    return make_args(data="cifar10", model="cnn_cifar", synthetic=128 * 8, synthetic_val=128, num_agents=8, agent_frac=0.5, num_corrupt=2,
                     poison_frac=0.5, local_ep=1, bs=64, log_dir="", seed=7, aggr="foolsgold", **({} if world > 1 else {"device": DEV}),
                     **kw)


def _ckpt_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200.engine import FLEngine
    eng = FLEngine(_engine_args(world, rounds=2, checkpoint=os.path.join(outdir, "ck.pt")), verbose=False)
    eng.fit()
    hist = eng.fused.foolsgold_history()
    admitted = list(eng.aggregator.last_admitted)
    allw = eng.ctx.all_gather(eng.global_params().clone())
    torch.save(dict(history=hist, admitted=admitted, same=bool((allw == allw[0:1]).all().item()), backend=eng.fused.backend,
                    sharded=eng.fused.sharded), os.path.join(outdir, f"ck_{rank}.pt"))
    eng.close()
    dist.barrier(); dist.destroy_process_group()


def test_checkpoint_at_world_size_two_resumes_at_one(tmp_path):
    from rlr_b200.engine import FLEngine
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_ckpt_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    res = [torch.load(tmp_path / f"ck_{r}.pt") for r in range(2)]
    assert res[0]["backend"] == "fused" and res[0]["sharded"] and res[0]["same"] and res[1]["admitted"] == res[0]["admitted"]
    ck = torch.load(tmp_path / "ck.pt", weights_only=False)
    assert torch.equal(ck["extra"]["foolsgold_history"], res[0]["history"]) and res[1]["history"] is None
    eng = FLEngine(_engine_args(1, rounds=3, resume=str(tmp_path / "ck.pt")), verbose=False)
    assert eng.start_round == 3 and torch.equal(eng.fused.foolsgold_history(), res[0]["history"])
    eng.fit()
    assert eng.aggregator.last_foolsgold is not None and torch.isfinite(eng.global_params()).all()
    eng.close()
