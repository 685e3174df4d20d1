"""SparseFed (``--server_topk``) on the H100: the accumulate / radix-select / apply passes against ``ops.sparsefed_statement`` bit for bit
(the new parameters, the bf16 shadow, the error vector, |M| and tau) at ResNet-18's n_vote and on adversarial vectors; native ResNet-18
runs that are bitwise reproducible and resume bit for bit; and, with >= 2 GPUs, the fused multi-GPU path (barrier-out and hand-off)
against one process."""
import math
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import rlr_b200  # noqa: F401
from rlr_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _bits(x):
    """fp32 bit patterns with every NaN mapped to one: the device's fp32 add returns the canonical NaN 0x7FFFFFFF where numpy keeps the
    operand's payload.  Either way the key sorts above +inf, which is all the statement asks of a NaN."""
    x = np.array(x, dtype=np.float32).reshape(-1)
    x[np.isnan(x)] = np.float32("nan")
    return x.tobytes()


def _device_vs_statement(w, wn, e, nv, k):
    ref = ops.sparsefed_statement(w, wn, e, nv, k)
    dw, dwn, de = (torch.as_tensor(np.asarray(x)).to(DEV) for x in (w, wn, e))
    wb = torch.full(dw.shape, float("nan"), dtype=torch.bfloat16, device=DEV)
    stats = torch.full((3,), float("nan"), dtype=torch.float64, device=DEV)
    ops.sparsefed_step(dw, dwn, de, nv, k, stats, wb)
    got_w, got_e, s = dw.cpu().numpy(), de.cpu().numpy(), stats.cpu().tolist()
    assert _bits(got_w) == _bits(ref[0]), "new parameters"
    assert _bits(got_e[:nv]) == _bits(ref[1]), "error vector"
    assert _bits(wb.cpu().float().numpy()) == _bits(torch.from_numpy(ref[0]).to(torch.bfloat16).float().numpy()), "bf16 shadow"
    assert int(s[0]) == ref[2], "|M|"
    assert _bits(s[1]) == _bits(ref[3]), "tau"
    assert (math.isnan(s[2]) and math.isnan(ref[4])) or math.isclose(s[2], ref[4], rel_tol=1e-12, abs_tol=0.0), "||e||"
    return ref


@pytest.mark.parametrize("p", [0.01, 0.1])
def test_device_pass_equals_the_statement_at_resnet18_size(p):
    from rlr_b200.models import get_layout
    lay = get_layout("resnet18")
    n, nv = lay.n_total, lay.n_vote
    k = math.floor(p * lay.n_params)
    rs = np.random.RandomState(1)
    w = rs.randn(n).astype(np.float32)
    wn = (w + 1e-3 * rs.randn(n)).astype(np.float32)
    e = (1e-3 * rs.randn(nv)).astype(np.float32)                     # a nonzero prior error
    e[rs.randint(0, nv, 1000)] = 0.0
    ref = _device_vs_statement(w, wn, e, nv, k)
    assert k <= ref[2] <= k + 16                                     # ties at tau are all taken


def _adversarial():
    z = lambda m: np.zeros(m, dtype=np.float32)
    base = np.float32(1.0).view(np.uint32)
    low = (base + np.array([0, 1, 2, 3, 0x100, 0x1FF, 0x1FE, 5], dtype=np.uint32)).view(np.float32)
    low = (low * np.array([1, -1, 1, -1, 1, -1, 1, -1], dtype=np.float32)).astype(np.float32)
    ties = np.array([0.5, -0.5, 0.5, 0.25, -0.5, 0.125] + [0.0625] * 10, dtype=np.float32)
    zeros = np.array([0.0, -0.0, 0.0, 1.0, np.nan, -0.0, 0.0, 0.0], dtype=np.float32)
    tail = np.array([3.0, -1.0, 2.5, 7.0], dtype=np.float32)
    cases = []
    for vec, ks in ((low, (1, 3, 8)), (ties, (1, 2, 16)), (zeros, (1, 2, 8))):
        nv = vec.size
        for k in ks:
            cases.append((z(nv + 4), np.concatenate([vec, tail]), z(nv), nv, k))
            prior = (np.arange(nv, dtype=np.float32) - nv / 2) / 16.0                 # a nonzero prior error
            cases.append((np.full(nv + 4, 0.25, dtype=np.float32), np.concatenate([vec + np.float32(0.25), tail]), prior, nv, k))
    return cases


@pytest.mark.parametrize("case", range(len(_adversarial())))
def test_device_pass_equals_the_statement_on_adversarial_vectors(case):
    _device_vs_statement(*_adversarial()[case])


def test_device_rounds_carry_the_error():
    rs = np.random.RandomState(2)
    n, nv, k = 1 << 16, (1 << 16) - 256, 500
    w, e = rs.randn(n).astype(np.float32), np.zeros(nv, dtype=np.float32)
    dw, de = torch.from_numpy(w).to(DEV), torch.from_numpy(e).to(DEV)
    stats = torch.zeros(3, dtype=torch.float64, device=DEV)
    for _ in range(4):
        wn = (w + 1e-2 * rs.randn(n)).astype(np.float32)
        w, e, applied, tau, norm = ops.sparsefed_statement(w, wn, e, nv, k)
        ops.sparsefed_step(dw, torch.from_numpy(wn).to(DEV), de, nv, k, stats)
        assert np.array_equal(dw.cpu().numpy(), w) and np.array_equal(de.cpu().numpy(), e)
        assert stats[0].item() == applied == k and np.float32(stats[1].item()) == np.float32(tau)


# ---- native ResNet-18 runs ---------------------------------------------------------------------------------------------------
def _engine(**kw):
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    base = dict(data="cifar10", model="resnet18", num_agents=3, local_ep=1, bs=64, synthetic=384, synthetic_val=64, log_dir="",
                device=DEV, seed=2, robustLR_threshold=2, server_opt="adam", server_lr=0.01, server_topk=0.01)
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def test_native_resnet18_runs_are_bitwise_reproducible_and_resume(tmp_path):
    runs = []
    for _ in range(2):
        ops.reset_fallbacks()
        eng = _engine(rounds=3)
        assert eng.trainer.name == "native" and eng.topk_k == math.floor(0.01 * eng.layout.n_params)
        hist = eng.fit()
        torch.cuda.synchronize()
        assert not ops.fallback_calls()
        runs.append((eng.global_params().clone(), eng.fused.sparse_e.clone(), [{k: v for k, v in h.items() if k.startswith("sparse")}
                                                                               for h in hist]))
        eng.close()
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]) and runs[0][2] == runs[1][2]
    assert all(h["sparse_applied"] > 0 and h["sparse_error_norm"] > 0 for h in runs[0][2])
    ck = str(tmp_path / "ck.pt")
    first = _engine(rounds=2, checkpoint=ck)
    first.fit()
    first.close()
    second = _engine(rounds=3, resume=ck)
    hist = second.fit()
    assert torch.equal(second.global_params(), runs[0][0]) and torch.equal(second.fused.sparse_e, runs[0][1])
    assert {k: v for k, v in hist[-1].items() if k.startswith("sparse")} == runs[0][2][-1]
    second.close()


# ---- fused multi-GPU path --------------------------------------------------------------------------------------------------
def _multi_worker(rank, world, port, outdir, handoff):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200 import ops as o
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed()
    n, nv, n_part, k = 1 << 20, (1 << 20) - 4096, 2 * world + 1, 5000
    kind = dict(kind="adam", beta1=0.9, beta2=0.99, tau=1e-3)
    fa = FusedAggregator(ctx, n, nv, (n_part + world - 1) // world, "fused", server_opt=kind, topk_k=k)
    if handoff:
        fa.enable_handoff()
    # one process: the same kernels on every participant, on this rank's GPU
    ref_w, ref_e = torch.empty(n, device=ctx.device), torch.zeros(nv, device=ctx.device)
    ref_b, ref_s = torch.empty(n, dtype=torch.bfloat16, device=ctx.device), torch.zeros(3, dtype=torch.float64, device=ctx.device)
    ref_opt = o.ServerOptState(n=n, device=ctx.device, **kind)
    gen = torch.Generator().manual_seed(0)
    w0 = torch.randn(n, generator=gen)
    fa.w_global.copy_(w0.to(ctx.device)); fa.w_bf16.copy_(fa.w_global.to(torch.bfloat16)); ref_w.copy_(w0.to(ctx.device))
    ref_b.copy_(ref_w.to(torch.bfloat16))
    torch.cuda.synchronize(); dist.barrier()
    same = True
    for rnd in range(1, 4):
        fa.acquire()
        parts = [ref_w + (0.05 * torch.randn(n, generator=gen)).to(ctx.device) for _ in range(n_part)]
        for j in range(n_part):
            r, s = fa.slot_owner(j)
            if r == ctx.rank:
                fa.slots[s].copy_(fa.w_global + (parts[j] - ref_w))
        weights = [float(50 + 7 * j) for j in range(n_part)]
        fa.aggregate(weights, "avg", 3, 1.0, 0.0, 0, rnd)
        scratch = o.fused_aggregate(ref_w, parts, weights, "avg", 3, 1.0, n_vote=nv, out=torch.empty_like(ref_w), opt=ref_opt)
        o.sparsefed_step(ref_w, scratch, ref_e, nv, k, ref_s, ref_b)
        fa.acquire()
        torch.cuda.synchronize()
        same &= bool(torch.equal(fa.w_global, ref_w) and torch.equal(fa.sparse_e, ref_e) and torch.equal(fa.w_bf16, ref_b)
                     and torch.equal(fa.sparse_stats, ref_s))
    torch.save({"same": same, "w": fa.w_global.cpu(), "e": fa.sparse_e.cpu(), "stats": fa.sparse_stats.cpu()},
               os.path.join(outdir, f"sf{int(handoff)}_{rank}.pt"))
    fa.close()
    dist.barrier(); dist.destroy_process_group()


def test_fused_multi_gpu_path_equals_one_process(tmp_path):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    for handoff in (False, True):
        mp.spawn(_multi_worker, args=(world, _free_port(), str(tmp_path), handoff), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"sf{h}_{r}.pt") for h in (0, 1) for r in range(world)]
    for x in res:
        assert x["same"]
        assert torch.equal(x["w"], res[0]["w"]) and torch.equal(x["e"], res[0]["e"]) and torch.equal(x["stats"], res[0]["stats"])
