"""FLDetector on the H100: the ring pass (``fld_ring_kernel``), the Hessian-vector product (``fld_hvp_kernel``) and the table writes of the
prediction pass (``fld_predict_kernel``) bitwise against the statements; the squared distances within the fp64 error bound of the statement
and bitwise from launch to launch, over grid sweeps; a native-trainer engine run with detection reproducible bit for bit and equal under
``--no_graphs``; and -- with two or more GPUs -- the fused sharded state against a single process."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.options import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("nv", [4, 4 * 1001, (1 << 20) + 12])
def test_ring_and_hvp_are_bitwise_the_statements(nv):
    gen = torch.Generator(device=DEV).manual_seed(nv)
    g = torch.randn(nv, generator=gen, device=DEV)
    prev = g + 1e-3 * torch.randn(nv, generator=gen, device=DEV)
    p0 = prev.clone()
    s = torch.full((nv,), 7.0, device=DEV)
    ops.fld_ring(g, prev, s, 0, nv)
    assert torch.equal(s, ops.fld_ring_statement(g, p0, 0, nv)) and torch.equal(prev, g)
    prev.copy_(p0)
    ops.fld_ring(g, prev, None, 0, nv)                                   # w_prev only
    assert torch.equal(prev, g)
    for N in (1, 4, 10):
        ring = [1e-2 * torch.randn(nv, generator=gen, device=DEV) for _ in range(N + 1)]
        coef = np.random.default_rng(N).standard_normal(N + 1) * 10.0 ** np.random.default_rng(N).uniform(-3, 3, N + 1)
        lo = 4 if nv > 8 else 0
        hv = ops.fld_hvp(ring, coef, lo, nv)
        assert torch.equal(hv, ops.fld_hvp_statement(ring, coef, lo, nv)), N


@pytest.mark.parametrize("nv", [4, 4 * 1001, (1 << 20) + 12])
@pytest.mark.parametrize("K", [1, 7, 8, 9, 64, 200])
def test_predict_pass_against_the_statement(nv, K):
    ops.reset_fallbacks()
    gen = torch.Generator(device=DEV).manual_seed(K * 7 + nv)
    g = torch.randn(nv, generator=gen, device=DEV)
    pool = [g + 1e-2 * torch.randn(nv, generator=gen, device=DEV) for _ in range(min(K, 9))]
    ws = [pool[k % len(pool)] for k in range(K)]
    T0 = 1e-2 * torch.randn((K, nv), generator=gen, device=DEV)
    hv = 1e-3 * torch.randn(nv, generator=gen, device=DEV)
    us, want = ops.fld_predict_statement([T0[k] for k in range(K)], ws, g, hv, 0, nv)
    T = T0.clone()
    d2 = ops.fld_predict([T[k] for k in range(K)], ws, g, hv, 0, nv)
    T2 = T0.clone()
    d2b = ops.fld_predict([T2[k] for k in range(K)], ws, g, hv, 0, nv)
    torch.cuda.synchronize()
    assert torch.equal(d2, d2b)                                          # fixed-order sums: bitwise from launch to launch
    assert all(torch.equal(T[k], us[k]) for k in range(K)) and torch.equal(T, T2)
    err = float(((d2 - want).abs() / want.abs().clamp_min(1e-300)).max())
    assert err <= nv * 2.0 ** -52, err                                   # fp64 sums of nv exact squares: at most nv roundings
    T3 = T0.clone()
    assert ops.fld_predict([T3[k] for k in range(K)], ws, g, None, 0, nv) is None                 # record only
    assert torch.equal(T3, T)
    assert ops.fallback_calls() == {}


def _args(world=1, **kw):
    base = dict(data="cifar10", model="cnn_cifar", synthetic=128 * 6, synthetic_val=128, num_agents=6, agent_frac=1.0, num_corrupt=2,
                poison_frac=0.5, attack_boost=10.0, local_ep=1, bs=64, log_dir="", seed=3, detect="fldetector", fld_window=2, rounds=8,
                snap=100, **({} if world > 1 else {"device": DEV}))
    base.update(kw)
    return make_args(**base)


def _run(**kw):
    from rlr_b200.engine import FLEngine
    eng = FLEngine(_args(**kw), verbose=False)
    hist = eng.fit()
    out = dict(w=eng.global_params().clone(), flagged=list(eng.aggregator.fld_flagged), det=eng.aggregator.fld_detect_round,
               fld=[{k: v for k, v in r.items() if k.startswith("fld")} for r in hist], table=eng.fused.fld_table.clone(),
               trainer=eng.trainer.name)
    eng.close()
    return out


def test_native_run_is_reproducible_and_equal_without_graphs():
    ops.reset_fallbacks()
    a, b, c = _run(), _run(), _run(no_graphs=True)
    assert a["trainer"] == "native"
    print("FLDetector native run: flagged", a["flagged"], "in round", a["det"])
    for o in (b, c):
        assert torch.equal(o["w"], a["w"]) and torch.equal(o["table"], a["table"])
        assert o["fld"] == a["fld"] and o["flagged"] == a["flagged"]
    assert a["flagged"] == [0, 1]
    assert ops.fallback_calls() == {}


# ---- two or more GPUs ------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _multi_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200.engine import FLEngine
    eng = FLEngine(_args(world), verbose=False)
    hist = eng.fit()
    tables = eng.fused.fld_tables()
    torch.save(dict(w=eng.global_params().clone().cpu(), flagged=eng.aggregator.fld_flagged, sharded=eng.fused.sharded,
                    fld=[{k: v for k, v in r.items() if k.startswith("fld")} for r in hist], tables=tables),
               os.path.join(outdir, f"m{rank}.pt"))
    eng.close()
    dist.barrier(); dist.destroy_process_group()


def test_fused_multi_gpu_matches_one_process(tmp_path):
    world = min(torch.cuda.device_count(), 2)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_multi_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"m{r}.pt", weights_only=False) for r in range(world)]
    one = _run()
    assert res[0]["sharded"]
    for r in res:
        assert r["flagged"] == one["flagged"] and torch.equal(r["w"], res[0]["w"])
    torch.testing.assert_close(res[0]["w"], one["w"].cpu(), rtol=1e-5, atol=1e-6)
    assert res[0]["tables"] is not None and res[1]["tables"] is None
    # rank-ordered partials add in another order than one launch: scores may differ in the last bits, the decision may not
    assert [set(x) - {"fld_avg_honest_score", "fld_avg_corrupt_score"} for x in res[0]["fld"]] == \
           [set(x) - {"fld_avg_honest_score", "fld_avg_corrupt_score"} for x in one["fld"]]
