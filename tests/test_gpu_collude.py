"""Colluding attackers on the H100: the crafted slots of ``collude_kernel`` bit for bit against ``ops.collude_statement`` at the ResNet-18
``n_vote`` and at a size that takes several grid sweeps with a remainder, for K from 2 to 257 (H = 1 included); the reduced a_k, e_k, q
and deviation within an fp64 bound of the statement and bitwise repeatable; native engine runs with each mode (graph replay against
``--no_graphs``, two runs bit-identical, no library fall-through); one round under every selection, defense and detector; and -- with
two or more GPUs -- the fused multi-GPU path against one GPU, with and without server clipping."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.models import get_layout
from rlr_b200.options import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# The kernel folds a_k, e_k, q and the deviation in fp64 in a fixed order different from the statement's: relative error ~1e-13 of the
# magnitudes involved (for e_k, of sqrt(a_k q), its Cauchy-Schwarz bound).
RTOL = 1e-9


def _sizes(which):
    if which == "resnet18":
        return get_layout("resnet18").n_vote
    return 3 * 132 * 2 * 1024 + 4 * 37                                   # several sweeps of a two-wave grid plus a remainder


def _participants(K, n, seed, scale=0.01):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randn(n + 8, generator=gen, device=DEV)
    ws = [g + torch.randn(n + 8, generator=gen, device=DEV) * (scale * (1 + k % 5)) for k in range(K)]
    return g, ws


def _craft(honest, corrupt, g, nv, mode, direction):
    """The engine's single-process sequence on fresh output buffers: distances, statistics, gamma*, write pass."""
    H = len(honest)
    outs = [c.clone() for c in corrupt]
    st = D = None
    gamma, z = 0.0, None
    if mode == "alie":
        z = ops.collude_z(H, len(corrupt))
    else:
        D = ops.pairwise_sqdist(honest, nv) if H > 1 else torch.zeros((1, 1), dtype=torch.float64)
        st = ops.collude_stats(honest, corrupt, g, nv, direction)
        gamma = ops.collude_gamma(mode, st[:H], st[H:2 * H], st[2 * H], D)
    dev2 = ops.collude_write(honest, corrupt, outs, g, nv, mode, direction, z, gamma)
    torch.cuda.synchronize()
    return outs, st, gamma, z, dev2, D


CASES = [("alie", "backdoor"), ("alie", "std"), ("minmax", "backdoor"), ("minsum", "sign")]


@pytest.mark.parametrize("mode,direction", CASES + [("minmax", "unit"), ("minsum", "std")])
@pytest.mark.parametrize("K,H", [(2, 1), (3, 1), (10, 7), (64, 56), (257, 250)])
@pytest.mark.parametrize("which", ["resnet18", "sweeps"])
def test_crafted_slots_match_the_statement(which, K, H, mode, direction):
    if which == "resnet18" and (mode, direction) not in CASES:
        pytest.skip("the other directions run at the sweeps size")
    ops.reset_fallbacks()
    nv = _sizes(which)
    g, ws = _participants(K, nv, K + H)
    honest, corrupt = ws[:H], ws[H:]
    tail = [c[nv:].clone() for c in corrupt]
    outs, st, gamma, z, dev2, D = _craft(honest, corrupt, g, nv, mode, direction)
    ref = ops.collude_statement(honest, corrupt, g, nv, mode, direction, z=z, gamma=gamma if mode != "alie" else None, D=D)
    for o, t in zip(outs, tail):
        assert torch.equal(o[:nv].view(torch.int32), ref["slot"].view(torch.int32))
        assert torch.equal(o[nv:], t)                                      # the BatchNorm tail is never touched
    assert float(dev2[0]) == pytest.approx(ref["dev2"], rel=RTOL, abs=1e-300)
    if st is not None:
        a, e, q = st[:H].cpu(), st[H:2 * H].cpu(), float(st[2 * H])
        ra, re = ref["a"].cpu(), ref["e"].cpu()
        assert q == pytest.approx(ref["q"], rel=RTOL)
        assert bool(((a - ra).abs() <= RTOL * ra.abs().max()).all())
        assert bool(((e - re).abs() <= RTOL * (ra * ref["q"]).sqrt().max() + 1e-300).all())
        if H == 1:
            assert gamma == 0.0 and torch.equal(outs[0][:nv], honest[0][:nv])
    assert ops.fallback_calls() == {}


@pytest.mark.parametrize("mode,direction", CASES)
def test_two_launches_are_bitwise_equal(mode, direction):
    nv = get_layout("resnet18").n_vote
    g, ws = _participants(40, nv, 9)
    a = _craft(ws[:32], ws[32:], g, nv, mode, direction)
    b = _craft(ws[:32], ws[32:], g, nv, mode, direction)
    assert all(torch.equal(x, y) for x, y in zip(a[0], b[0]))
    assert torch.equal(a[4], b[4]) and a[2] == b[2]
    if a[1] is not None:
        assert torch.equal(a[1], b[1])


def test_non_finite_honest_values_are_left_out():
    nv = _sizes("sweeps")
    g, ws = _participants(6, nv, 4)
    ws[1][17] = float("nan")
    ws[2][nv - 3] = float("inf")
    outs, st, gamma, z, dev2, D = _craft(ws[:4], ws[4:], g, nv, "alie", "backdoor")
    ref = ops.collude_statement(ws[:4], ws[4:], g, nv, "alie", "backdoor", z=z)
    assert torch.equal(outs[0][:nv].view(torch.int32), ref["slot"].view(torch.int32))
    assert bool(torch.isfinite(outs[0][:nv]).all())


# ---- the native trainer and the engine ---------------------------------------------------------------------------------------------
def _resnet_run(**kw):
    from rlr_b200.engine import FLEngine
    ops.reset_fallbacks()
    args = make_args(data="cifar10", model="resnet18", num_agents=5, num_corrupt=2, poison_frac=0.5, local_ep=1, bs=64, synthetic=640,
                     synthetic_val=128, log_dir="", seed=3, robustLR_threshold=2, device=DEV, **kw)
    eng = FLEngine(args, verbose=False)
    assert eng.trainer.name == "native"
    out = []
    for r in range(1, 3):
        chosen = eng.run_round(r)["chosen"]
        corrupt = eng.fused.slots[eng.fused.slot_owner(chosen.index(0))[1]].clone()
        eng.round_result()
        out.append((eng.global_params().clone(), corrupt, dict(eng.last_collude)))
    torch.cuda.synchronize()
    assert ops.fallback_calls() == {}
    eng.close()
    return out


@pytest.mark.parametrize("mode", ["alie", "minmax", "minsum"])
def test_native_engine_graphs_equal_eager_and_runs_repeat(mode):
    graphs = _resnet_run(attack_collude=mode)
    eager = _resnet_run(attack_collude=mode, no_graphs=True)
    again = _resnet_run(attack_collude=mode)
    for (wa, xa, la), (wb, xb, lb), (wc, xc, lc) in zip(graphs, eager, again):
        assert torch.equal(wa, wb) and torch.equal(xa, xb) and la == lb
        assert torch.equal(wa, wc) and torch.equal(xa, xc) and la == lc
        assert la["collude_honest"] == 3 and la["collude_deviation"] > 0


@pytest.mark.parametrize("kw", [dict(select="multikrum", num_agents=10), dict(select="dnc", num_agents=10), dict(aggr="rfa"),
                                dict(aggr="flame"), dict(aggr="foolsgold"), dict(detect="fldetector", num_agents=5)])
def test_one_round_under_each_defense(kw):
    from rlr_b200.engine import FLEngine
    ops.reset_fallbacks()
    base = dict(data="cifar10", model="cnn_cifar", num_agents=6, num_corrupt=2, poison_frac=0.5, local_ep=1, bs=64, synthetic=1280,
                synthetic_val=128, log_dir="", seed=4, robustLR_threshold=0, device=DEV, attack_collude="minmax", rounds=1)
    base.update(kw)
    eng = FLEngine(make_args(**base), verbose=False)
    hist = eng.fit()
    torch.cuda.synchronize()
    assert hist[0]["collude_honest"] > 0 and bool(torch.isfinite(eng.global_params()).all())
    assert ops.fallback_calls() == {}
    eng.close()


# ---- two or more GPUs: the fused multi-GPU path ----------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _multi_args(world, clip):
    return dict(data="cifar10", model="cnn_cifar", synthetic=128 * 2 * world, synthetic_val=128, num_agents=2 * world, num_corrupt=2,
                poison_frac=0.5, local_ep=1, bs=64, log_dir="", seed=7, robustLR_threshold=0, attack_collude="minsum",
                collude_dir="std", server_clip=clip)


def _multi_worker(rank, world, port, outdir, clip):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200.engine import FLEngine
    eng = FLEngine(make_args(**_multi_args(world, clip)), verbose=False)
    devs = []
    for r in range(1, 3):
        eng.run_round(r)
        eng.round_result()
        devs.append(eng.last_collude["collude_deviation"])
    torch.save({"w": eng.global_params().clone().cpu(), "devs": devs, "backend": eng.fused.backend}, os.path.join(outdir, f"r{rank}.pt"))
    eng.close()
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("clip", [False, True])
def test_fused_multi_gpu_agrees_with_one_gpu(tmp_path, clip):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_multi_worker, args=(world, _free_port(), str(tmp_path), clip), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"r{r}.pt") for r in range(world)]
    assert res[0]["backend"] == "fused"
    for r in res[1:]:
        assert torch.equal(r["w"], res[0]["w"]) and r["devs"] == res[0]["devs"]
    from rlr_b200.engine import FLEngine
    one = FLEngine(make_args(device=DEV, **_multi_args(world, clip)), verbose=False)
    devs = []
    for r in range(1, 3):
        one.run_round(r)
        devs.append(one.last_collude["collude_deviation"])
    np.testing.assert_allclose(devs, res[0]["devs"], rtol=1e-4)
    torch.testing.assert_close(one.global_params().cpu(), res[0]["w"], rtol=1e-3, atol=1e-4)
    one.close()
