"""FLARE on the H100: ``flare_mmd_kernel`` (ops/csrc/flare.cu) against the fp64 statement for 1 to 200 candidates, 1 to 300 root samples
and feature widths 128 / 256 / 512, with the neighbour counts and weights it yields; run-to-run bitwise equality; the native feature tap
against the torch trainer's for every zoo model; the dict and slots forms of the server step against each other and the oracle; a
reproducible CIFAR-10 ResNet-18 engine run; the engine with the fused hand-off against the barrier path, on one GPU and -- with two or
more -- on the fused multi-GPU path."""
import math
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.aggregation import Aggregation
from rlr_b200.options import MODELS, make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def kappa_tol(d: int) -> float:
    """Bound on |kappa - exp(-D/sigma^2)| of one kernel value: the fp32 distance (d rounded differences squared, d - 1 additions) and
    the fp32 exponent carry a relative error of at most (d + 3) 2^-24, which moves exp(-x) by at most x e^-x (d + 3) 2^-24 <= (d + 3)
    2^-24 / e; expf adds at most 2 ulp.  Every M entry combines three kernel-sum averages with weights 1, 1 and 2: |dM| <= 4 kappa_tol."""
    return (d + 3) * 2.0 ** -24 / math.e + 2.0 ** -23


def _features(K, n, d, seed, bad=()):
    """K candidates' features in four clusters (candidate k in cluster k % 4, its own offset on top), ReLU-like non-negative values
    as a head's input has; candidates in ``bad`` get one NaN."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    centres = torch.randn(4, d, generator=gen, device=DEV)
    Z = torch.empty(K, n, d, device=DEV)
    for k in range(K):
        off = 0.3 * torch.randn(d, generator=gen, device=DEV)
        Z[k] = torch.relu(centres[k % 4] + off + 0.5 * torch.randn(n, d, generator=gen, device=DEV))
    for k in bad:
        Z[k, n // 2, d // 3] = float("nan")
    return Z


def _boundary_clear(M, k, tol):
    """True when no row of M has its k-th and (k+1)-th smallest off-diagonal entries within 2 tol of each other, so an error of tol
    per entry cannot change any neighbour list."""
    F = M.shape[0]
    k = max(0, min(k, F - 1))
    if k == 0 or k == F - 1:
        return True
    for i in range(F):
        row = np.sort(np.delete(M[i], i))
        if row[k] - row[k - 1] <= 2 * tol:
            return False
    return True


@pytest.mark.parametrize("K,n,d,bad", [(1, 37, 128, ()), (2, 1, 256, ()), (3, 300, 512, (1,)), (8, 100, 512, ()), (8, 300, 256, (0, 5)),
                                       (40, 100, 512, ()), (100, 37, 256, (7,)), (200, 1, 512, ()), (200, 37, 128, (3, 150))])
def test_kernel_matches_fp64_statement(K, n, d, bad):
    Z = _features(K, n, d, K * 7 + n, bad)
    finite = torch.isfinite(Z.reshape(K, -1)).all(1)
    F = [j for j in range(K) if bool(finite[j])]
    s2 = ops.flare_sigma2(Z, F)
    if s2 is None:                                                   # one candidate, one sample: nothing to pool
        assert len(F) * n < 2
        return
    S = ops.flare_sums(Z, finite, s2)
    ref = ops.flare_sums_statement(Z, finite.cpu().tolist(), s2)
    tol = kappa_tol(d)
    err_k = float(np.abs(S - ref).max()) / (n * n)
    M, Mr = ops.flare_mmd_matrix(S, F, n), ops.flare_mmd_matrix(ref, F, n)
    err_m = float(np.abs(M - Mr).max())
    print(f"K={K} n={n} d={d}: max |dS|/n^2 {err_k:.2e}, max |dM| {err_m:.2e} (bounds {tol:.2e}, {4 * tol:.2e}), M up to {Mr.max():.3f}")
    assert err_k <= tol and err_m <= 4 * tol
    for j in range(K):
        if j not in F:
            assert (S[j] == 0).all() and (S[:, j] == 0).all()
    assert np.array_equal(np.diag(M), np.zeros(len(F))) and np.array_equal(M, M.T)
    k = len(F) // 2
    if _boundary_clear(Mr, k, 4 * tol):
        ts, c = ops.flare_weights(M, F, k, 1.0)
        ts_r, c_r = ops.flare_weights(Mr, F, k, 1.0)
        assert np.array_equal(c, c_r) and np.array_equal(ts, ts_r)
    else:
        print("  a neighbour boundary lies within the tolerance: counts not compared")


@pytest.mark.parametrize("K,n,d", [(8, 100, 512), (40, 37, 256), (100, 100, 512)])
def test_two_launches_are_bitwise_equal(K, n, d):
    Z = _features(K, n, d, 11)
    finite = torch.ones(K, dtype=torch.bool, device=DEV)
    s2 = ops.flare_sigma2(Z, list(range(K)))
    a = ops.flare_sums(Z, finite, s2)
    b = ops.flare_sums(Z, finite, s2)
    assert np.array_equal(a, b)


def test_identical_candidates_have_zero_mmd_on_the_device():
    Z = _features(6, 100, 256, 4)
    Z[3] = Z[1]
    res = ops.flare(Z)
    i, j = res.members.index(1), res.members.index(3)
    assert res.M[i, j] == 0.0 and res.M[j, i] == 0.0


# ---- the feature tap --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", [m for m in MODELS if m != "auto"])
def test_native_feature_tap_matches_the_torch_trainer(model):
    from rlr_b200.models import get_layout
    from rlr_b200.models.graph import feature_dim
    from rlr_b200.models.native import NativeTrainer
    from rlr_b200.trainers import TorchTrainer
    lay = get_layout(model)
    data = "fmnist" if lay.in_shape[0] == 1 else "cifar10"
    args = make_args(data=data, model=model, bs=32, device=DEV)
    w = torch.zeros(lay.n_total, device=DEV)
    lay.init_(w, 3)
    gen = torch.Generator(device=DEV).manual_seed(5)
    for b in lay.buffers:                                            # non-trivial running statistics: eval mode must use them
        v = lay.view(w, b)
        v.copy_(0.1 * torch.randn(v.shape, generator=gen, device=DEV) if b.kind == "bn_mean" else
                0.5 + torch.rand(v.shape, generator=gen, device=DEV))
    C, H, W = lay.in_shape
    x = torch.randn(70, C, H, W, generator=gen, device=DEV)         # three chunks of --bs 32
    ref_tr = TorchTrainer(lay, make_args(data=data, model=model, bs=32, dtype="fp32", device=DEV), DEV, 64)
    ref = ref_tr.root_features(w, x)
    nat = NativeTrainer(lay, args, DEV, 64)
    ops.reset_fallbacks()
    nat.eval_forward(w)(x[:32])
    eval_fb = set(ops.fallback_calls())
    ops.reset_fallbacks()
    z = nat.root_features(w, x)
    torch.cuda.synchronize()
    assert set(ops.fallback_calls()) <= eval_fb                       # the tap runs no path the eval forward does not
    assert z.shape == ref.shape == (70, feature_dim(lay)) and z.dtype == torch.float32
    assert torch.equal(z, z.to(torch.bfloat16).float())               # bf16 activations widened to fp32
    rel = float((z - ref).norm() / ref.norm())
    print(f"{model}: d={z.shape[1]} rel err vs the fp32 torch trainer {rel:.2e}")
    assert rel < 3e-2
    w2 = w.clone()
    w2[: lay.n_vote] += 0.01
    assert not torch.equal(nat.root_features(w2, x), z)               # the executor follows the parameters it is handed
    assert torch.equal(nat.root_features(w, x), z)


# ---- the server step ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("theta,bad,k", [(0, (), None), (2, (4,), None), (2, (), 2), (0, tuple(range(10)), None)])
def test_dict_and_slots_forms_match_each_other_and_the_oracle(theta, bad, k):
    from rlr_b200.parallel import FusedAggregator, init_distributed
    K, n, nv, R, d = 10, 1 << 20, (1 << 20) - 4096, 64, 256
    gen = torch.Generator(device=DEV).manual_seed(21)
    g = torch.randn(n, generator=gen, device=DEV)
    ws = [g + 0.01 * (1 + j % 3) * torch.randn(n, generator=gen, device=DEV) for j in range(K)]
    Z = _features(K, R, d, 3, bad)
    a = make_args(num_agents=K, num_corrupt=2, aggr="flare", robustLR_threshold=theta, flare_k=k, device=DEV)
    sizes = {i: 100 + 13 * i for i in range(K)}
    wg = g.clone()
    dict_form = Aggregation(sizes, n, None, a)
    dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv, features=Z)
    fa = FusedAggregator(init_distributed(DEV), n, nv, K, "local")
    fa.w_global.copy_(g)
    for j, w in enumerate(ws):
        fa.slots[j].copy_(w)
    slots_form = Aggregation(sizes, n, None, a, fused=fa)
    slots_form.aggregate_slots(list(range(K)), 1, Z.clone())
    torch.cuda.synchronize()
    assert torch.equal(fa.w_global, wg) and slots_form.last_admitted == dict_form.last_admitted
    assert slots_form.last_flare == dict_form.last_flare
    res = ops.flare_statement(Z, k, 1.0)
    F = res.members
    assert dict_form.last_admitted == F == [j for j in range(K) if j not in bad]
    if F:
        wts = [float(np.float32(res.weights[j])) for j in F]
        ref, _ = ops.aggregate_oracle(g, [ws[j] for j in F], wts, "avg", theta, 1.0, None, nv, None, None)
    else:
        ref = g
    err = float((wg - ref).abs().max())
    print(f"theta={theta} bad={bad} k={k}: max |w - oracle| {err:.2e}, trust {dict_form.last_flare}")
    assert err < 2e-6


def test_engine_resnet18_flare_is_reproducible():
    from rlr_b200.engine import FLEngine

    def run():
        ops.reset_fallbacks()
        args = make_args(data="cifar10", model="resnet18", num_agents=4, num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, synthetic=512,
                         synthetic_val=128, log_dir="", seed=3, aggr="flare", root_size=80, robustLR_threshold=2, device=DEV)
        eng = FLEngine(args, verbose=False)
        out = []
        for r in range(1, 3):
            eng.run_round(r)
            out.append((eng.global_params().clone(), dict(eng.aggregator.last_flare), list(eng.aggregator.last_admitted)))
        torch.cuda.synchronize()
        assert ops.fallback_calls() == {}
        eng.close()
        return out

    a, b = run(), run()
    for (wa, fa, aa), (wb, fb, ab) in zip(a, b):
        assert torch.equal(wa, wb) and fa == fb and aa == ab and sorted(aa) == [0, 1, 2, 3]
        assert fa["FLARE/Bandwidth"] > 0 and abs(fa["FLARE/Avg_Honest_Trust"] * 3 + fa["FLARE/Corrupt_Weight"] - 1.0) < 1e-9
    print("FLARE per round:", [f for _, f, _ in a])


# ---- the fused hand-off against the barrier path, on one GPU and on the fused multi-GPU path -------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _engine_run(world, handoff):
    from rlr_b200.engine import FLEngine
    args = make_args(data="cifar10", model="cnn_cifar", synthetic=128 * max(5, 2 * world), synthetic_val=128, num_agents=max(5, 2 * world),
                     num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, log_dir="", seed=7, aggr="flare", root_size=64, robustLR_threshold=2,
                     no_fused_handoff=not handoff, **({} if world > 1 else {"device": DEV}))
    eng = FLEngine(args, verbose=False)
    assert eng.handoff == handoff
    snaps, trust = [], []
    for r in range(1, 5):
        eng.run_round(r)
        snaps.append(eng.global_params().clone().cpu())
        trust.append(dict(eng.aggregator.last_flare))
    torch.cuda.synchronize()
    same = True
    if world > 1:
        allw = eng.ctx.all_gather(eng.global_params().clone())
        same = bool((allw == allw[0:1]).all().item())
        same = same and all(t == trust[i] for i, t in enumerate(eng.ctx.all_gather_object(trust)[0]))
    out = {"w": snaps, "trust": trust, "same": same, "backend": eng.fused.backend}
    eng.close()
    return out


def _engine_worker(rank, world, port, outdir, handoff, tag):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    torch.save(_engine_run(world, handoff), os.path.join(outdir, f"eng_{tag}_{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("multi", [False, True])
def test_engine_flare_with_fused_handoff_equals_barrier_path(tmp_path, multi):
    """Two barrier-path runs (a, b) measure the run-to-run noise of the native trainer; the hand-off run (f) must stay within that noise.
    multi: every GPU, one rank each, on the fused multi-GPU path, where every rank must hold the same weights and parameters."""
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
            assert res[t][r]["same"], (t, r)
    print("trust per round:", res["a"][0]["trust"])
    rel = lambda x, y: float((x.double() - y.double()).norm() / (y.double().norm() + 1e-12))
    for i in range(4):
        noise, diff = rel(res["b"][0]["w"][i], res["a"][0]["w"][i]), rel(res["f"][0]["w"][i], res["a"][0]["w"][i])
        print(f"world {world} round {i + 1}: barrier-vs-barrier {noise:.2e}  handoff-vs-barrier {diff:.2e}")
        assert diff <= 3 * noise + (1e-5 if i == 0 else 1e-4), (i, diff, noise)
