"""DeepSight on the H100: the statistics pass (ops/csrc/deepsight.cu) against the fp64 statement for 1 to 200 candidates, 1 to 2048
samples per seed and 1 to 1024 classes (the pass's bound); run-to-run bitwise equality; the refusal above the bound; the native logits
against the torch trainer's for every zoo model; the dict and slots forms of the server step against each other; a reproducible CIFAR-10
ResNet-18 engine run; and, with two or more GPUs, the fused multi-GPU path against one GPU."""
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
S = ops.DEEPSIGHT_SEEDS


def ddif_rtol(P: int, N: int, L: float) -> float:
    """Relative bound on |DDif_device - DDif_statement|.  Both sides take the same fp32 logits.  An lse is a max (exact), P exps of
    arguments <= 0 (1 ulp each on the device and in libm), a left-to-right sum of P terms ((P - 1) roundings) and a log (1 ulp), so it is
    off by at most (P + 3) 2^-53 max(1, L) absolute, L the largest |logit| + log P.  The exponent of a term adds two lse errors and three
    subtractions (3 roundings of a value <= 4L), so exp moves by a relative 2 (P + 3) 2^-53 max(1, L) + 12 L 2^-53, and exp adds 1 ulp
    on each side.  The N terms are positive and added left to right on both sides: at most N - 1 roundings each, relative.  Twice the
    sum covers both sides."""
    u = 2.0 ** -53
    L = max(1.0, L)
    return 2.0 * ((2 * (P + 3) + 12) * L * u + 4 * u + 2 * N * u)


def _case(K, N, P, d, seed, bad=(), scale=3.0):
    """K candidates: random logits (scale ``scale``) on S seeds of N rows, the global model's, and flat parameter vectors holding a head
    weight [P][d] and bias [P] at offsets that are not multiples of 4; candidates in ``bad`` get a non-finite logit."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    z = scale * torch.randn(K, S * N, P, generator=gen, device=DEV)
    zg = scale * torch.randn(S * N, P, generator=gen, device=DEV)
    for j, k in enumerate(bad):
        z[k, (7 * j) % (S * N), j % P] = (float("nan"), float("inf"), -float("inf"))[j % 3]
    w_off, b_off = 5, 5 + P * d + 3
    n = (b_off + P + 3) // 4 * 4 + 4
    wg = torch.randn(n, generator=gen, device=DEV)
    ws = [wg + 0.01 * (1 + k % 5) * torch.randn(n, generator=gen, device=DEV) for k in range(K)]
    return z, zg, ws, wg, (w_off, b_off, P, d)


@pytest.mark.parametrize("K,N,P,d,bad", [(1, 1, 1, 1, ()), (2, 16, 10, 512, ()), (8, 256, 10, 512, (3,)), (40, 256, 62, 128, (0, 7, 39)),
                                         (200, 64, 10, 256, ()), (3, 2048, 10, 64, ()), (2, 8, 1024, 32, (1,)), (5, 300, 1024, 16, ())])
def test_kernel_matches_fp64_statement(K, N, P, d, bad):
    z, zg, ws, wg, head = _case(K, N, P, d, 11 + K + N + P, bad)
    got = ops.deepsight_stats(z, zg, ws, wg, head)
    torch.cuda.synchronize()
    ref = ops.deepsight_stats_statement(z, zg, ws, wg, head)
    g, r = got.cpu().numpy(), ref.numpy()
    assert g.shape == r.shape == (K, (S + 2) * P)
    # eps and db: exact fp32 differences and fp64 additions of |values| in the same left-to-right order on both sides
    assert np.array_equal(g[:, S * P:], r[:, S * P:])
    L = float(z[torch.isfinite(z)].abs().max()) + float(np.log(P))
    tol = ddif_rtol(P, N, L)
    worst = 0.0
    for k in range(K):
        a, b = g[k, :S * P], r[k, :S * P]
        assert np.array_equal(np.isnan(a), np.isnan(b))
        if k in bad:                                                  # a non-finite logit makes its seed's DDif NaN
            assert np.isnan(a).any()
        else:
            assert np.isfinite(a).all()
        ok = np.isfinite(b)
        rel = np.abs(a[ok] - b[ok]) / np.abs(b[ok])
        worst = max(worst, float(rel.max()) if rel.size else 0.0)
    print(f"K={K} N={N} P={P} d={d}: worst relative DDif error {worst:.2e}, bound {tol:.2e}")
    assert worst <= tol


@pytest.mark.parametrize("K,N,P", [(8, 256, 10), (100, 256, 10), (40, 512, 62)])
def test_two_launches_are_bitwise_equal(K, N, P):
    z, zg, ws, wg, head = _case(K, N, P, 512, 3)
    a = ops.deepsight_stats(z, zg, ws, wg, head).clone()
    b = ops.deepsight_stats(z, zg, ws, wg, head)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_a_class_count_above_the_bound_is_refused():
    z, zg, ws, wg, head = _case(2, 4, 1025, 8, 1)
    with pytest.raises(RuntimeError, match="classes"):
        ops.deepsight_stats(z, zg, ws, wg, head)


def test_a_candidate_equal_to_the_global_model_on_the_device():
    z, zg, ws, wg, head = _case(3, 64, 10, 128, 2)
    z[1] = zg
    ws[1] = wg.clone()
    st = ops.deepsight_stats(z, zg, ws, wg, head).cpu().numpy()
    assert np.array_equal(st[1, :S * 10], np.ones(S * 10)) and not st[1, S * 10:].any()


# ---- the logits -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", [m for m in MODELS if m != "auto"])
def test_native_logits_match_the_torch_trainer(model):
    """The native eval-mode logits (bf16 activations, the head's output widened to fp32) against the fp32 torch trainer's.  A bf16
    forward carries a relative error of a few 2^-8 per layer in the activations; 3e-2 of the logits' norm is the bound the feature tap
    meets, and the head adds one more bf16 rounding (2^-9 relative)."""
    from rlr_b200.data import DATASET_META
    from rlr_b200.models import get_layout
    from rlr_b200.models.graph import head_slices
    from rlr_b200.models.native import NativeTrainer
    from rlr_b200.trainers import TorchTrainer
    lay = get_layout(model)
    data = "fmnist" if lay.in_shape[0] == 1 else "cifar10"
    w = torch.zeros(lay.n_total, device=DEV)
    lay.init_(w, 3)
    gen = torch.Generator(device=DEV).manual_seed(5)
    for b in lay.buffers:
        v = lay.view(w, b)
        v.copy_(0.1 * torch.randn(v.shape, generator=gen, device=DEV) if b.kind == "bn_mean" else
                0.5 + torch.rand(v.shape, generator=gen, device=DEV))
    x = ops.deepsight_inputs(DATASET_META[data], 4, 40, DEV)          # 120 random images: several chunks of --bs 32
    ref = TorchTrainer(lay, make_args(data=data, model=model, bs=32, dtype="fp32", device=DEV), DEV, 64).root_features(w, x, tap=False)
    nat = NativeTrainer(lay, make_args(data=data, model=model, bs=32, device=DEV), DEV, 64)
    ops.reset_fallbacks()
    nat.eval_forward(w)(x[:32])
    eval_fb = set(ops.fallback_calls())
    ops.reset_fallbacks()
    z = nat.root_features(w, x, tap=False)
    torch.cuda.synchronize()
    assert set(ops.fallback_calls()) <= eval_fb
    assert z.shape == ref.shape == (120, head_slices(lay)[2]) and z.dtype == torch.float32
    rel = float((z - ref).norm() / ref.norm())
    print(f"{model}: P={z.shape[1]} rel err of the logits vs the fp32 torch trainer {rel:.2e}")
    assert rel < 3e-2 + 2.0 ** -9
    assert torch.equal(nat.root_features(w, x, tap=False), z)


# ---- the server step ------------------------------------------------------------------------------------------------------------
def _round(lay, K, seed):
    """A round on ``lay``'s flat vectors: honest candidates move every parameter a little and answer the random inputs like the global
    model; candidates 0 and 1 (corrupt) move only row 0 of the head and its bias, and raise logit 0 -- a one-label poisoned head."""
    from rlr_b200.models.graph import head_slices
    w_off, b_off, P, d = head = head_slices(lay)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randn(lay.n_total, generator=gen, device=DEV)
    zg = torch.randn(S * 32, P, generator=gen, device=DEV)
    ws, z = [], []
    for k in range(K):
        w = g + 0.01 * torch.randn(lay.n_total, generator=gen, device=DEV)
        zk = zg + 0.05 * torch.randn(S * 32, P, generator=gen, device=DEV)
        if k < 2:
            w[w_off:w_off + P * d] = g[w_off:w_off + P * d]
            w[b_off:b_off + P] = g[b_off:b_off + P]
            w[w_off:w_off + d] += 0.5
            w[b_off] += 0.5
            zk[:, 0] += 2.0
        ws.append(w)
        z.append(zk)
    return g, ws, torch.stack(z), zg, head


def test_dict_and_slots_forms_match_each_other():
    from rlr_b200.models import get_layout
    from rlr_b200.parallel import FusedAggregator, init_distributed
    K = 10
    lay = get_layout("cnn_cifar")
    g, ws, z, zg, head = _round(lay, K, 21)
    n = g.numel()
    a = make_args(num_agents=K, num_corrupt=2, aggr="deepsight", robustLR_threshold=2, noise=0.01, clip=0.5, device=DEV)
    sizes = {i: 100 + 13 * i for i in range(K)}
    wg = g.clone()
    dict_form = Aggregation(sizes, lay.n_params, None, a, layout=lay)
    dict_form.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, logits=z, global_logits=zg)
    fa = FusedAggregator(init_distributed(DEV), n, lay.n_vote, K, "local")
    fa.w_global.copy_(g)
    for j, w in enumerate(ws):
        fa.slots[j].copy_(w)
    local = ops.deepsight_stats(z, zg, [fa.slots[j] for j in range(K)], fa.w_global, head)
    slots_form = Aggregation(sizes, lay.n_params, None, a, layout=lay, fused=fa)
    slots_form.aggregate_slots(list(range(K)), 1, deepsight_local=local)
    torch.cuda.synchronize()
    assert torch.equal(fa.w_global, wg) and slots_form.last_admitted == dict_form.last_admitted
    assert slots_form.last_deepsight == dict_form.last_deepsight
    assert dict_form.last_admitted == list(range(2, K)), dict_form.last_deepsight
    assert dict_form.last_deepsight["DeepSight/Corrupt_Suspicious"] == 2
    fa.close()


def test_engine_resnet18_deepsight_is_reproducible():
    from rlr_b200.engine import FLEngine

    def run():
        ops.reset_fallbacks()
        args = make_args(data="cifar10", model="resnet18", num_agents=4, num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, synthetic=512,
                         synthetic_val=128, log_dir="", seed=3, aggr="deepsight", deepsight_samples=64, device=DEV)
        eng = FLEngine(args, verbose=False)
        out = []
        for r in range(1, 3):
            eng.run_round(r)
            out.append((eng.global_params().clone(), dict(eng.aggregator.last_deepsight), list(eng.aggregator.last_admitted),
                        eng.ds_local.clone()))
        torch.cuda.synchronize()
        assert ops.fallback_calls() == {}
        eng.close()
        return out

    a, b = run(), run()
    for (wa, fa, aa, sa), (wb, fb, ab, sb) in zip(a, b):
        assert torch.equal(wa, wb) and fa == fb and aa == ab and torch.equal(sa, sb)
        assert torch.isfinite(sa).all() and fa["DeepSight/Clip_Bound"] > 0
    print("DeepSight per round:", [f for _, f, _, _ in a])


# ---- the fused multi-GPU path against one GPU -------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _engine_run(world):
    from rlr_b200.engine import FLEngine
    args = make_args(data="cifar10", model="cnn_cifar", synthetic=128 * 8, synthetic_val=128, num_agents=8, num_corrupt=2,
                     poison_frac=0.5, local_ep=1, bs=64, log_dir="", seed=7, aggr="deepsight", deepsight_samples=64, robustLR_threshold=2,
                     **({} if world > 1 else {"device": DEV}))
    eng = FLEngine(args, verbose=False)
    snaps, recs = [], []
    for r in range(1, 4):
        eng.run_round(r)
        snaps.append(eng.global_params().clone().cpu())
        recs.append((dict(eng.aggregator.last_deepsight), list(eng.aggregator.last_admitted)))
    torch.cuda.synchronize()
    same = True
    if world > 1:
        allw = eng.ctx.all_gather(eng.global_params().clone())
        same = bool((allw == allw[0:1]).all().item())
        same = same and all(t == recs[i] for i, t in enumerate(eng.ctx.all_gather_object(recs)[0]))
    out = {"w": snaps, "recs": recs, "same": same, "backend": eng.fused.backend}
    eng.close()
    return out


def _engine_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    torch.save(_engine_run(world), os.path.join(outdir, f"eng_{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


def test_engine_fused_multi_gpu_equals_one_gpu(tmp_path):
    """Every GPU, one rank each, on the fused multi-GPU path: every rank holds the same parameters and decisions, and the decisions
    of the first round (before training noise between the two placements can build up) equal one GPU's."""
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_engine_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    multi = [torch.load(tmp_path / f"eng_{r}.pt") for r in range(world)]
    one = _engine_run(1)
    assert multi[0]["backend"] == "fused" and all(m["same"] for m in multi)
    assert multi[0]["recs"][0] == one["recs"][0]
    rel = float((multi[0]["w"][0].double() - one["w"][0].double()).norm() / one["w"][0].double().norm())
    print(f"world {world}: round-1 relative difference to one GPU {rel:.2e}; decisions {multi[0]['recs']}")
    assert rel < 1e-4
