"""GPU: the model-poisoning attack kernels (ops/csrc/attack.cu and the masked optimizer instantiations of ops/csrc/elementwise.cu).

* Neurotoxin's mask pass against ``ops.neurotoxin_statement``, bitwise (mask words, |M|, the refreshed ``w_prev``), at the ResNet-18
  ``n_vote`` and at sizes that take several sweeps of the capped grid with a remainder that is not a multiple of 32, on the CPU test's
  edge inputs, and repeatably across launches;
* the masked ``sqnorm`` / ``sgd_step`` / ``pgd_project`` (plain, PGD, first step) against the fp64 statement and error bound of
  tests/test_gpu_flat_kernels.py, masked coordinates bit for bit, an empty mask bit for bit like the unmasked launch;
* ``boost_update`` bitwise against its statement;
* the native trainer and the engine with both attacks (graph replay against --no_graphs, reproducibility, no library fall-through),
  and the fused multi-GPU hand-off (skipped below two GPUs)."""
import importlib.util
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
from rlr_b200.models import get_layout
from rlr_b200.options import make_args

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_spec = importlib.util.spec_from_file_location("_flat", os.path.join(os.path.dirname(__file__), "test_gpu_flat_kernels.py"))
flat = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(flat)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def hist_sweep():
    """Coordinates one sweep of the histogram passes covers (ops/csrc/attack.cu: 4 CTAs / SM x 512 threads x 4 coordinates)."""
    return _sms() * 4 * 512 * 4


def _mask_inputs(n, seed, zero_frac=0.1):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    w_prev = torch.randn(n, generator=gen, device=DEV)
    w_g = w_prev + 1e-3 * torch.randn(n, generator=gen, device=DEV)
    keep = torch.rand(n, generator=gen, device=DEV) < zero_frac
    w_g[keep] = w_prev[keep]                                        # exact zero changes: never masked
    return w_g, w_prev


def _run_mask(w_g, w_prev, n_vote, k):
    mask = torch.full((ops.mask_words(n_vote),), -1, dtype=torch.int32, device=DEV)
    count = torch.full((1,), -1, dtype=torch.int64, device=DEV)
    wp = w_prev.clone()
    ops.neurotoxin_mask(w_g, wp, n_vote, k, mask, count)
    torch.cuda.synchronize()
    return mask.cpu().numpy().view(np.uint32), int(count), wp


def _check_mask(w_g, w_prev, n_vote, k):
    words, count, wp = _run_mask(w_g, w_prev, n_vote, k)
    ref, ref_count = ops.neurotoxin_statement(w_g, w_prev, n_vote, k)
    assert np.array_equal(words, ref), (n_vote, k, int((words != ref).sum()))
    assert count == ref_count, (n_vote, k, count, ref_count)
    assert torch.equal(wp[:n_vote].view(torch.int32), w_g[:n_vote].view(torch.int32))         # w_prev refreshed bit for bit
    assert torch.equal(wp[n_vote:], w_prev[n_vote:])
    return words, count


def _size(which):
    """The ResNet-18 n_vote; three sweeps of the histogram grid plus a remainder that is a multiple of 4 but not of 32; one CTA's worth."""
    if which == "resnet18":
        return get_layout("resnet18").n_vote
    if which == "sweeps":
        S = hist_sweep()
        n = 3 * S + (S // 2) // 8 * 8 + 4
        assert n % 4 == 0 and n % 32
        return n
    return 1028


@pytest.mark.parametrize("which", ["resnet18", "sweeps", "small"])
def test_mask_kernel_matches_the_statement(which):
    n = _size(which)
    w_g, w_prev = _mask_inputs(n, n % 1000)
    for k in (1, int(0.01 * n), int(0.5 * n), int(0.9 * n), n):
        _check_mask(w_g, w_prev, n, k)


def test_mask_kernel_on_edge_inputs():
    n = 3 * hist_sweep() + 36
    w_prev = torch.zeros(n, device=DEV)
    assert _check_mask(w_prev.clone(), w_prev, n, 100)[1] == 0      # no change: empty mask
    assert _check_mask(torch.randn(n, device=DEV), w_prev, n, 0)[1] == 0
    gen = torch.Generator(device=DEV).manual_seed(9)
    levels = torch.tensor([0.0, 1e-3, 2e-3], device=DEV)
    ties = levels[torch.randint(0, 3, (n,), generator=gen, device=DEV)] * torch.where(torch.rand(n, generator=gen, device=DEV) < .5, 1., -1.)
    n_top, n_nz = int((ties.abs() == 2e-3).sum()), int((ties != 0).sum())
    for k in (1, n_top, n_top + 1, n_nz, n):
        assert _check_mask(ties, w_prev, n, k)[1] == (n_top if k <= n_top else n_nz)
    edge = 1e-3 * torch.randn(n, generator=gen, device=DEV)
    idx = torch.randperm(n, generator=gen, device=DEV)[:70]
    vals = torch.tensor([0.0, -0.0, 1e-45, -1e-44, 1e-39, float("inf"), -float("inf"), float("nan")], device=DEV)
    edge[idx] = vals.repeat(9)[:70]
    for k in (1, 10, 30, 1000, n // 2, n):
        _check_mask(edge, w_prev, n, k)


def test_mask_kernel_is_bitwise_repeatable():
    n = get_layout("resnet18").n_vote
    w_g, w_prev = _mask_inputs(n, 4)
    k = int(0.01 * n)
    runs = [_run_mask(w_g, w_prev, n, k) for _ in range(3)]
    for words, count, _ in runs[1:]:
        assert np.array_equal(words, runs[0][0]) and count == runs[0][1] >= k


# ---- the masked optimizer step ------------------------------------------------------------------------------------------------------
def _mask_of(k, seed, frac=0.2):
    gen = torch.Generator().manual_seed(seed)
    bits = torch.rand(k, generator=gen) < frac
    pad = np.zeros(ops.mask_words(k) * 32 - k, dtype=bool)
    words = np.packbits(np.concatenate([bits.numpy(), pad]), bitorder="little").view(np.int32).copy()
    return bits, torch.from_numpy(words).to(DEV)


@pytest.mark.parametrize("pgd", ["off", "inside", "projected"])
def test_masked_step_matches_fp64_statement(pgd):
    n, k = flat._sizes(flat.flat_sweep(), 2)
    gen = torch.Generator(device=DEV).manual_seed(21 + len(pgd))
    bits, words = _mask_of(k, len(pgd))
    dbits = bits.to(DEV)
    w0 = torch.randn(n, generator=gen, device=DEV)
    w0[:k][dbits & (torch.rand(k, generator=gen, device=DEV) < 0.01)] = -0.0
    w = w0.clone()
    m = 1e-3 * torch.randn(n, generator=gen, device=DEV)
    m[:k][dbits] = 0                                                # a masked coordinate never gains momentum in a round
    shadow = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
    clip = flat.PGD_CLIP[pgd]
    opt = ops.FlatSGD(n, DEV, flat.LR, flat.MU, flat.MAX_NORM, clip, n_pgd=k)
    for _ in range(3):
        g = torch.randn(n, generator=gen, device=DEV) * 30.0
        gm = g.cpu().clone()
        gm[:k][bits] = 0
        ref = flat._sgd_statement(w.cpu(), gm, m.cpu(), w0.cpu(), clip, k)
        opt.step(w, g, m, w0=w0 if pgd != "off" else None, w_bf16=shadow, grad_mask=words)
        flat._check_step(opt, w, m, shadow, ref, n, k)
        assert torch.equal(w[:k][dbits].view(torch.int32), w0[:k][dbits].view(torch.int32))    # bit for bit, -0 included


@pytest.mark.parametrize("pgd", ["off", "projected"])
def test_masked_first_step_matches_fp64_statement(pgd):
    n, k = flat._sizes(flat.flat_sweep(), 2)
    gen = torch.Generator(device=DEV).manual_seed(31 + len(pgd))
    bits, words = _mask_of(k, 7)
    w_in = torch.randn(n, generator=gen, device=DEV)
    w = torch.full((n,), float("nan"), device=DEV)
    w[k:] = 7.0
    m = torch.full((n,), float("nan"), device=DEV)
    shadow = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
    g = torch.randn(n, generator=gen, device=DEV) * 30.0
    gm = g.cpu().clone()
    gm[:k][bits] = 0
    opt = ops.FlatSGD(n, DEV, flat.LR, flat.MU, flat.MAX_NORM, flat.PGD_CLIP[pgd], n_pgd=k)
    ref = flat._sgd_statement(w.cpu(), gm, torch.zeros(n), w_in.cpu(), flat.PGD_CLIP[pgd], k, w_in=w_in.cpu())
    opt.step(w, g, m, w0=w_in if pgd != "off" else None, w_bf16=shadow, w_in=w_in, grad_mask=words)
    flat._check_step(opt, w, m, shadow, ref, n, k, shadow_upto=None if pgd != "off" else k)
    dbits = bits.to(DEV)
    assert torch.equal(w[:k][dbits], w_in[:k][dbits]) and bool((w[k:] == 7.0).all())


@pytest.mark.parametrize("first", [False, True])
@pytest.mark.parametrize("pgd", ["off", "projected"])
def test_empty_mask_equals_the_unmasked_launch(pgd, first):
    n, k = flat._sizes(flat.flat_sweep(), 2)
    gen = torch.Generator(device=DEV).manual_seed(41)
    w0, g, m0 = (torch.randn(n, generator=gen, device=DEV) for _ in range(3))
    empty = torch.zeros(ops.mask_words(k), dtype=torch.int32, device=DEV)
    out = []
    for mask in (None, empty):
        w, m, shadow = w0.clone() + 0.01, m0.clone(), torch.zeros(n, dtype=torch.bfloat16, device=DEV)
        opt = ops.FlatSGD(n, DEV, flat.LR, flat.MU, flat.MAX_NORM, flat.PGD_CLIP[pgd], n_pgd=k)
        opt.step(w, g * 30.0, m, w0=w0 if pgd != "off" else None, w_bf16=shadow, w_in=w0 if first else None, grad_mask=mask)
        out.append((w, m, shadow, opt.norms.clone()))
    for a, b in zip(*out):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


@pytest.mark.parametrize("gamma", [0.5, 8.0, 100.0])
def test_boost_update_matches_the_statement_bitwise(gamma):
    n = 3 * _sms() * 8 * 256 * 4 + 68
    nv = n - 36
    gen = torch.Generator(device=DEV).manual_seed(int(gamma * 10))
    w_g = torch.randn(n, generator=gen, device=DEV)
    slot = w_g + 1e-2 * torch.randn(n, generator=gen, device=DEV)
    slot[:100] = w_g[:100]                                          # zero updates stay zero
    before = slot.clone()
    ops.boost_update(slot, w_g, gamma, nv)
    ref = ops.boost_statement(before.cpu(), w_g.cpu(), gamma, nv)
    assert np.array_equal(slot[:nv].cpu().numpy().view(np.uint32), ref.view(np.uint32))
    assert torch.equal(slot[nv:], before[nv:])


# ---- the native trainer and the engine ---------------------------------------------------------------------------------------------
def _resnet_run(**kw):
    from rlr_b200.engine import FLEngine
    ops.reset_fallbacks()
    args = make_args(data="cifar10", model="resnet18", num_agents=4, num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, synthetic=512,
                     synthetic_val=128, log_dir="", seed=3, robustLR_threshold=2, device=DEV, attack_neurotoxin=0.01, **kw)
    eng = FLEngine(args, verbose=False)
    assert eng.trainer.name == "native"
    nv = eng.layout.n_vote
    out = []
    for r in range(1, 3):
        w_start = eng.global_params().clone()
        chosen = eng.run_round(r)["chosen"]
        corrupt = eng.fused.slots[eng.fused.slot_owner(chosen.index(0))[1]].clone()
        eng.round_result()
        out.append((eng.global_params().clone(), eng.last_masked_coords, eng.attack_mask.clone(), w_start, corrupt))
    torch.cuda.synchronize()
    assert ops.fallback_calls() == {}
    eng.close()
    return out, nv


def test_native_trainer_masks_the_corrupt_agent_and_graphs_equal_eager():
    graphs, nv = _resnet_run()
    eager, _ = _resnet_run(no_graphs=True)
    assert graphs[0][1] == 0 and graphs[1][1] >= math.floor(0.01 * get_layout("resnet18").n_params)
    for (wa, ca, ma, sa, xa), (wb, cb, mb, sb, xb) in zip(graphs, eager):
        assert torch.equal(wa, wb) and ca == cb and torch.equal(ma, mb) and torch.equal(xa, xb)
    w_start, corrupt, mask = graphs[1][3], graphs[1][4], graphs[1][2]
    bits = ops.mask_bits(mask, nv)
    assert torch.equal(corrupt[:nv][bits].view(torch.int32), w_start[:nv][bits].view(torch.int32))
    assert not torch.equal(corrupt[:nv], w_start[:nv])


def test_resnet18_with_both_attacks_is_reproducible():
    a, _ = _resnet_run(attack_boost=8.0)
    b, _ = _resnet_run(attack_boost=8.0)
    for (wa, ca, ma, _, xa), (wb, cb, mb, _, xb) in zip(a, b):
        assert torch.equal(wa, wb) and ca == cb and torch.equal(ma, mb) and torch.equal(xa, xb)
    w_start, corrupt, mask = a[1][3], a[1][4], a[1][2]
    bits = ops.mask_bits(mask, get_layout("resnet18").n_vote)
    assert bool((corrupt[:bits.numel()][bits] == w_start[:bits.numel()][bits]).all())       # 0 * boost = 0 on the mask


# ---- two or more GPUs: the fused hand-off ----------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _multi_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200.engine import FLEngine
    eng = FLEngine(make_args(data="cifar10", model="cnn_cifar", synthetic=128 * 2 * world, synthetic_val=128, num_agents=2 * world,
                             num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, log_dir="", seed=7, robustLR_threshold=2,
                             attack_neurotoxin=0.01, attack_boost=4.0), verbose=False)
    counts = []
    for r in range(1, 4):
        eng.run_round(r)
        eng.round_result()
        counts.append(eng.last_masked_coords)
    torch.save({"w": eng.global_params().clone().cpu(), "counts": counts, "mask": eng.attack_mask.cpu(), "handoff": eng.handoff,
                "backend": eng.fused.backend}, os.path.join(outdir, f"r{rank}.pt"))
    eng.close()
    dist.barrier(); dist.destroy_process_group()


def test_fused_handoff_ranks_agree_on_the_mask(tmp_path):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_multi_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"r{r}.pt") for r in range(world)]
    assert res[0]["backend"] == "fused" and res[0]["handoff"]
    assert res[0]["counts"][0] == 0 and res[0]["counts"][1] > 0
    for r in res[1:]:
        assert r["counts"] == res[0]["counts"] and torch.equal(r["w"], res[0]["w"]) and torch.equal(r["mask"], res[0]["mask"])
