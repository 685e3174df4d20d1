"""GPU: attack schedules (``ops.swap_samples`` in ops/csrc/attack.cu, and the engine's toggles on the native trainer).

* the swap kernel bitwise against the torch-indexing statement for uint8 [N,28,28,1] and [N,32,32,3], fp32 [N,28,28,1], a 12-byte
  fp32 row and a 75-byte uint8 row (the 16-, 4- and 1-byte word paths), N from 1 to several hundred thousand; two swaps are the
  identity, and an empty index changes nothing;
* the native trainer on ResNet-18 under a schedule that toggles several times: graph replay equal to ``--no_graphs``, a quiet-round
  corrupt slot equal to the clean run's slot, a full-window run equal to the default one, no library fall-through;
* the fused multi-GPU path: the ranks agree across toggles (skipped below two GPUs)."""
import os
import socket
import sys

import pytest
import torch
import torch.multiprocessing as mp

import rlr_b200  # noqa: F401
from rlr_b200 import ops
from rlr_b200.options import make_args

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHAPES = {"fmnist": ((28, 28, 1), torch.uint8), "cifar10": ((32, 32, 3), torch.uint8), "fedemnist": ((28, 28, 1), torch.float32),
          "row12": ((3,), torch.float32), "row75": ((5, 5, 3), torch.uint8)}


def _data(n, shape, dtype, gen):
    if dtype == torch.uint8:
        return torch.randint(0, 256, (n, *shape), generator=gen, device=DEV, dtype=torch.uint8)
    return torch.randn((n, *shape), generator=gen, device=DEV)


def _statement(data, targets, idx, side, side_t):
    x, y = data[idx].clone(), targets[idx].clone()
    data[idx] = side
    targets[idx] = side_t
    side.copy_(x)
    side_t.copy_(y)


@pytest.mark.parametrize("k", [1, 37, 4096, 300_000])
@pytest.mark.parametrize("kind", list(SHAPES))
def test_swap_kernel_matches_the_statement(kind, k):
    shape, dtype = SHAPES[kind]
    n = k + k // 3 + 5
    gen = torch.Generator(device=DEV).manual_seed(k + len(kind))
    data, targets = _data(n, shape, dtype, gen), torch.randint(0, 10, (n,), generator=gen, device=DEV)
    idx = torch.randperm(n, generator=gen, device=DEV)[:k].contiguous()
    side, side_t = _data(k, shape, dtype, gen), torch.randint(100, 110, (k,), generator=gen, device=DEV)
    d0, t0, s0, st0 = data.clone(), targets.clone(), side.clone(), side_t.clone()
    ref = [d0.clone(), t0.clone(), s0.clone(), st0.clone()]
    _statement(ref[0], ref[1], idx, ref[2], ref[3])
    ops.swap_samples(data, targets, idx, side, side_t)
    torch.cuda.synchronize()
    for got, want in zip((data, targets, side, side_t), ref):
        assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))
    ops.swap_samples(data, targets, idx, side, side_t)                    # a swap is its own inverse
    for got, want in zip((data, targets, side, side_t), (d0, t0, s0, st0)):
        assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))


def test_an_empty_swap_changes_nothing():
    data, targets = torch.zeros(10, 28, 28, 1, dtype=torch.uint8, device=DEV), torch.zeros(10, dtype=torch.int64, device=DEV)
    ops.swap_samples(data, targets, torch.zeros(0, dtype=torch.int64, device=DEV), data[:0].clone(), targets[:0].clone())
    torch.cuda.synchronize()
    assert not bool(data.any()) and not bool(targets.any())


# ---- the native trainer and the engine ---------------------------------------------------------------------------------------------
def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="cifar10", model="resnet18", num_agents=4, num_corrupt=1, poison_frac=0.5, local_ep=1, bs=64, synthetic=512,
                synthetic_val=128, log_dir="", seed=3, robustLR_threshold=2, device=DEV)
    base.update(kw)
    eng = FLEngine(make_args(**base), verbose=False)
    assert eng.trainer.name == "native"
    return eng


def _corrupt_slot(eng, chosen):
    return eng.fused.slots[eng.fused.slot_owner(chosen.index(0))[1]].clone()


def _run(rounds=5, **kw):
    """Rounds 1, 3, 5 attack, 2 and 4 quiet: every round from 2 on toggles the data."""
    ops.reset_fallbacks()
    eng = _engine(attack_every=2, attack_boost=4.0, attack_neurotoxin=0.01, **kw)
    out = []
    for r in range(1, rounds + 1):
        chosen = eng.run_round(r)["chosen"]
        eng.round_result()
        out.append((eng.global_params().clone(), _corrupt_slot(eng, chosen), eng.last_masked_coords,
                    eng.train_dataset.data.clone()))
    torch.cuda.synchronize()
    assert ops.fallback_calls() == {}
    eng.close()
    return out


def test_graph_replay_equals_eager_across_toggles():
    graphs, eager = _run(), _run(no_graphs=True)
    for r, ((wa, sa, ca, da), (wb, sb, cb, db)) in enumerate(zip(graphs, eager), 1):
        assert torch.equal(wa, wb) and torch.equal(sa, sb) and ca == cb and torch.equal(da, db), r
    assert [c for _, _, c, _ in graphs][1::2] == [0, 0]                  # quiet rounds: no mask
    assert graphs[2][2] > 0
    assert torch.equal(graphs[0][3], graphs[2][3]) and torch.equal(graphs[1][3], graphs[3][3])
    assert not torch.equal(graphs[0][3], graphs[1][3])


def test_a_quiet_corrupt_slot_equals_the_clean_run():
    ops.reset_fallbacks()
    eng = _engine(attack_every=2, attack_boost=4.0, attack_neurotoxin=0.01)
    clean = _engine(poison_frac=0.0)
    eng.run_round(1)
    for r in (2, 3, 4):
        clean.fused.w_global.copy_(eng.global_params())
        if clean.fused.w_bf16 is not None:
            clean.fused.w_bf16.copy_(eng.fused.w_bf16)
        chosen = eng.run_round(r)["chosen"]
        assert clean.run_round(r)["chosen"] == chosen
        torch.cuda.synchronize()
        if r % 2 == 0:
            assert torch.equal(_corrupt_slot(eng, chosen).view(torch.int32), _corrupt_slot(clean, chosen).view(torch.int32))
            assert torch.equal(eng.train_dataset.data, clean.train_dataset.data)
            assert torch.equal(eng.train_dataset.targets, clean.train_dataset.targets)
        else:
            assert not torch.equal(_corrupt_slot(eng, chosen), _corrupt_slot(clean, chosen))
    assert ops.fallback_calls() == {}
    eng.close(); clean.close()


def test_a_full_window_resnet18_run_equals_the_default_one():
    kw = dict(attack_boost=4.0, attack_neurotoxin=0.01)
    a, b = _engine(**kw), _engine(attack_stop=1000, **kw)
    for r in range(1, 4):
        a.run_round(r); b.run_round(r)
        a.round_result(); b.round_result()
        assert a.last_masked_coords == b.last_masked_coords
    assert torch.equal(a.global_params(), b.global_params())
    a.close(); b.close()


# ---- two or more GPUs: the fused hand-off ----------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _multi_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200.engine import FLEngine
    eng = FLEngine(make_args(data="cifar10", model="cnn_cifar", synthetic=128 * 2 * world, synthetic_val=128, num_agents=2 * world,
                             num_corrupt=2, poison_frac=0.5, local_ep=1, bs=64, log_dir="", seed=7, robustLR_threshold=2,
                             attack_every=2, attack_neurotoxin=0.01, attack_boost=4.0), verbose=False)
    out = []
    for r in range(1, 5):
        eng.run_round(r)
        eng.round_result()
        out.append((eng.global_params().clone().cpu(), eng.train_dataset.data.cpu(), eng.train_dataset.targets.cpu(),
                    eng.last_masked_coords))
    torch.save({"rounds": out, "handoff": eng.handoff, "backend": eng.fused.backend}, os.path.join(outdir, f"r{rank}.pt"))
    eng.close()
    dist.barrier(); dist.destroy_process_group()


def test_fused_ranks_agree_across_toggles(tmp_path):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    mp.spawn(_multi_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"r{r}.pt") for r in range(world)]
    assert res[0]["backend"] == "fused"
    for other in res[1:]:
        for a, b in zip(res[0]["rounds"], other["rounds"]):
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) and a[3] == b[3]
