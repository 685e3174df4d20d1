"""Attack schedules (``--attack_start / --attack_stop / --attack_every / --attack_force``) and the backdoor's lifespan on CPU: option
validation, the banner and the attack-round predicate; forced participation against a direct statement of the rule; the side copy of
the poisoned samples and the swap; bitwise equivalence of engine runs (defaults, a schedule covering every round, one covering none);
a quiet round against the clean run; Neurotoxin's mask after a quiet gap; resume; ``backdoor_lifespan`` on fabricated evaluations;
two gloo ranks; the logged fields of ``federated.py``; input streaming under a schedule."""
import json
import os
import random
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.data import poison_dataset
from rlr_b200.data.datasets import DeviceDataset
from rlr_b200.engine import force_participants
from rlr_b200.options import is_attack_round, last_attack_round, make_args, print_exp_details
from rlr_b200.utils import backdoor_lifespan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- options ------------------------------------------------------------------------------------------------------------------
def test_defaults_and_the_banner(capsys):
    a = make_args()
    assert (a.attack_start, a.attack_stop, a.attack_every, a.attack_force, a.lifespan_threshold) == (1, 0, 1, False, 0.5)
    print_exp_details(make_args(num_corrupt=1))
    assert "Attack schedule" not in capsys.readouterr().out
    print_exp_details(make_args(num_corrupt=1, attack_start=20, attack_stop=20, attack_force=True))
    assert "Attack schedule (start / stop / every / force): 20 / 20 / 1 / True" in capsys.readouterr().out
    print_exp_details(make_args(num_corrupt=1, attack_every=3))
    assert "Attack schedule (start / stop / every / force): 1 / 0 / 3 / False" in capsys.readouterr().out


@pytest.mark.parametrize("kw", [
    dict(attack_start=0), dict(attack_start=-3), dict(attack_stop=-1), dict(attack_start=5, attack_stop=4), dict(attack_every=0),
    dict(attack_every=-2), dict(attack_stop=5, lifespan_threshold=0.0), dict(attack_stop=5, lifespan_threshold=-0.1),
    dict(attack_stop=5, lifespan_threshold=1.5), dict(attack_stop=5, lifespan_threshold=float("nan")),
    dict(attack_stop=5, lifespan_threshold=float("inf")), dict(lifespan_threshold=0.3),
])
def test_rejects_invalid_schedules(kw):
    with pytest.raises(ValueError):
        make_args(num_corrupt=1, **kw)


@pytest.mark.parametrize("kw", [dict(attack_start=2), dict(attack_stop=3), dict(attack_every=2), dict(attack_force=True)])
def test_a_schedule_needs_corrupt_agents(kw):
    with pytest.raises(ValueError, match="num_corrupt"):
        make_args(num_corrupt=0, **kw)
    make_args(num_corrupt=1, **kw)


def test_accepted_edge_values():
    a = make_args(num_corrupt=1, attack_start=4, attack_stop=4, lifespan_threshold=1.0)
    assert (a.attack_start, a.attack_stop, a.lifespan_threshold) == (4, 4, 1.0)


# (start, stop, every) -> attack rounds among 1..12
SCHEDULES = [
    ((1, 0, 1), list(range(1, 13))),
    ((3, 0, 1), list(range(3, 13))),
    ((1, 5, 1), [1, 2, 3, 4, 5]),
    ((2, 9, 3), [2, 5, 8]),
    ((2, 10, 4), [2, 6, 10]),
    ((20, 20, 1), []),
    ((7, 7, 5), [7]),
    ((1, 0, 5), [1, 6, 11]),
    ((4, 11, 2), [4, 6, 8, 10]),
]


@pytest.mark.parametrize("sched,rounds", SCHEDULES)
def test_attack_round_predicate_against_a_table(sched, rounds):
    assert [r for r in range(1, 13) if is_attack_round(r, *sched)] == rounds
    last = last_attack_round(*sched)
    if sched[1] == 0:
        assert last is None
    else:
        expect = [r for r in range(1, sched[1] + 1) if is_attack_round(r, *sched)]
        assert last == expect[-1]


# ---- forced participation -------------------------------------------------------------------------------------------------------
def _force_statement(drawn, c):
    """The rule read literally: M = the corrupt ids not drawn, ascending; honest positions from the end receive them in turn."""
    m = sorted(set(range(c)) - set(drawn))
    honest_from_end = [p for p in reversed(range(len(drawn))) if drawn[p] >= c]
    out = list(drawn)
    for p, a in zip(honest_from_end, m):
        out[p] = a
    return out


def test_force_against_the_statement():
    rng = random.Random(0)
    for _ in range(500):
        n = rng.randint(1, 30)
        k = rng.randint(1, n)
        c = rng.randint(1, n)
        drawn = rng.sample(range(n), k)
        got = force_participants(drawn, c)
        assert got == _force_statement(drawn, c)
        assert len(set(got)) == len(got) == k
        assert sum(a < c for a in got) == min(c, k)


def test_force_edge_cases():
    assert force_participants([5, 0, 1, 7], 2) == [5, 0, 1, 7]             # every corrupt agent already drawn
    assert force_participants([9, 8, 7], 5) == [2, 1, 0]                    # K < num_corrupt: an all-corrupt round
    assert force_participants([3, 9, 0, 8], 3) == [3, 2, 0, 1]
    assert force_participants([3, 9, 0, 8], 2) == [3, 9, 0, 1]
    assert force_participants([3, 9, 8, 4], 3) == [3, 2, 1, 0]


def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="fmnist", synthetic=800, synthetic_val=200, num_agents=5, local_ep=1, bs=64, device="cpu", num_corrupt=1,
                poison_frac=0.5, robustLR_threshold=0, log_dir="", seed=5, trainer="torch")
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def test_forced_rounds_keep_the_draws_of_later_rounds():
    kw = dict(num_agents=10, agent_frac=0.3, num_corrupt=2, synthetic=1000)
    plain, forced = _engine(**kw), _engine(attack_start=2, attack_every=2, attack_force=True, **kw)
    for r in range(1, 7):
        draw = plain.sample_agents(r)
        assert forced.sample_agents(r) == draw
        chosen = forced.run_round(r)["chosen"]
        assert chosen == (force_participants(draw, 2) if r % 2 == 0 else draw)
        if r % 2 == 0:
            assert {0, 1} <= set(chosen)
    plain.close(); forced.close()


# ---- the side copy and the swap ---------------------------------------------------------------------------------------------------
def _fmnist(n=400, seed=0):
    g = torch.Generator().manual_seed(seed)
    return DeviceDataset("fmnist", torch.randint(0, 256, (n, 28, 28, 1), generator=g, dtype=torch.uint8),
                         torch.randint(0, 10, (n,), generator=g))


def test_side_copy_holds_the_clean_samples_and_draws_no_extra_randomness():
    args = make_args(data="fmnist", num_corrupt=1, poison_frac=0.5, pattern_type="square")
    a, b = _fmnist(), _fmnist()
    clean = _fmnist()
    side = []
    ra, rb = random.Random(3), random.Random(3)
    ia = poison_dataset(a, args, torch.arange(200), agent_idx=0, rng=ra)
    ib = poison_dataset(b, args, torch.arange(200), agent_idx=0, rng=rb, clean_copy=side)
    assert ia == ib and torch.equal(a.data, b.data) and torch.equal(a.targets, b.targets)
    assert ra.getstate() == rb.getstate()
    (sel, x, y), = side
    assert sel.tolist() == ib
    assert torch.equal(x, clean.data[sel]) and torch.equal(y, clean.targets[sel])
    assert not torch.equal(b.data[sel], clean.data[sel])
    ops.swap_samples(b.data, b.targets, sel, x, y)
    assert torch.equal(b.data, clean.data) and torch.equal(b.targets, clean.targets)
    ops.swap_samples(b.data, b.targets, sel, x, y)
    assert torch.equal(b.data, a.data) and torch.equal(b.targets, a.targets)


def test_cpu_swap_on_float_rows_and_an_empty_index():
    g = torch.Generator().manual_seed(1)
    data, tg = torch.randn(50, 28, 28, 1, generator=g), torch.arange(50)
    idx = torch.tensor([3, 17, 40])
    side, side_t = torch.randn(3, 28, 28, 1, generator=g), torch.tensor([-1, -2, -3])
    d0, t0, s0, st0 = data.clone(), tg.clone(), side.clone(), side_t.clone()
    ops.swap_samples(data, tg, idx, side, side_t)
    assert torch.equal(data[idx], s0) and torch.equal(side, d0[idx]) and torch.equal(tg[idx], st0) and torch.equal(side_t, t0[idx])
    ops.swap_samples(data, tg, torch.zeros(0, dtype=torch.int64), side[:0], side_t[:0])
    assert torch.equal(side, d0[idx])


# ---- engine runs ----------------------------------------------------------------------------------------------------------------
def _rounds(eng, n):
    for r in range(1, n + 1):
        eng.run_round(r)
    return eng.w_global.clone()


def test_defaults_are_the_plain_run_bit_for_bit():
    a = _engine(attack_boost=3.0)
    b = _engine(attack_boost=3.0, attack_start=1, attack_stop=0, attack_every=1, attack_force=False, lifespan_threshold=0.5)
    assert b.schedule is False and b._swaps == [] and all(ag.clean_copy is None for ag in b.agents)
    assert torch.equal(_rounds(a, 2), _rounds(b, 2))
    a.close(); b.close()


def test_a_schedule_covering_every_round_is_the_default_run():
    kw = dict(attack_boost=3.0, attack_neurotoxin=0.02, clip=1.0)
    a, b = _engine(**kw), _engine(attack_stop=50, attack_force=True, **kw)
    assert b.schedule and len(b._swaps) == 1
    for r in range(1, 4):
        ca, cb = a.run_round(r)["chosen"], b.run_round(r)["chosen"]
        assert ca == cb and b.last_attack_active
        a.round_result(); b.round_result()
        assert a.last_masked_coords == b.last_masked_coords
    assert torch.equal(a.w_global, b.w_global) and torch.equal(a.train_dataset.data, b.train_dataset.data)
    a.close(); b.close()


def test_a_schedule_covering_no_round_is_the_clean_run():
    clean = _engine(poison_frac=0.0)
    quiet = _engine(attack_start=10, attack_boost=5.0, attack_neurotoxin=0.02)
    assert torch.equal(_rounds(clean, 3), _rounds(quiet, 3))
    assert torch.equal(quiet.train_dataset.data, clean.train_dataset.data)
    assert torch.equal(quiet.train_dataset.targets, clean.train_dataset.targets)
    quiet.round_result()
    assert quiet.last_masked_coords == 0 and not quiet.last_attack_active
    clean.close(); quiet.close()


def test_a_quiet_round_is_an_honest_round():
    kw = dict(num_corrupt=2, attack_boost=4.0, attack_neurotoxin=0.02)
    eng = _engine(attack_stop=2, **kw)                                   # rounds 1-2 attack, 3-4 quiet
    clean = _engine(num_corrupt=2, poison_frac=0.0)
    poisoned = (eng.train_dataset.data.clone(), eng.train_dataset.targets.clone())
    _rounds(eng, 2)
    assert torch.equal(eng.train_dataset.data, poisoned[0])
    for r in (3, 4):
        w = eng.global_params().clone()
        clean.w_global.copy_(w)
        chosen = eng.run_round(r)["chosen"]
        assert clean.run_round(r)["chosen"] == chosen
        eng.round_result()
        assert not eng.last_attack_active and eng.last_masked_coords == 0
        assert torch.equal(eng.train_dataset.data, clean.train_dataset.data)
        assert torch.equal(eng.train_dataset.targets, clean.train_dataset.targets)
        for j, a in enumerate(chosen):
            s = eng.fused.slot_owner(j)[1]
            assert torch.equal(eng.fused.slots[s], clean.fused.slots[s]), a         # corrupt slots too: no mask, no boost
        assert torch.equal(eng.w_prev, w[:eng.layout.n_vote])
    eng.close(); clean.close()


def test_the_data_toggles_back_to_poisoned():
    eng = _engine(attack_start=1, attack_every=2)                        # attack rounds 1, 3, 5
    clean = _engine(poison_frac=0.0)
    poisoned = eng.train_dataset.data.clone(), eng.train_dataset.targets.clone()
    for r in range(1, 5):
        eng.run_round(r)
        ref = poisoned if r % 2 else (clean.train_dataset.data, clean.train_dataset.targets)
        assert torch.equal(eng.train_dataset.data, ref[0]) and torch.equal(eng.train_dataset.targets, ref[1]), r
    eng.close(); clean.close()


def test_neurotoxin_mask_after_a_quiet_gap():
    eng = _engine(attack_every=3, attack_neurotoxin=0.02)                # attack rounds 1, 4
    nv, k = eng.layout.n_vote, eng.neurotoxin_k
    for r in (1, 2):
        eng.run_round(r)
    w3 = eng.global_params().clone()
    eng.run_round(3)
    w4 = eng.global_params().clone()
    eng.run_round(4)
    eng.round_result()
    ref, count = ops.neurotoxin_statement(w4, w3, nv, k)
    assert np.array_equal(eng.attack_mask.numpy().view(np.uint32), ref) and eng.last_masked_coords == count >= k
    eng.close()


# ---- lifespan -------------------------------------------------------------------------------------------------------------------
def test_backdoor_lifespan_on_fabricated_evaluations():
    ev = [(r, a) for r, a in zip(range(1, 11), [.9, .95, .97, .96, .8, .6, .45, .3, .2, .1])]
    assert backdoor_lifespan(ev, 4, 0.5) == 3                           # round 7 is the first below 0.5
    assert backdoor_lifespan(ev, 4, 0.97) == 0                           # already below at the last attack round
    assert backdoor_lifespan(ev, 4, 0.05) is None                        # never reached
    assert backdoor_lifespan(ev, 2, 0.95) == 3                           # 0.95 at 2 is not below; 0.8 at 5 is
    assert backdoor_lifespan([(r, 0.1) for r in (1, 2)], 3, 0.5) is None                     # nothing evaluated after the attack
    assert backdoor_lifespan([(5, 0.5), (6, 0.49)], 5, 0.5) == 1         # equal to the threshold is not below it
    snap = [(r, a) for r, a in ev if r % 3 == 0]                          # --snap 3: rounds 3, 6, 9
    assert backdoor_lifespan(snap, 4, 0.5) == 5                          # 0.6 at 6, 0.2 at 9
    assert backdoor_lifespan(snap, 3, 0.98) == 0
    assert backdoor_lifespan([], 3, 0.5) is None


def test_resume_equals_the_uninterrupted_run(tmp_path):
    kw = dict(attack_stop=3, lifespan_threshold=1.0, attack_neurotoxin=0.02, attack_boost=3.0, clip=1.0, agent_frac=0.6,
              attack_force=True)
    full = _engine(rounds=6, **kw)
    hist = full.fit()
    assert [h["attack_active"] for h in hist] == [True, True, True, False, False, False]
    assert full.backdoor_lifespan is not None
    for stop in (2, 4):                                                  # inside the attack window, then inside the quiet span
        ck = str(tmp_path / f"ck{stop}.pt")
        first = _engine(rounds=stop, checkpoint=ck, **kw)
        first.fit()
        assert torch.load(ck, weights_only=False)["extra"]["backdoor_lifespan"] == first.backdoor_lifespan
        second = _engine(rounds=6, resume=ck, **kw)
        assert second.start_round == stop + 1
        h2 = second.fit()
        assert torch.equal(second.w_global, full.w_global) and torch.equal(second.w_prev, full.w_prev)
        assert torch.equal(second.train_dataset.data, full.train_dataset.data)
        assert second.backdoor_lifespan == full.backdoor_lifespan
        assert [h.get("backdoor_lifespan") for h in h2] == [h.get("backdoor_lifespan") for h in hist[stop:]]
        first.close(); second.close()
    full.close()


def test_resume_without_the_lifespan_is_an_error(tmp_path):
    ck = str(tmp_path / "ck.pt")
    plain = _engine(rounds=1, checkpoint=ck, attack_start=1, attack_every=2)
    plain.fit()
    assert "backdoor_lifespan" not in torch.load(ck, weights_only=False)["extra"]            # format unchanged without a stop round
    with pytest.raises(ValueError, match="lifespan"):
        _engine(rounds=3, resume=ck, attack_stop=2)
    plain.close()


def test_lifespan_not_reached_is_reported_at_least(capsys):
    from rlr_b200.engine import FLEngine
    eng = FLEngine(make_args(data="fmnist", synthetic=800, synthetic_val=200, num_agents=5, local_ep=1, bs=64, device="cpu",
                             num_corrupt=1, poison_frac=0.5, log_dir="", seed=5, trainer="torch", rounds=4, attack_stop=2,
                             snap=5), verbose=True)                       # no round is evaluated: the backdoor is never seen gone
    hist = eng.fit()
    assert eng.backdoor_lifespan is None and all("backdoor_lifespan" not in h for h in hist)
    assert hist[-1]["backdoor_lifespan_at_least"] == 2 and all("backdoor_lifespan_at_least" not in h for h in hist[:-1])
    assert "| Backdoor lifespan: > 2 rounds |" in capsys.readouterr().out
    eng.close()


# ---- two ranks ------------------------------------------------------------------------------------------------------------------
def _gloo_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args as mk
    eng = FLEngine(mk(data="fmnist", synthetic=800, synthetic_val=200, num_agents=4, local_ep=1, bs=64, device="cpu", num_corrupt=2,
                      poison_frac=0.5, log_dir="", seed=3, attack_start=2, attack_every=2, attack_neurotoxin=0.02, attack_boost=2.0),
                   verbose=False)
    out = []
    for r in range(1, 5):
        eng.run_round(r)
        eng.round_result()
        out.append((eng.train_dataset.data.clone(), eng.train_dataset.targets.clone(), eng.w_global.clone(), eng.last_masked_coords))
    torch.save(out, os.path.join(outdir, f"r{rank}.pt"))
    eng.close()
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_ranks_agree_on_the_toggled_data():
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_gloo_worker, args=(2, _free_port(), d), nprocs=2, join=True)
        outs = [torch.load(os.path.join(d, f"r{r}.pt")) for r in range(2)]
    for a, b in zip(*outs):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) and a[3] == b[3]
    assert not torch.equal(outs[0][0][0], outs[0][1][0])                 # round 1 quiet, round 2 attacked
    assert torch.equal(outs[0][0][0], outs[0][2][0]) and torch.equal(outs[0][1][0], outs[0][3][0])
    assert [o[3] for o in outs[0]][::2] == [0, 0]                        # quiet rounds: no mask


# ---- federated.py ---------------------------------------------------------------------------------------------------------------
def test_federated_py_writes_the_schedule_fields_and_tags(tmp_path):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "federated.py", "--data=fmnist", "--local_ep=1", "--bs=64", "--num_agents=4", "--rounds=3",
                        "--num_corrupt=1", "--poison_frac=0.5", "--synthetic=400", "--synthetic_val=80", "--attack_stop=1",
                        "--lifespan_threshold=1.0", f"--log_dir={tmp_path}", "--device=cpu"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "Attack schedule (start / stop / every / force): 1 / 1 / 1 / False" in r.stdout
    run_dirs = os.listdir(tmp_path)
    assert len(run_dirs) == 1
    recs = [json.loads(l) for l in open(tmp_path / run_dirs[0] / "metrics.jsonl")]
    assert [rec["attack_active"] for rec in recs] == [True, False, False]
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    acc = EventAccumulator(str(tmp_path / run_dirs[0]))
    acc.Reload()
    assert [(e.step, e.value) for e in acc.Scalars("Attack/Active")] == [(1, 1.0), (2, 0.0), (3, 0.0)]
    spans = [(rec["round"], rec["backdoor_lifespan"]) for rec in recs if "backdoor_lifespan" in rec]
    if spans:
        (rnd, span), = spans
        assert int(span) == span == rnd - 1 and f"| Backdoor lifespan: {int(span)} rounds |" in r.stdout
        assert [(e.step, e.value) for e in acc.Scalars("Poison/Lifespan")] == [(rnd, float(span))]
    else:                                                                # poison accuracy 1.0 in every round: not reached
        assert recs[-1]["backdoor_lifespan_at_least"] == 2 and "| Backdoor lifespan: > 2 rounds |" in r.stdout


def test_input_streaming_refuses_a_schedule():
    eng = _engine(attack_every=2)
    with pytest.raises(ValueError, match="schedule"):
        eng.enable_input_streaming()
    eng.close()
    plain = _engine()
    assert plain.enable_input_streaming() > 0
    plain.close()
