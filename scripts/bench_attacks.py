"""Cost of the model-poisoning attackers (``--attack_boost``, ``--attack_neurotoxin``) on one GPU.

    python scripts/bench_attacks.py [--iters 20] [--rounds 12] [--skip 4] [--reps 2] [--out FILE]

1. Kernels at the ResNet-18 voted coordinates (``n_vote``), CUDA events around ``--iters`` launches after warm-up:
   - Neurotoxin's mask pass (three histogram passes, three one-CTA bin searches, the mask build with the ``w_prev`` refresh) at
     k = 1 % of the parameters.  The pass overwrites ``w_prev``, so every timed launch is preceded by a copy that restores it; that copy
     is timed on its own and subtracted.  Bytes: 8 per coordinate per histogram pass, 12 for the mask build, plus the mask words.
   - The boost pass: 12 bytes per coordinate (slot and w_g read, slot written).
2. One local step of CIFAR-10 ResNet-18 (batch 256, native trainer), graph replay: the corrupt agent's masked step against an honest
   agent's unmasked one, alternated; both include the reset of the batch cursor that precedes every replay.
3. Engine: ms per round (local training + aggregation, device-timed phases) of CIFAR-10 ResNet-18 with 8 agents, 2 of them corrupt,
   without an attack, with ``--attack_boost 8``, with ``--attack_neurotoxin 0.01`` and with both, alternated.  The first ``--skip``
   rounds of each run are not counted: the trainers capture their CUDA graphs there, and with Neurotoxin a trainer captures the masked
   step graphs in the first round in which it hosts a corrupt agent, which need not be round 2.

The card's name, power limit and maximum SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_select import card, time_ms  # noqa: E402

CONFIGS = {"none": {}, "boost": {"attack_boost": 8.0}, "neurotoxin": {"attack_neurotoxin": 0.01},
           "both": {"attack_boost": 8.0, "attack_neurotoxin": 0.01}}


def bench_kernels(iters):
    import torch
    from rlr_b200 import ops
    from rlr_b200.models import get_layout
    lay = get_layout("resnet18")
    nv, k = lay.n_vote, math.floor(0.01 * lay.n_params)
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    prev = torch.randn(nv, generator=gen, device=dev)
    w_g = prev + 1e-3 * torch.randn(nv, generator=gen, device=dev)
    wp = prev.clone()
    mask = torch.zeros(ops.mask_words(nv), dtype=torch.int32, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    restore = lambda: wp.copy_(prev)
    t_copy = time_ms(restore, iters)
    t_both = time_ms(lambda: (restore(), ops.neurotoxin_mask(w_g, wp, nv, k, mask, count)), iters)
    t_copy2 = time_ms(restore, iters)
    t_mask = t_both - min(t_copy, t_copy2)
    bytes_mask = 3 * 8 * nv + 12 * nv + 4 * ops.mask_words(nv)
    slot = w_g + 1e-3 * torch.randn(nv, generator=gen, device=dev)
    t_boost = time_ms(lambda: ops.boost_update(slot, w_g, 1.0 + 1e-7, nv), iters)
    bytes_boost = 12 * nv
    return dict(n_vote=nv, k=k, masked=int(count), mask_ms=round(t_mask, 4), restore_copy_ms=round(min(t_copy, t_copy2), 4),
                mask_TBps=round(bytes_mask / t_mask / 1e9, 3), mask_bytes=bytes_mask, mask_hbm_floor_ms=round(bytes_mask / 3.35e12 * 1e3, 4),
                boost_ms=round(t_boost, 4), boost_TBps=round(bytes_boost / t_boost / 1e9, 3),
                boost_hbm_floor_ms=round(bytes_boost / 3.35e12 * 1e3, 4))


def _engine(rounds, **kw):
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    args = make_args(data="cifar10", model="resnet18", num_agents=8, num_corrupt=2, poison_frac=0.5, local_ep=1, bs=256,
                     synthetic=8 * 1024, synthetic_val=256, log_dir="", device="cuda:0", rounds=rounds, snap=10 ** 6, **kw)
    return FLEngine(args, verbose=False)


def bench_step(iters):
    """Replay the captured full-batch step of an honest agent and of a corrupt (masked) one, alternated."""
    import torch
    eng = _engine(2, attack_neurotoxin=0.01)
    for r in (1, 2):                                     # round 2 captures the corrupt agents' masked graphs
        eng.run_round(r)
    torch.cuda.synchronize()
    full = [(tr, key, g) for tr in eng.trainers for key, g in tr._graphs.items() if key[0] == tr.bs and not key[3]]
    masked = [(tr, g) for tr, key, g in full if key[4]]
    plain = [(tr, g) for tr, key, g in full if not key[4]]
    assert masked and plain, "both step graphs are captured"

    def step(tr, g):
        # each replay advances the trainer's batch cursor: reset it so every replay reads the first batch of the shard
        return lambda: (tr.cursor.zero_(), g.replay())
    ts = {"masked": [], "unmasked": []}
    for _ in range(3):
        ts["unmasked"].append(time_ms(step(*plain[0]), iters))
        ts["masked"].append(time_ms(step(*masked[0]), iters))
    eng.close()
    return {k: dict(median_ms=round(statistics.median(v), 4), min_ms=round(min(v), 4), max_ms=round(max(v), 4)) for k, v in ts.items()}


def bench_engine(rounds, reps, skip):
    import torch
    res = {c: {"round": [], "local_train": []} for c in CONFIGS}
    for _ in range(reps):
        for name, kw in CONFIGS.items():
            eng = _engine(rounds, **kw)
            for r in range(1, rounds + 1):
                eng.run_round(r)
                torch.cuda.synchronize()
                el = eng.timer.elapsed()
                if r > skip:
                    res[name]["round"].append(el["local_train"] + el["aggregate"])
                    res[name]["local_train"].append(el["local_train"])
            eng.close()
            del eng
            torch.cuda.empty_cache()
    stat = lambda v: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3), rounds=len(v))
    return {c: {k: stat(v) for k, v in d.items()} for c, d in res.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--rounds", type=int, default=12, help="engine rounds per run")
    p.add_argument("--skip", type=int, default=4, help="leading rounds of each run not counted (graph capture)")
    p.add_argument("--reps", type=int, default=2, help="alternations of the four engine configurations")
    p.add_argument("--out", type=str, default="", help="also write the JSON result here")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_attacks.py needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    kern = bench_kernels(a.iters)
    print(json.dumps({"kernels": kern}))
    step = bench_step(a.iters)
    print(json.dumps({"step": step}))
    eng = bench_engine(a.rounds, a.reps, a.skip) if a.rounds > a.skip else {}
    print(json.dumps({"engine": eng}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"card": info, "kernels": kern, "step": step, "engine": eng}, fh, indent=1)


if __name__ == "__main__":
    main()
