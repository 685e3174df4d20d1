"""Cost of attack schedules (``--attack_start / --attack_stop / --attack_every``) on one GPU.

    python scripts/bench_attack_schedule.py [--iters 200] [--rounds 12] [--skip 4] [--reps 2] [--out FILE]

1. The swap that toggles a poisoned dataset between its poisoned and its clean samples (``ops.swap_samples``, one launch), CUDA events
   around ``--iters`` launches after warm-up, on random distinct indices:
   - the CIFAR-10 runner config: 4 corrupt agents of 40 with ``--poison_frac 0.5`` poison 4 x floor(0.5 x 125) = 248 rows of 3072 B
     in the 50,000-image uint8 set;
   - Fed-EMNIST-sized sets: 338 corrupt clients of the 341,873-image fp32 set (3136 B rows) at 5 and 10 poisoned samples per client;
   - a 10x larger synthetic set: 2,480 rows of 3072 B in a 500,000-image uint8 set.
   Bytes: each row and label is read and written on both sides (4 x row + 32 B per row) plus the 8-byte index.
2. Engine: ms per round (local training + aggregation, device-timed phases) of CIFAR-10 ResNet-18 with 8 agents, 2 of them corrupt,
   ``--poison_frac 0.5``, without a schedule and under three schedules, alternated: every round an attack round (``--attack_stop``
   beyond the run), no round an attack round (``--attack_start`` beyond the run) and attack rounds every other round
   (``--attack_every 2``, so every round toggles).  The rounds under a schedule are pooled and split into attack rounds without a
   toggle, quiet rounds without a toggle, and toggle rounds.  The first ``--skip`` rounds of each run are not counted (graph capture).

The card's name, power limit and maximum SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_select import card, time_ms  # noqa: E402

# name: (dataset rows, row shape, dtype, poisoned rows)
SWAPS = {
    "cifar10_runner": (50_000, (32, 32, 3), "uint8", 248),
    "fedemnist_5_per_client": (341_873, (28, 28, 1), "float32", 338 * 5),
    "fedemnist_10_per_client": (341_873, (28, 28, 1), "float32", 338 * 10),
    "synthetic_10x_cifar10": (500_000, (32, 32, 3), "uint8", 2_480),
}
CONFIGS = {"none": {}, "all_attack": {"attack_stop": 10 ** 6}, "all_quiet": {"attack_start": 10 ** 6},
           "every_2": {"attack_every": 2}}


def bench_swaps(iters):
    import torch
    from rlr_b200 import ops
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    out = {}
    for name, (n, shape, dt, k) in SWAPS.items():
        dtype = getattr(torch, dt)
        data = (torch.randint(0, 256, (n, *shape), generator=gen, device=dev, dtype=torch.uint8) if dtype == torch.uint8
                else torch.rand((n, *shape), generator=gen, device=dev))
        targets = torch.randint(0, 10, (n,), generator=gen, device=dev)
        idx = torch.randperm(n, generator=gen, device=dev)[:k].contiguous()
        side, side_t = data[idx].clone(), targets[idx].clone()
        row = data[0].numel() * data.element_size()
        t = time_ms(lambda: ops.swap_samples(data, targets, idx, side, side_t), iters)
        moved = k * (4 * row + 32 + 8)
        out[name] = dict(rows=k, row_bytes=row, poisoned_bytes=k * row, bytes_moved=moved, swap_us=round(t * 1e3, 2),
                         GBps=round(moved / t / 1e6, 1), hbm_floor_us=round(moved / 3.35e12 * 1e6, 3))
        del data, targets, side, side_t
    torch.cuda.empty_cache()
    return out


def _engine(rounds, **kw):
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    args = make_args(data="cifar10", model="resnet18", num_agents=8, num_corrupt=2, poison_frac=0.5, local_ep=1, bs=256,
                     synthetic=8 * 1024, synthetic_val=256, log_dir="", device="cuda:0", rounds=rounds, snap=10 ** 6, **kw)
    return FLEngine(args, verbose=False)


def bench_engine(rounds, reps, skip):
    import torch
    res = {"none": [], "attack": [], "quiet": [], "toggle": []}
    for _ in range(reps):
        for name, kw in CONFIGS.items():
            eng = _engine(rounds, **kw)
            for r in range(1, rounds + 1):
                before = eng._data_poisoned
                eng.run_round(r)
                torch.cuda.synchronize()
                el = eng.timer.elapsed()
                if r <= skip:
                    continue
                kind = ("none" if name == "none" else "toggle" if eng._data_poisoned != before else
                        "attack" if eng.last_attack_active else "quiet")
                res[kind].append(el["local_train"] + el["aggregate"])
            eng.close()
            del eng
            torch.cuda.empty_cache()
    stat = lambda v: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3), rounds=len(v))
    return {k: stat(v) for k, v in res.items() if v}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=200)
    p.add_argument("--rounds", type=int, default=12, help="engine rounds per run")
    p.add_argument("--skip", type=int, default=4, help="leading rounds of each run not counted (graph capture)")
    p.add_argument("--reps", type=int, default=2, help="alternations of the four engine configurations")
    p.add_argument("--out", type=str, default="", help="also write the JSON result here")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_attack_schedule.py needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    swaps = bench_swaps(a.iters)
    print(json.dumps({"swaps": swaps}))
    eng = bench_engine(a.rounds, a.reps, a.skip) if a.rounds > a.skip else {}
    print(json.dumps({"engine": eng}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"card": info, "swaps": swaps, "engine": eng}, fh, indent=1)


if __name__ == "__main__":
    main()
