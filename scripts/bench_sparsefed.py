"""Cost of SparseFed (``--server_topk``) on one GPU.

    python scripts/bench_sparsefed.py [--iters 50] [--rounds 10] [--skip 3] [--reps 2] [--out FILE]

1. The SparseFed pass alone (``ops.sparsefed_step``: accumulate + first histogram, two more histogram passes, three one-CTA bin
   searches, apply, finish) at the ResNet-18 size for k = 1 % and 10 % of the parameters, CUDA events around ``--iters`` launches after
   warm-up.  The pass updates the parameters and the error vector in place; every launch still reads and writes the same bytes.
   Bytes per voted coordinate: 16 accumulate (w', w, e read, e written), 4 + 4 for the two later histogram passes, 10 apply (e, w read,
   bf16 shadow written), plus 8 per applied coordinate (w, e written); 10 per BatchNorm-tail coordinate (w' read, w and shadow written).
2. Engine: ms per round (device-timed local-training and aggregation phases) and the ``aggregate`` phase alone, for CIFAR-10 ResNet-18
   with 8 agents, without and with ``--server_topk 0.01``, alternated.  The first ``--skip`` rounds of each run (graph capture) are
   not counted.

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

CONFIGS = {"plain": {}, "topk_0.01": {"server_topk": 0.01}}


def pass_bytes(n, nv, applied):
    return 34 * nv + 8 * applied + 10 * (n - nv)


def bench_pass(iters):
    import torch
    from rlr_b200 import ops
    from rlr_b200.models import get_layout
    lay = get_layout("resnet18")
    n, nv = lay.n_total, lay.n_vote
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    out = {"n_total": n, "n_vote": nv}
    for p in (0.01, 0.1):
        k = math.floor(p * lay.n_params)
        w = torch.randn(n, generator=gen, device=dev)
        wn = w + 1e-3 * torch.randn(n, generator=gen, device=dev)
        wb = w.to(torch.bfloat16)
        e = torch.zeros(nv, device=dev)
        stats = torch.zeros(3, dtype=torch.float64, device=dev)
        t = time_ms(lambda: ops.sparsefed_step(w, wn, e, nv, k, stats, wb), iters)
        applied = int(stats[0])
        b = pass_bytes(n, nv, applied)
        out[f"k_{p}"] = dict(k=k, applied_last=applied, ms=round(t, 4), bytes=b, GBps=round(b / t / 1e6, 1),
                             hbm_floor_ms=round(b / 3.35e12 * 1e3, 4))
    return out


def _engine(rounds, **kw):
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    args = make_args(data="cifar10", model="resnet18", num_agents=8, local_ep=1, bs=256, synthetic=8 * 1024, synthetic_val=256,
                     log_dir="", device="cuda:0", rounds=rounds, snap=10 ** 6, **kw)
    return FLEngine(args, verbose=False)


def bench_engine(rounds, reps, skip):
    import torch
    res = {c: {"round": [], "aggregate": []} for c in CONFIGS}
    for _ in range(reps):
        for name, kw in CONFIGS.items():
            eng = _engine(rounds, **kw)
            for r in range(1, rounds + 1):
                eng.run_round(r)
                torch.cuda.synchronize()
                el = eng.timer.elapsed()
                if r > skip:
                    res[name]["round"].append(el["local_train"] + el["aggregate"])
                    res[name]["aggregate"].append(el["aggregate"])
            eng.close()
            del eng
            torch.cuda.empty_cache()
    stat = lambda v: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3), rounds=len(v))
    return {c: {k: stat(v) for k, v in d.items()} for c, d in res.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=50)
    p.add_argument("--rounds", type=int, default=10, help="engine rounds per run")
    p.add_argument("--skip", type=int, default=3, help="leading rounds of each run not counted (graph capture)")
    p.add_argument("--reps", type=int, default=2, help="alternations of the two engine configurations")
    p.add_argument("--out", type=str, default="", help="also write the JSON result here")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_sparsefed.py needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    kern = bench_pass(a.iters)
    print(json.dumps({"pass": kern}))
    eng = bench_engine(a.rounds, a.reps, a.skip) if a.rounds > a.skip else {}
    print(json.dumps({"engine": eng}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"card": info, "pass": kern, "engine": eng}, fh, indent=1)


if __name__ == "__main__":
    main()
