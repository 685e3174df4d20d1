"""Cost of FLAME aggregation (``--aggr flame``) on one GPU.

    python scripts/bench_flame.py [--ks 8,10,40,64,200] [--iters 20] [--rounds 5] [--reps 2] [--out FILE]

1. Kernel: one Gram pass (``pairwise_sqdist_kernel<true>``) over the ResNet-18 voted coordinates (``n_vote``) for each K, next to the
   Krum distance pass (``pairwise_sqdist_kernel<false>``, no clip scales) over the same K vectors and ``fused_aggregate_kernel`` (avg, the
   engine's single-GPU launch with its bf16 shadow) -- the aggregate kernel is the memory yardstick.  CUDA events around ``--iters``
   launches after warm-up; the Gram pass is timed again after the others to show the spread.  Bytes are computed from the shapes: the
   distance pass reads each participant's n_vote fp32 values once per tile, 4 * K * n_vote bytes with K <= 64, and the Gram pass also
   reads w_global, 4 * n_vote more.  A round of ``--aggr flame`` runs one Gram pass before the aggregate.
2. Engine: ms per round (local training + aggregation, device-timed phases) and ``ms_aggregate`` of CIFAR-10 ResNet-18 with 8 agents,
   ``--aggr avg`` against ``--aggr flame``, alternated; the first round of each run is not counted.

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


def bench_kernels(ks, iters):
    import torch
    from rlr_b200 import ops
    from rlr_b200.models import get_layout
    lay = get_layout("resnet18")
    n, nv = lay.n_total, lay.n_vote
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    g = torch.randn(n, generator=gen, device=dev)
    pool = [g + 0.01 * torch.randn(n, generator=gen, device=dev) for _ in range(max(ks))]
    out = torch.empty(n, device=dev)
    out_b = torch.empty(n, dtype=torch.bfloat16, device=dev)
    outs, outs_b = ops.PtrTable([out.data_ptr()], dev), ops.PtrTable([out_b.data_ptr()], dev)
    rows = []
    for K in ks:
        ws = pool[:K]
        tab = ops.PtrTable([w.data_ptr() for w in ws], dev)
        G = torch.empty(K, K, dtype=torch.float64, device=dev)
        wt = torch.full((K,), 1.0, dtype=torch.float64, device=dev)
        gram = lambda: ops.ext().pairwise_gram(tab.tensor, g.data_ptr(), 0, nv, G, None, None, 0, 1, 0)
        dist = lambda: ops.ext().pairwise_sqdist(tab.tensor, 0, None, 0, nv, G, None, None, 0, 1, 0)
        agg = lambda: ops.ext().fused_aggregate(tab.tensor, wt, None, float(K), g.data_ptr(), outs.tensor, outs_b.tensor, False, 0, n,
                                                nv, 0, 0, 1.0, 0.0, 0, 0, None, None, None, 0, 1, 0, False, *ops.opt_launch_args(None))
        t_g, t_d, t_a = time_ms(gram, iters), time_ms(dist, iters), time_ms(agg, iters)
        t_g2 = time_ms(gram, iters)                         # again after the others: the spread of the measurement
        bytes_d = 4 * K * nv
        bytes_g = bytes_d + 4 * nv
        bytes_a = 4 * K * n + 4 * n + 4 * n + 2 * n
        best = min(t_g, t_g2)
        rows.append(dict(K=K, n_vote=nv, gram_ms=round(best, 4), gram_ms_repeat=round(max(t_g, t_g2), 4), sqdist_ms=round(t_d, 4),
                         agg_ms=round(t_a, 4), gram_over_sqdist=round(best / t_d, 3), gram_over_agg=round(best / t_a, 3),
                         gram_GBps=round(bytes_g / best / 1e6, 1), sqdist_GBps=round(bytes_d / t_d / 1e6, 1),
                         agg_GBps=round(bytes_a / t_a / 1e6, 1), hbm_floor_ms=round(bytes_g / 3.35e12 * 1e3, 4)))
        del tab, G
    return rows


def bench_engine(rounds, reps):
    import torch
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    res = {a: {"round": [], "aggregate": []} for a in ("avg", "flame")}
    for _ in range(reps):
        for aggr in ("avg", "flame"):
            args = make_args(data="cifar10", model="resnet18", num_agents=8, num_corrupt=1, poison_frac=0.5, local_ep=1, bs=256,
                             synthetic=8 * 1024, synthetic_val=256, log_dir="", device="cuda:0", aggr=aggr, rounds=rounds, snap=10 ** 6)
            eng = FLEngine(args, verbose=False)
            for r in range(1, rounds + 1):
                eng.run_round(r)
                torch.cuda.synchronize()
                el = eng.timer.elapsed()
                if r > 1:                                    # the first round captures the CUDA graphs
                    res[aggr]["round"].append(el["local_train"] + el["aggregate"])
                    res[aggr]["aggregate"].append(el["aggregate"])
            eng.close()
            del eng
            torch.cuda.empty_cache()
    stat = lambda v: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3), rounds=len(v))
    return {a: {k: stat(v) for k, v in d.items()} for a, d in res.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--ks", type=str, default="8,10,40,64,200")
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--rounds", type=int, default=5, help="engine rounds per run (the first is not counted)")
    p.add_argument("--reps", type=int, default=2, help="alternations of the avg / flame engine runs")
    p.add_argument("--out", type=str, default="", help="also write the JSON result here")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_flame.py needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    rows = bench_kernels([int(k) for k in a.ks.split(",")], a.iters)
    for r in rows:
        print(json.dumps(r))
    eng = bench_engine(a.rounds, a.reps) if a.rounds > 1 else {}
    print(json.dumps({"engine": eng}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"card": info, "kernels": rows, "engine": eng}, fh, indent=1)


if __name__ == "__main__":
    main()
