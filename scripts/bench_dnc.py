"""Cost of DnC selection (``--select dnc``) on one GPU.

    python scripts/bench_dnc.py [--ks 8,10,40,64] [--dims 10000,100000,0] [--iters 20] [--rounds 5] [--out FILE]

1. Kernels: the DnC pass -- one ``dnc_gather_kernel`` launch and one ``pairwise_sqdist_kernel<true, true>`` Gram launch over the
   gathered rows (T = 1) -- over the ResNet-18 voted coordinates (``n_vote``) for each K and subsample size b (0 = b = n_vote), next to
   ``fused_aggregate_kernel`` (avg, the engine's single-GPU launch with its bf16 shadow) over the same K vectors, the memory yardstick
   of a full pass over the participants.  CUDA events around ``--iters`` passes after warm-up; the subsample is drawn once, outside the
   timing (``ops.dnc_sample``'s host cost is timed on its own).
2. Engine: ``ms_aggregate`` (host-timed phase: the draw, the DnC pass, its device->host read of the Gram matrix, the host rule and the
   server step) of ``federated.py``-style rounds of CIFAR-10 ResNet-18 with 8 agents, ``--select none`` against ``--select dnc``,
   alternated.

The card's name, power limit and maximum SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_select import card, time_ms  # noqa: E402


def bench_kernels(ks, dims, iters):
    import numpy as np
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
    for b in dims:
        b = nv if b <= 0 else b
        t0 = time.perf_counter()
        sample = ops.dnc_sample(0, 1, 0, b, nv)
        draw_ms = (time.perf_counter() - t0) * 1e3
        samples = sample[None]
        for K in ks:
            ws = pool[:K]
            tab = ops.PtrTable([w.data_ptr() for w in ws], dev)
            G = torch.empty(1, K, K, dtype=torch.float64, device=dev)
            wt = torch.full((K,), 100.0, dtype=torch.float64, device=dev)
            dnc = lambda: ops.dnc_launch(tab.tensor, K, g.data_ptr(), samples, None, G, dev, 0, nv)
            agg = lambda: ops.ext().fused_aggregate(tab.tensor, wt, None, 100.0 * K, g.data_ptr(), outs.tensor, outs_b.tensor, False, 0,
                                                    n, nv, 0, 0, 1.0, 0.0, 0, 0, None, None, None, 0, 1, 0, False,
                                                    *ops.opt_launch_args(None))
            t_d, t_a = time_ms(dnc, iters), time_ms(agg, iters)
            t_d2 = time_ms(dnc, iters)                      # again after the aggregate: the spread of the measurement
            rows.append(dict(K=K, n_vote=nv, b=len(sample), draw_ms=round(draw_ms, 3), dnc_ms=round(min(t_d, t_d2), 4),
                             dnc_ms_repeat=round(max(t_d, t_d2), 4), agg_ms=round(t_a, 4), ratio=round(min(t_d, t_d2) / t_a, 4)))
            del tab, G
    return rows


def bench_engine(rounds, reps):
    import torch
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    res = {"none": [], "dnc": []}
    for rep in range(reps):
        for sel in ("none", "dnc"):
            args = make_args(data="cifar10", model="resnet18", num_agents=8, num_corrupt=1, poison_frac=0.5, local_ep=1, bs=256,
                             synthetic=8 * 1024, synthetic_val=256, log_dir="", device="cuda:0", select=sel, rounds=rounds, snap=10 ** 6)
            eng = FLEngine(args, verbose=False)
            for r in range(1, rounds + 1):
                eng.run_round(r)
                torch.cuda.synchronize()
                ms = eng.timer.elapsed()["aggregate"]
                if r > 1:
                    res[sel].append(ms)
            eng.close()
            del eng
            torch.cuda.empty_cache()
    return {k: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3), rounds=len(v))
            for k, v in res.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--ks", type=str, default="8,10,40,64")
    p.add_argument("--dims", type=str, default="10000,100000,0", help="subsample sizes b (0 = every voted coordinate)")
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--rounds", type=int, default=5, help="engine rounds per run (the first is not counted)")
    p.add_argument("--reps", type=int, default=2, help="alternations of the none / dnc engine runs")
    p.add_argument("--out", type=str, default="", help="also write the JSON result here")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_dnc.py needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    rows = bench_kernels([int(k) for k in a.ks.split(",")], [int(b) for b in a.dims.split(",")], a.iters)
    for r in rows:
        print(json.dumps(r))
    eng = bench_engine(a.rounds, a.reps) if a.rounds > 1 else {}
    print(json.dumps({"ms_aggregate": eng}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"card": info, "kernels": rows, "ms_aggregate": eng}, fh, indent=1)


if __name__ == "__main__":
    main()
