"""Cost of FoolsGold aggregation (``--aggr foolsgold``) on one GPU.

    python scripts/bench_foolsgold.py [--ks 8,10,40,64,200] [--iters 20] [--rounds 5] [--reps 2] [--out FILE]

1. Kernels over the ResNet-18 voted coordinates (``n_vote``) for each K: the history accumulate (``history_accumulate_kernel``) and the
   history Gram (``pairwise_sqdist_kernel<true, true>``), next to FLAME's Gram (``pairwise_sqdist_kernel<true>``) and
   ``fused_aggregate_kernel`` (avg, the engine's single-GPU launch with its bf16 shadow) over the same K vectors.  CUDA events around
   ``--iters`` launches after warm-up.  Bytes are computed from the shapes: the accumulate reads each slot once, reads and writes each
   history row once and reads w_global once per group of 8 candidates; a Gram tile reads the rows of its participants once, so the Gram
   passes read every row once for K <= 64 and once per tile it sits in above (FLAME's also reads w_global once per tile read).  A round
   of ``--aggr foolsgold`` runs one accumulate and one history Gram before the aggregate.
2. Engine: ms per round (local training + aggregation, device-timed phases) and ``ms_aggregate`` of CIFAR-10 ResNet-18 with 8 agents,
   ``--aggr avg`` against ``--aggr foolsgold``, alternated; the first round of each run is not counted.

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

HBM = 3.35e12        # H100 SXM HBM3 bandwidth from NVIDIA's data sheet (bytes/s): the floor the ms columns are compared with


def gram_row_reads(K, tile=64):
    """Rows the Gram kernel reads: a diagonal tile reads its participants once, an off-diagonal tile both of its sets."""
    sizes = [min(tile, K - t) for t in range(0, K, tile)]
    return sum(sizes[i] if i == j else sizes[i] + sizes[j] for i in range(len(sizes)) for j in range(i, len(sizes)))


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
    hist = torch.zeros((max(ks), nv), dtype=torch.float32, device=dev)
    out = torch.empty(n, device=dev)
    out_b = torch.empty(n, dtype=torch.bfloat16, device=dev)
    outs, outs_b = ops.PtrTable([out.data_ptr()], dev), ops.PtrTable([out_b.data_ptr()], dev)
    rows = []
    for K in ks:
        tab = ops.PtrTable([w.data_ptr() for w in pool[:K]], dev)
        htab = ops.PtrTable([hist[k].data_ptr() for k in range(K)], dev)
        G = torch.empty(K, K, dtype=torch.float64, device=dev)
        wt = torch.full((K,), 1.0, dtype=torch.float64, device=dev)
        acc = lambda: ops.ext().history_accumulate(tab.tensor, htab.tensor, g.data_ptr(), 0, nv, None, None, 0, 1, 0)
        hgram = lambda: ops.ext().history_gram(htab.tensor, 0, nv, G)
        fgram = lambda: ops.ext().pairwise_gram(tab.tensor, g.data_ptr(), 0, nv, G, None, None, 0, 1, 0)
        agg = lambda: ops.ext().fused_aggregate(tab.tensor, wt, None, float(K), g.data_ptr(), outs.tensor, outs_b.tensor, False, 0, n,
                                                nv, 0, 0, 1.0, 0.0, 0, 0, None, None, None, 0, 1, 0, False, *ops.opt_launch_args(None))
        t_acc, t_hg, t_fg, t_a = time_ms(acc, iters), time_ms(hgram, iters), time_ms(fgram, iters), time_ms(agg, iters)
        t_acc2, t_hg2 = time_ms(acc, iters), time_ms(hgram, iters)      # again after the others: the spread of the measurement
        reads = gram_row_reads(K)
        bytes_acc = 4 * K * nv + 8 * K * nv + 4 * nv * ((K + 7) // 8)
        bytes_hg = 4 * reads * nv
        bytes_fg = 8 * reads * nv
        bytes_a = 4 * K * n + 4 * n + 4 * n + 2 * n
        b_acc, b_hg = min(t_acc, t_acc2), min(t_hg, t_hg2)
        rows.append(dict(K=K, n_vote=nv,
                         accumulate_ms=round(b_acc, 4), accumulate_ms_repeat=round(max(t_acc, t_acc2), 4),
                         accumulate_GBps=round(bytes_acc / b_acc / 1e6, 1), accumulate_floor_ms=round(bytes_acc / HBM * 1e3, 4),
                         history_gram_ms=round(b_hg, 4), history_gram_ms_repeat=round(max(t_hg, t_hg2), 4),
                         history_gram_GBps=round(bytes_hg / b_hg / 1e6, 1), history_gram_floor_ms=round(bytes_hg / HBM * 1e3, 4),
                         flame_gram_ms=round(t_fg, 4), flame_gram_GBps=round(bytes_fg / t_fg / 1e6, 1),
                         agg_ms=round(t_a, 4), agg_GBps=round(bytes_a / t_a / 1e6, 1),
                         foolsgold_passes_over_agg=round((b_acc + b_hg) / t_a, 3)))
        del tab, htab, G
    return rows


def bench_engine(rounds, reps):
    import torch
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    res = {a: {"round": [], "aggregate": []} for a in ("avg", "foolsgold")}
    for _ in range(reps):
        for aggr in ("avg", "foolsgold"):
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
    p.add_argument("--reps", type=int, default=2, help="alternations of the avg / foolsgold engine runs")
    p.add_argument("--out", type=str, default="", help="also write the JSON result here")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_foolsgold.py needs a GPU")
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
