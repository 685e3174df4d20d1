"""Cost of FLDetector (``--detect fldetector``) on one GPU.

    python scripts/bench_fldetector.py [--ks 8,32,200] [--window 10] [--iters 20] [--rounds 16] [--reps 2] [--out FILE]

1. Kernels over the ResNet-18 voted coordinates (``n_vote``): the ring pass (``fld_ring_kernel``), the ring Gram over the N + 1 ring rows
   (``pairwise_sqdist_kernel<true, true>``), the Hessian-vector product (``fld_hvp_kernel``) and, for each K, the prediction pass
   (``fld_predict_kernel<true>``, with its ordered sum) and the record-only pass (``<false>``).  CUDA events around ``--iters`` launches
   after warm-up.  Bytes are computed from the shapes: the ring pass reads w_g and w_prev and writes s and w_prev (16 B per coordinate);
   the Gram reads the N + 1 rows once; the product reads them and writes Hv; the prediction reads each slot and table row and writes the
   row (12 B per candidate and coordinate) and reads w_g and Hv once per group of 8 candidates.
2. Engine: ms per round (local training + aggregation, device-timed phases) and ``ms_aggregate`` of CIFAR-10 ResNet-18 with 8 agents,
   ``--aggr avg`` without detection against ``--detect fldetector`` with window ``--window``, alternated.  For the avg run every round but
   the first counts; for the detection run the rounds from N + 2 on, the ones that run the whole pass (ring, Gram, product, prediction).

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


def bench_kernels(ks, window, iters):
    import torch
    from rlr_b200 import ops
    from rlr_b200.models import get_layout
    lay = get_layout("resnet18")
    n, nv = lay.n_total, lay.n_vote
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    g = torch.randn(n, generator=gen, device=dev)
    w_prev = g[:nv] - 0.01 * torch.randn(nv, generator=gen, device=dev)
    ring = 0.01 * torch.randn((window + 1, nv), generator=gen, device=dev)
    pool = [g + 0.01 * torch.randn(n, generator=gen, device=dev) for _ in range(max(ks))]
    table = torch.zeros((max(ks), nv), dtype=torch.float32, device=dev)
    hv = torch.empty(nv, device=dev)
    rtab = ops.PtrTable([ring[i].data_ptr() for i in range(window + 1)], dev)
    coef = torch.as_tensor(ops.fld_hvp_coefficients(ops.history_gram_statement([ring[i] for i in range(window + 1)], 0, nv))).to(dev)
    G = torch.empty(window + 1, window + 1, dtype=torch.float64, device=dev)
    t_ring = time_ms(lambda: ops.ext().fld_ring(g.data_ptr(), w_prev.data_ptr(), ring[0].data_ptr(), 0, nv), iters)
    t_gram = time_ms(lambda: ops.ext().history_gram(rtab.tensor, 0, nv, G), iters)
    t_hvp = time_ms(lambda: ops.ext().fld_hvp(rtab.tensor, coef, hv.data_ptr(), 0, nv), iters)
    head = dict(n_vote=nv, window=window,
                ring_ms=round(t_ring, 4), ring_GBps=round(16 * nv / t_ring / 1e6, 1), ring_floor_ms=round(16 * nv / HBM * 1e3, 4),
                ring_gram_ms=round(t_gram, 4), ring_gram_GBps=round(4 * (window + 1) * nv / t_gram / 1e6, 1),
                hvp_ms=round(t_hvp, 4), hvp_GBps=round(4 * (window + 2) * nv / t_hvp / 1e6, 1))
    rows = []
    for K in ks:
        tab = ops.PtrTable([w.data_ptr() for w in pool[:K]], dev)
        htab = ops.PtrTable([table[k].data_ptr() for k in range(K)], dev)
        out = torch.empty(K, dtype=torch.float64, device=dev)
        pred = lambda: ops.ext().fld_predict(tab.tensor, htab.tensor, g.data_ptr(), hv.data_ptr(), 0, nv, out, None, None, 0, 1, 0)
        rec = lambda: ops.ext().fld_predict(tab.tensor, htab.tensor, g.data_ptr(), 0, 0, nv, None, None, None, 0, 1, 0)
        t_p, t_r = time_ms(pred, iters), time_ms(rec, iters)
        t_p2 = time_ms(pred, iters)                                      # again after the other: the spread of the measurement
        groups = (K + 7) // 8
        bytes_p = 12 * K * nv + 8 * nv * groups
        bytes_r = 8 * K * nv + 4 * nv * groups
        b_p = min(t_p, t_p2)
        rows.append(dict(K=K, predict_ms=round(b_p, 4), predict_ms_repeat=round(max(t_p, t_p2), 4),
                         predict_GBps=round(bytes_p / b_p / 1e6, 1), predict_floor_ms=round(bytes_p / HBM * 1e3, 4),
                         record_ms=round(t_r, 4), record_GBps=round(bytes_r / t_r / 1e6, 1),
                         round_passes_ms=round(t_ring + t_gram + t_hvp + b_p, 4)))
        del tab, htab, out
    return head, rows


def bench_engine(rounds, reps, window):
    import torch
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    res = {a: {"round": [], "aggregate": []} for a in ("avg", "fldetector")}
    for _ in range(reps):
        for det in ("avg", "fldetector"):
            kw = dict(detect="fldetector", fld_window=window) if det == "fldetector" else {}
            args = make_args(data="cifar10", model="resnet18", num_agents=8, num_corrupt=1, poison_frac=0.5, local_ep=1, bs=256,
                             synthetic=8 * 1024, synthetic_val=256, log_dir="", device="cuda:0", rounds=rounds, snap=10 ** 6, **kw)
            eng = FLEngine(args, verbose=False)
            first = window + 2 if det == "fldetector" else 2          # the first round captures the CUDA graphs
            for r in range(1, rounds + 1):
                eng.run_round(r)
                torch.cuda.synchronize()
                el = eng.timer.elapsed()
                if r >= first:
                    res[det]["round"].append(el["local_train"] + el["aggregate"])
                    res[det]["aggregate"].append(el["aggregate"])
            eng.close()
            del eng
            torch.cuda.empty_cache()
    stat = lambda v: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3), rounds=len(v))
    return {a: {k: stat(v) for k, v in d.items()} for a, d in res.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--ks", type=str, default="8,32,200")
    p.add_argument("--window", type=int, default=10)
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--rounds", type=int, default=16, help="engine rounds per run (must exceed --window + 1)")
    p.add_argument("--reps", type=int, default=2, help="alternations of the avg / fldetector engine runs")
    p.add_argument("--out", type=str, default="", help="also write the JSON result here")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_fldetector.py needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    head, rows = bench_kernels([int(k) for k in a.ks.split(",")], a.window, a.iters)
    print(json.dumps(head))
    for r in rows:
        print(json.dumps(r))
    eng = bench_engine(a.rounds, a.reps, a.window) if a.rounds > a.window + 1 else {}
    print(json.dumps({"engine": eng}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"card": info, "passes": head, "kernels": rows, "engine": eng}, fh, indent=1)


if __name__ == "__main__":
    main()
