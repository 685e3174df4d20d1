"""Cost of Krum / Multi-Krum selection (``--select``) on one GPU.

    python scripts/bench_select.py [--ks 8,10,40,64] [--iters 20] [--rounds 5] [--out FILE]

1. Kernel: ``pairwise_sqdist_kernel`` over the ResNet-18 voted coordinates (``n_vote``) for each K, next to ``fused_aggregate_kernel``
   (avg, the engine's single-GPU launch with its bf16 shadow) over the same K vectors -- both read the same K parameter vectors, so the
   aggregate kernel is the memory yardstick.  CUDA events around ``--iters`` launches after warm-up.  Bytes and FLOPs are computed from
   the shapes: the distance pass reads K * n_vote fp32 values once (K <= 64); its useful work is K (K - 1) / 2 pairs x n_vote x 3 FLOPs
   (subtract, fused multiply-add), and the FP32 issue floor counts the pairs the kernel actually computes (4 x 4 blocks of the upper
   triangle) at 2 instructions per pair and coordinate.
2. Engine: ``ms_aggregate`` (host-timed phase: selection, its device->host read of the K x K matrix, and the server step) of
   ``federated.py``-style rounds of CIFAR-10 ResNet-18 with 8 agents, ``--select none`` against ``--select multikrum``, alternated.

The card's name, power limit and maximum SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0), "sms": torch.cuda.get_device_properties(0).multi_processor_count}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["max_sm_mhz"] = float(q[0]), float(q[1])
    except Exception:  # noqa: BLE001
        info["power_limit_w"], info["max_sm_mhz"] = None, None
    return info


def time_ms(fn, iters, warmup=3):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench_kernels(ks, iters, info):
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
    peak_fp32_instr = info["sms"] * 128 * (info["max_sm_mhz"] or 1980.0) * 1e6      # FP32 lanes x clock: instructions per second
    rows = []
    for K in ks:
        ws = pool[:K]
        tab = ops.PtrTable([w.data_ptr() for w in ws], dev)
        D = torch.empty(K, K, dtype=torch.float64, device=dev)
        wt = torch.full((K,), 100.0, dtype=torch.float64, device=dev)
        dist = lambda: ops.ext().pairwise_sqdist(tab.tensor, 0, None, 0, nv, D, None, None, 0, 1, 0)
        agg = lambda: ops.ext().fused_aggregate(tab.tensor, wt, None, 100.0 * K, g.data_ptr(), outs.tensor, outs_b.tensor, False, 0, n,
                                                nv, 0, 0, 1.0, 0.0, 0, 0, None, None, None, 0, 1, 0, False, *ops.opt_launch_args(None))
        t_d, t_a = time_ms(dist, iters), time_ms(agg, iters)
        t_d2 = time_ms(dist, iters)                         # again after the aggregate: the spread of the measurement
        nb = (K + 3) // 4
        computed_pairs = 16 * nb * (nb + 1) // 2
        bytes_d = 4 * K * nv
        bytes_a = 4 * K * n + 4 * n + 4 * n + 2 * n
        flops_d = 3 * (K * (K - 1) // 2) * nv
        floor_issue_ms = 2 * computed_pairs * nv / peak_fp32_instr * 1e3
        floor_mem_ms = bytes_d / 3.35e12 * 1e3
        rows.append(dict(K=K, n_vote=nv, dist_ms=round(min(t_d, t_d2), 4), dist_ms_repeat=round(max(t_d, t_d2), 4), agg_ms=round(t_a, 4),
                         ratio=round(min(t_d, t_d2) / t_a, 3), dist_GBps=round(bytes_d / min(t_d, t_d2) / 1e6, 1),
                         agg_GBps=round(bytes_a / t_a / 1e6, 1), dist_TFLOPs=round(flops_d / min(t_d, t_d2) / 1e9, 2),
                         fp32_issue_floor_ms=round(floor_issue_ms, 4), hbm_floor_ms=round(floor_mem_ms, 4),
                         larger_floor="FP32 issue" if floor_issue_ms > floor_mem_ms else "HBM"))
        del tab, D
    return rows


def bench_engine(rounds, reps):
    import torch
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    res = {"none": [], "multikrum": []}
    for rep in range(reps):
        for sel in ("none", "multikrum"):
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
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--rounds", type=int, default=5, help="engine rounds per run (the first is not counted)")
    p.add_argument("--reps", type=int, default=2, help="alternations of the none / multikrum engine runs")
    p.add_argument("--out", type=str, default="", help="also write the JSON result here")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_select.py needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    rows = bench_kernels([int(k) for k in a.ks.split(",")], a.iters, info)
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
