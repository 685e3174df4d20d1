"""Weight-gradient launches of ResNet-18's stride-1 3x3 convs alone, the filter-row kernel against the kernels it replaces.

    python scripts/bench_wgrad.py [--bs 256] [--reps 50] [--rounds 3] [--out DIR]

Each shape the filter-row kernel takes (layer 1 on 16 x 8 tiles, layers 2 and 3 on whole-row tiles) is run through
``ops.conv2d_wgrad_sm100`` with ``set_wgrad_rows(False)`` and ``set_wgrad_rows(True)`` alternated, ``--rounds`` times each, ``--reps``
back-to-back launches per timing (CUDA events).  Per row: us per call (median over the rounds, with the spread), TFLOP/s,
L2 operand TB/s and CTAs (launch shapes from ``scripts/profile_step.py:wgrad_launch``), and the time of the ordered split-K sum
that follows the kernel (torch.profiler, in a separate run of the same launches).  The card's name, power limit and maximum SM
clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from profile_step import gpu_info, short_name, wgrad_launch  # noqa: E402

SHAPES = [("layer1", 32, 64, 64), ("layer2", 16, 128, 128), ("layer3", 8, 256, 256)]   # name, H = W, Cin, Cout


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bs", type=int, default=256)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write DIR/bench_wgrad.json")
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from rlr_b200 import ops

    if not torch.cuda.is_available():
        raise SystemExit("bench_wgrad.py measures on the GPU; no CUDA device is visible")
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ext = ops.ext()
    rows = []
    for name, H, Cin, Cout in SHAPES:
        torch.manual_seed(H + Cin)
        x = torch.randn(a.bs, H, H, Cin, device=dev).to(torch.bfloat16)
        dy = torch.randn(a.bs, H, H, Cout, device=dev).to(torch.bfloat16)
        gw = torch.zeros(Cout, 3, 3, Cin, device=dev)
        call = lambda: ops.conv2d_wgrad_sm100(x, dy, gw, None, 1, 1, tag=("bench-wgrad", H), zero=False)  # noqa: E731
        times = {False: [], True: []}
        for on in (False, True):                                  # warm-up: module load, scratch allocation
            ext.set_wgrad_rows(on)
            for _ in range(5):
                call()
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for on in (False, True):
                ext.set_wgrad_rows(on)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.reps):
                    call()
                e1.record()
                torch.cuda.synchronize()
                times[on].append(e0.elapsed_time(e1) * 1e3 / a.reps)
        for on in (False, True):
            ext.set_wgrad_rows(on)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.reps):
                    call()
                torch.cuda.synchronize()
            kern, sums = 0.0, 0.0
            for e in prof.events():
                if e.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                nm = short_name(e.name)
                if nm.startswith("umma_wgrad"):
                    kern += e.device_time
                elif "ordered_sum" in nm:
                    sums += e.device_time
            rec = wgrad_launch(a.bs, H, H, Cin, H, H, Cout, 3, 1, 1, sms, rows=on)
            us = statistics.median(times[on])
            rows.append({"shape": name, "H": H, "Cin": Cin, "Cout": Cout, "kernel": rec["kernel"], "ctas": rec["ctas"], "splits": rec["splits"],
                         "us_per_call": us, "us_min": min(times[on]), "us_max": max(times[on]),
                         "kernel_us": kern / a.reps, "sum_us": sums / a.reps, "tflops": rec["flop"] / (us * 1e-6) / 1e12,
                         "kernel_l2_tb_s": rec["l2_bytes"] / (kern / a.reps * 1e-6) / 1e12 if kern else None,
                         "kernel_tflops": rec["flop"] / (kern / a.reps * 1e-6) / 1e12 if kern else None,
                         "l2_mb": rec["l2_bytes"] / 1e6})
    ext.set_wgrad_rows(True)
    gpu = gpu_info()
    md = [f"GPU: {gpu} (name, power limit, max SM clock); batch {a.bs}, {a.reps} launches per timing, {a.rounds} alternated rounds", "",
          "| shape | kernel | CTAs | us/call (min-max) | TFLOP/s | kernel us | kernel TFLOP/s | L2 operand MB | L2 TB/s | split-K sum us |",
          "|---|---|---:|---:|---:|---:|---:|---:|---:|---:|"]
    for r in rows:
        md.append(f'| {r["shape"]} {r["H"]}x{r["H"]} {r["Cin"]}->{r["Cout"]} | `{r["kernel"]}` | {r["ctas"]} | {r["us_per_call"]:.1f} '
                  f'({r["us_min"]:.1f}-{r["us_max"]:.1f}) | {r["tflops"]:.0f} | {r["kernel_us"]:.1f} | {r["kernel_tflops"] or 0:.0f} | '
                  f'{r["l2_mb"]:.0f} | {r["kernel_l2_tb_s"] or 0:.2f} | {r["sum_us"]:.1f} |')
    print("\n".join(md))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_wgrad.json"), "w") as f:
            json.dump({"gpu": gpu, "batch": a.bs, "rows": rows}, f, indent=1)
    print(json.dumps({"gpu": gpu, "rows": [{k: r[k] for k in ("shape", "kernel", "us_per_call", "sum_us")} for r in rows]}))


if __name__ == "__main__":
    main()
