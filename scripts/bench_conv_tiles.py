"""Per-shape A/B of the conv tile rule (pick_conv_tile in gemm.cu): the layer-3 / layer-4 convolutions of the ResNet-18 training
step (CIFAR shape), each timed alone, one-wave tiles off and on in alternation.

    python scripts/bench_conv_tiles.py [--bs 256] [--rounds 6] [--launches 10] [--out DIR]

Every shape is warmed up in both modes, then ``--rounds`` times: mode off, ``--launches`` back-to-back launches between two CUDA
events; mode on, the same.  Reported per mode: the median microseconds per call over the rounds, TFLOP/s (2 M N K of useful work)
and the L2 operand TB/s (what the CTAs' TMA loads read, from the tile and the grid).  A stride-2 data gradient is its parity-plane
launches together.  The card's name, power limit and maximum SM clock are read in the same run.  Timings of a launch alone do not
include the weight-gradient kernels that share the SMs with the data gradients inside the step: scripts/profile_step.py measures that.
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

from profile_step import BK, BM, conv_tiles, gpu_info, pick_bn  # noqa: E402

# kind, H (input of the forward conv), Cin, Cout, k, stride, pad, calls per step
SHAPES = [
    ("fwd", 8, 256, 256, 3, 1, 1, 3), ("fwd", 16, 128, 256, 3, 2, 1, 1), ("fwd", 16, 128, 256, 1, 2, 0, 1),
    ("fwd", 4, 512, 512, 3, 1, 1, 3), ("fwd", 8, 256, 512, 3, 2, 1, 1), ("fwd", 8, 256, 512, 1, 2, 0, 1),
    ("dgrad", 8, 256, 256, 3, 1, 1, 3), ("dgrad", 4, 512, 512, 3, 1, 1, 3),
    ("dgrad", 16, 128, 256, 3, 2, 1, 1), ("dgrad", 16, 128, 256, 1, 2, 0, 1),
]


def launches_of(kind, B, H, Cin, Cout, k, s, p):
    """(M, N, K, m_tiles) of every generic-kernel launch behind one call."""
    Ho = (H + 2 * p - k) // s + 1
    if kind == "fwd":
        return [(B * Ho * Ho, Cout, k * k * Cin, conv_tiles(B, Ho, Ho))]
    if s == 1:
        return [(B * H * H, Cin, k * k * Cout, conv_tiles(B, H, H))]
    taps = [sum(1 for fy in range(k) for fx in range(k) if (pi + p - fy) % 2 == 0 and (pj + p - fx) % 2 == 0)
            for pi in range(2) for pj in range(2)]
    return [(B * Ho * Ho, Cin, t * Cout, conv_tiles(B, Ho, Ho)) for t in taps if t]


def figures(recs, sms, one_wave):
    flop = l2 = 0.0
    tiles = []
    for M, N, K, m_tiles in recs:
        bn = pick_bn(N, K, m_tiles, sms, True, one_wave)
        ctas = m_tiles * -(-N // bn)
        flop += 2.0 * M * N * K
        l2 += ctas * -(-K // BK) * (BM + bn) * BK * 2
        tiles.append(f"{BM}x{bn} {m_tiles}x{-(-N // bn)}")
    return flop, l2, sorted(set(tiles))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bs", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    from rlr_b200 import ops

    if not torch.cuda.is_available():
        raise SystemExit("bench_conv_tiles.py measures on the GPU; no CUDA device is visible")
    dev, bf = torch.device("cuda", 0), torch.bfloat16
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ext = ops.ext()
    rows = []
    try:
        for kind, H, Cin, Cout, k, s, p, per_step in SHAPES:
            B = a.bs
            Ho = (H + 2 * p - k) // s + 1
            torch.manual_seed(H + Cin + k)
            x = torch.randn(B, H, H, Cin, device=dev).to(bf)
            w = (torch.randn(Cout, k, k, Cin, device=dev) / (k * k * Cin) ** 0.5).to(bf)
            y = torch.randn(B, Ho, Ho, Cout, device=dev).to(bf)
            dx = torch.empty_like(x)
            if kind == "fwd":
                call = lambda: ops.conv2d_fwd_sm100(x, w, None, y, s, p, False, None, tag=("tiles", H, Cin, k, s))  # noqa: E731
            else:
                call = lambda: ops.conv2d_dgrad_sm100(y, w, dx, s, p, False)  # noqa: E731
            outs, us = {}, {False: [], True: []}
            for on in (False, True):
                ext.set_conv_one_wave(on)
                for _ in range(3):
                    call()
                torch.cuda.synchronize()
                outs[on] = (y if kind == "fwd" else dx).clone()
            for _ in range(a.rounds):
                for on in (False, True):
                    ext.set_conv_one_wave(on)
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    ev0.record()
                    for _ in range(a.launches):
                        call()
                    ev1.record()
                    torch.cuda.synchronize()
                    us[on].append(ev0.elapsed_time(ev1) * 1e3 / a.launches)
            recs = launches_of(kind, B, H, Cin, Cout, k, s, p)
            row = {"kind": kind, "shape": f"{H}x{H} {Cin}->{Cout} {k}x{k}/s{s}", "calls_per_step": per_step,
                   "same_bits": bool(torch.equal(outs[False], outs[True]))}
            for on in (False, True):
                flop, l2, tiles = figures(recs, sms, on)
                t = statistics.median(us[on])
                row["on" if on else "off"] = {"tiles": tiles, "us": t, "us_min": min(us[on]), "us_max": max(us[on]),
                                              "tflops": flop / t / 1e6, "l2_tb_s": l2 / t / 1e6}
            rows.append(row)
    finally:
        ext.set_conv_one_wave(True)
    gpu = gpu_info()
    md = [f"GPU: {gpu} (name, power limit, max SM clock); batch {a.bs}; {a.rounds} rounds x {a.launches} launches per mode, alternated; "
          "median us per call (min-max over the rounds).", "",
          "| conv | calls/step | tiles off | us off | TFLOP/s | L2 TB/s | tiles on | us on | TFLOP/s | L2 TB/s | on/off | same bits |",
          "|---|---:|---|---:|---:|---:|---|---:|---:|---:|---:|---|"]
    for r in rows:
        cells = []
        for m in ("off", "on"):
            v = r[m]
            cells += ["; ".join(v["tiles"]), f'{v["us"]:.1f} ({v["us_min"]:.1f}-{v["us_max"]:.1f})', f'{v["tflops"]:.0f}', f'{v["l2_tb_s"]:.2f}']
        md.append(f'| {r["kind"]} {r["shape"]} | {r["calls_per_step"]} | ' + " | ".join(cells) +
                  f' | {r["on"]["us"] / r["off"]["us"]:.3f} | {"yes" if r["same_bits"] else "NO"} |')
    print("\n".join(md))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_conv_tiles.json"), "w") as f:
            json.dump({"gpu": gpu, "batch": a.bs, "rows": rows}, f, indent=1)
        with open(os.path.join(a.out, "bench_conv_tiles.md"), "w") as f:
            f.write("\n".join(md) + "\n")


if __name__ == "__main__":
    main()
