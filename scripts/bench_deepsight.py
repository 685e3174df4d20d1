"""Cost of DeepSight (``--aggr deepsight``) on one GPU.

    python scripts/bench_deepsight.py [--iters 20] [--rounds 10] [--skip 3] [--reps 2] [--out FILE]

1. The logits pass and the statistics pass separately, for K = 8, 40 and 100 candidates on the default 3 x 256 random inputs, for
   cnn_cifar and ResNet-18, CUDA events around ``--iters`` repetitions after warm-up:
   - logits: ``NativeTrainer.root_features(..., tap=False)`` of one parameter vector on the 768 inputs (copied into the feature
     executor, eval-mode forward), which one rank runs for every participant it owns and once for the global model;
   - statistics: the ``deepsight_stats`` launch pair over K candidates (``ops.ext().deepsight_stats``), and the whole pass with the
     pointer table and the host read (``ops.deepsight_stats`` + ``.cpu()``).
2. Engine: ms per round (device-timed local-training and aggregation phases) and the ``aggregate`` phase alone, for CIFAR-10 ResNet-18
   with 8 agents under ``--aggr avg`` and ``--aggr deepsight``, alternated.  The first ``--skip`` rounds of each run (graph capture) are
   not counted.

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

CONFIGS = {"avg": {"aggr": "avg"}, "deepsight": {"aggr": "deepsight"}}
KS = (8, 40, 100)
SAMPLES = 256


def bench_passes(iters):
    import torch
    from rlr_b200 import ops
    from rlr_b200.data import DATASET_META
    from rlr_b200.models import get_layout
    from rlr_b200.models.graph import head_slices
    from rlr_b200.models.native import NativeTrainer
    from rlr_b200.options import make_args
    dev = torch.device("cuda:0")
    out = {}
    x = ops.deepsight_inputs(DATASET_META["cifar10"], 0, SAMPLES, dev)
    for model in ("cnn_cifar", "resnet18"):
        lay = get_layout(model)
        head = head_slices(lay)
        tr = NativeTrainer(lay, make_args(data="cifar10", model=model, device="cuda:0"), dev, 256)
        w = torch.zeros(lay.n_total, device=dev)
        lay.init_(w, 0)
        t_one = time_ms(lambda: tr.root_features(w, x, tap=False), iters)
        res = {"P": head[2], "d": head[3], "inputs": x.shape[0], "logits_ms_per_candidate": round(t_one, 4)}
        gen = torch.Generator(device=dev).manual_seed(0)
        for K in KS:
            ws = [w + 0.01 * torch.randn(lay.n_total, generator=gen, device=dev) for _ in range(min(K, 8))]
            ws = [ws[k % len(ws)] for k in range(K)]
            z = torch.randn(K, x.shape[0], head[2], generator=gen, device=dev)
            zg = torch.randn(x.shape[0], head[2], generator=gen, device=dev)
            tab = ops.PtrTable([v.data_ptr() for v in ws], dev, ws)
            outp = torch.empty(K, (ops.DEEPSIGHT_SEEDS + 2) * head[2], dtype=torch.float64, device=dev)
            t_kernel = time_ms(lambda: ops.ext().deepsight_stats(z, zg, tab.tensor, w.data_ptr(), head[0], head[1], ops.DEEPSIGHT_SEEDS,
                                                                 head[3], outp), iters)
            t_pass = time_ms(lambda: ops.deepsight_stats(z, zg, ws, w, head).cpu(), iters)
            res[f"stats_K{K}"] = dict(kernel_ms=round(t_kernel, 4), pass_ms=round(t_pass, 4), logits_ms=round(t_one * (K + 1), 3))
        out[model] = res
        del tr
        torch.cuda.empty_cache()
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
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--rounds", type=int, default=10, help="engine rounds per run")
    p.add_argument("--skip", type=int, default=3, help="leading rounds of each run not counted (graph capture)")
    p.add_argument("--reps", type=int, default=2, help="alternations of the two engine configurations")
    p.add_argument("--out", type=str, default="", help="also write the JSON result here")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_deepsight.py needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    passes = bench_passes(a.iters)
    print(json.dumps({"passes": passes}))
    eng = bench_engine(a.rounds, a.reps, a.skip) if a.rounds > a.skip else {}
    print(json.dumps({"engine": eng}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"card": info, "passes": passes, "engine": eng}, fh, indent=1)


if __name__ == "__main__":
    main()
