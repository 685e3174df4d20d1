"""Cost of the local objectives (``--prox_mu``, ``--attack_constrain``) on one GPU.

    python scripts/bench_prox.py [--iters 50] [--reps 5] [--out FILE]

Three arms, alternated ``--reps`` times in one process: the default objective (plain cross-entropy), FedProx (``--prox_mu 0.01``:
``(a, b, mu) = (1, 0, 0.01)``) and constrain-and-scale's corrupt agent (``--attack_constrain 0.7``: ``(0.7, 0.3, 0)``).

1. The optimizer alone (``ops.FlatSGD.step`` at the ResNet-18 flat size, no PGD, bf16 shadow written), CUDA events around ``--iters``
   steps after warm-up.  Bytes: the default step reads g in the norm pass and g, m, w and writes m, w and the shadow in the step
   (26 bytes per coordinate); an objective adds w and w0 to the norm pass and w0 to the step over the model parameters (12 bytes per
   voted coordinate).
2. One local step of CIFAR-10 ResNet-18 (batch 256, native trainer), graph replay: one trainer captures its full-batch step under each
   objective, and each replay is preceded by the reset of the batch cursor, as in ``scripts/bench_attacks.py``.

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

ARMS = {"default": None, "prox_mu 0.01": (1.0, 0.0, 0.01), "attack_constrain 0.7": (0.7, 0.3, 0.0)}


def _stat(v):
    return dict(median_ms=round(statistics.median(v), 4), min_ms=round(min(v), 4), max_ms=round(max(v), 4))


def bench_optimizer(iters, reps):
    import torch
    from rlr_b200 import ops
    from rlr_b200.models import get_layout
    lay = get_layout("resnet18")
    n, nv = lay.n_total, lay.n_vote
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    w0 = torch.randn(n, generator=gen, device=dev)
    g = torch.randn(n, generator=gen, device=dev)
    w, m = w0 + 1e-3 * torch.randn(n, generator=gen, device=dev), torch.zeros(n, device=dev)
    wb = torch.empty(n, dtype=torch.bfloat16, device=dev)
    opt = ops.FlatSGD(n, dev, 1e-6, 0.9, 10.0, 0.0, n_pgd=nv)
    ts = {k: [] for k in ARMS}
    for _ in range(reps):
        for name, obj in ARMS.items():
            ts[name].append(time_ms(lambda: opt.step(w, g, m, w0=w0, w_bf16=wb, objective=obj), iters))
    out = {k: _stat(v) for k, v in ts.items()}
    for name, obj in ARMS.items():
        b = 26 * n + (0 if obj is None else 12 * nv)
        out[name].update(bytes=b, TBps=round(b / out[name]["median_ms"] / 1e9, 3), hbm_floor_ms=round(b / 3.35e12 * 1e3, 4))
    return dict(n=n, n_vote=nv, **out)


def bench_step(iters, reps):
    import torch
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    args = make_args(data="cifar10", model="resnet18", num_agents=2, local_ep=1, bs=256, synthetic=2 * 1024, synthetic_val=256, log_dir="",
                     device="cuda:0", rounds=1, snap=10 ** 6)
    eng = FLEngine(args, verbose=False)
    assert eng.trainer.name == "native"
    eng.run_round(1)
    torch.cuda.synchronize()
    tr, agent = eng.trainer, eng.agents[0]
    graphs = {}
    for name, obj in ARMS.items():
        tr._objective = obj
        graphs[name] = tr._get_graph(agent.dataset, tr.bs, eng.w_global)
    tr.perm[:agent.n_data].copy_(agent.idxs)
    ts = {k: [] for k in ARMS}

    def step(gr):
        # each replay advances the trainer's batch cursor: reset it so every replay reads the first batch of the shard
        return lambda: (tr.cursor.zero_(), gr.replay())
    for _ in range(reps):
        for name, gr in graphs.items():
            ts[name].append(time_ms(step(gr), iters))
    eng.close()
    return {k: _stat(v) for k, v in ts.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=50)
    p.add_argument("--reps", type=int, default=5, help="alternations of the three arms")
    p.add_argument("--out", type=str, default="", help="also write the JSON result here")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_prox.py needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    opt = bench_optimizer(a.iters, a.reps)
    print(json.dumps({"optimizer": opt}))
    step = bench_step(a.iters, a.reps)
    print(json.dumps({"step": step}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"card": info, "optimizer": opt, "step": step}, fh, indent=1)


if __name__ == "__main__":
    main()
