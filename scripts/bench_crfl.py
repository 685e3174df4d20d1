"""Cost of CRFL (``--param_clip`` / ``--param_noise`` / ``--certify``) on one GPU.

    python scripts/bench_crfl.py [--iters 200] [--draws 8] [--val 10000] [--out FILE]

1. The clip-and-perturb pass alone (``ops.crfl_step``: the masked fp64 norm, the ordered sum of its per-CTA slots, the apply pass) at the
   ResNet-18 size, with the clip active and sigma = 0.01, CUDA events around ``--iters`` launches after warm-up.  Bytes: 4 per real
   coordinate and 1/8 per voted coordinate (the mask) in the norm pass; 4 read, 4 + 2 written per coordinate and 1/8 per voted coordinate
   in the apply pass.  Reported against the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.
2. Certification of cnn_cifar and resnet18 on a ``--val``-image synthetic CIFAR-10 validation set (and its poisoned copy, as
   ``FLEngine.certify`` sweeps both): ms per draw (the smoothing pass, then every batch's forward and vote count), and the share of a
   draw spent outside the forwards, from a second timing of the forwards alone over the same prepared batches.

The card's name, power limit and maximum SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_select import card, time_ms  # noqa: E402


def pass_bytes(n, nv, n_params):
    return 4 * n_params + nv // 8 + 10 * n + nv // 8


def bench_pass(iters):
    import torch
    from rlr_b200 import ops
    from rlr_b200.models import get_layout
    lay = get_layout("resnet18")
    n, nv = lay.n_total, lay.n_vote
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    wn = 0.05 * torch.randn(n, generator=gen, device=dev)
    w, wb = torch.empty_like(wn), torch.empty(n, dtype=torch.bfloat16, device=dev)
    mask = ops.real_mask(lay).to(dev)
    stats = torch.zeros(2, dtype=torch.float64, device=dev)
    t = time_ms(lambda: ops.crfl_step(w, wn, mask, nv, 10.0, 0.01, 1, 3, stats, wb), iters)
    b = pass_bytes(n, nv, lay.n_params)
    return {"n_total": n, "n_vote": nv, "n_params": lay.n_params, "scale": float(stats[1]), "ms": round(t, 4), "bytes": b,
            "GBps": round(b / t / 1e6, 1), "share_of_3.35TBps": round(b / t / 1e6 / 3350, 3)}


def bench_certify(model, draws, val):
    import torch
    from rlr_b200 import ops
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    args = make_args(data="cifar10", model=model, num_agents=2, local_ep=1, bs=256, synthetic=512, synthetic_val=val, log_dir="",
                     device="cuda:0", num_corrupt=1, poison_frac=0.5, param_noise=0.01, certify=True)
    eng = FLEngine(args, verbose=False)
    w = eng.global_params()
    cw, cwb, prepare, forward = eng.trainer.certify_executor()
    mask = eng.fused.crfl_mask
    sets = []
    for ds in (eng.val_dataset, eng.poisoned_val):
        idx = torch.arange(len(ds), device=ds.device)
        batches = [(s, prepare(ds.batch(idx[s:s + args.bs])[0])) for s in range(0, len(ds), args.bs)]
        sets.append((batches, torch.zeros((len(ds), eng.n_classes), dtype=torch.int32, device=w.device)))
    m = [0]

    def draw():
        ops.crfl_smooth(w, mask, eng.layout.n_vote, args.param_noise, args.seed, m[0], cw, cwb)
        m[0] += 1
        for batches, counts in sets:
            for s, xb in batches:
                ops.vote_count(forward(xb), counts, s)

    def forwards():
        for batches, _ in sets:
            for _, xb in batches:
                forward(xb)

    t_draw = time_ms(draw, draws, warmup=2)
    t_fwd = time_ms(forwards, draws, warmup=2)
    inputs = sum(c.shape[0] for _, c in sets)
    eng.close()
    return {"inputs_per_draw": inputs, "ms_per_draw": round(t_draw, 3), "ms_forwards_per_draw": round(t_fwd, 3),
            "share_outside_forwards": round(1.0 - t_fwd / t_draw, 4),
            "default_certify_s": round(t_draw * (args.certify_n0 + args.certify_n) / 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--draws", type=int, default=8)
    ap.add_argument("--val", type=int, default=10000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_crfl.py measures on a GPU; none is visible")
    res = {"card": card(), "pass_resnet18": bench_pass(a.iters)}
    for model in ("cnn_cifar", "resnet18"):
        res[f"certify_{model}"] = bench_certify(model, a.draws, a.val)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
