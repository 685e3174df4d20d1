"""Cost of the colluding attackers (``--attack_collude``) on one GPU.

    python scripts/bench_collude.py [--ks 8,40] [--iters 20] [--out FILE]

Each pass of ``ops/csrc/collude.cu`` over the ResNet-18 voted coordinates (``n_vote``), with K participants of which C = K / 4 are
corrupt, timed with CUDA events around ``--iters`` launches after warm-up:
- ``alie``: the one write pass (ALIE's whole attack);
- ``stats``: the Min-Max / Min-Sum statistics pass;
- ``write``: the Min-Max / Min-Sum write pass once gamma* is known;
- ``dist``: the honest squared distances (``pairwise_sqdist_kernel`` over the H honest participants), which Min-Max / Min-Sum also need.
Bytes are computed from the shapes: every collude pass reads the K participants and w_global once, 4 (K + 1) n_vote bytes, and a write
pass also writes the C corrupt slots, 4 C n_vote bytes; the distance pass reads 4 H n_vote bytes.  The rate is set against the H100 SXM
data sheet's 3.35 TB/s.  The card's name, power limit and maximum SM clock are read in the same run and printed with the numbers.
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

HBM = 3.35e12


def bench(ks, iters):
    import torch
    from rlr_b200 import ops
    from rlr_b200.models import get_layout
    nv = get_layout("resnet18").n_vote
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    g = torch.randn(nv, generator=gen, device=dev)
    pool = [g + 0.01 * torch.randn(nv, generator=gen, device=dev) for _ in range(max(ks))]
    rows = []
    for K in ks:
        C = max(1, K // 4)
        H = K - C
        ws = pool[:K]
        outs = [torch.empty_like(g) for _ in range(C)]
        tab = ops.PtrTable([w.data_ptr() for w in ws], dev)
        htab = ops.PtrTable([w.data_ptr() for w in ws[:H]], dev)
        otab = ops.PtrTable([o.data_ptr() for o in outs], dev)
        st = torch.empty(2 * H + 1, dtype=torch.float64, device=dev)
        d2 = torch.empty(1, dtype=torch.float64, device=dev)
        D = torch.empty((H, H), dtype=torch.float64, device=dev)
        z = ops.collude_z(H, C)
        bd = ops.COLLUDE_DIR_IDS["backdoor"]
        passes = {
            "alie": (lambda: ops.ext().collude_write(tab.tensor, H, otab.tensor, g.data_ptr(), 0, bd, z, 0.0, 0, nv, d2, None, None, 0, 1, 0),
                     4 * (K + 1 + C) * nv),
            "stats": (lambda: ops.ext().collude_stats(tab.tensor, H, g.data_ptr(), bd, 0, nv, st, None, None, 0, 1, 0), 4 * (K + 1) * nv),
            "write": (lambda: ops.ext().collude_write(tab.tensor, H, otab.tensor, g.data_ptr(), 1, bd, 0.0, 0.5, 0, nv, d2, None, None, 0, 1,
                                                      0), 4 * (K + 1 + C) * nv),
            "dist": (lambda: ops.ext().pairwise_sqdist(htab.tensor, 0, None, 0, nv, D, None, None, 0, 1, 0), 4 * H * nv),
        }
        for name, (fn, nbytes) in passes.items():
            t = min(time_ms(fn, iters), time_ms(fn, iters))             # two windows; the lower one
            rows.append(dict(K=K, H=H, C=C, n_vote=nv, pass_=name, ms=round(t, 4), GBps=round(nbytes / t / 1e6, 1),
                             hbm_share=round(nbytes / (t / 1e3) / HBM, 3)))
        del tab, htab, otab, outs
    return rows


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--ks", type=str, default="8,40")
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--out", type=str, default="", help="also write the JSON result here")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_collude.py needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    rows = bench([int(k) for k in a.ks.split(",")], a.iters)
    for r in rows:
        print(json.dumps(r))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"card": info, "passes": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
