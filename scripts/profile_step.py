"""Per-kernel profile of one training step of the bench.py workload (ResNet-18, CIFAR shape, batch 256, one GPU).

    python scripts/profile_step.py [--out DIR] [--replays N] [--bs 256] [--model resnet18] [--previous_tiles] [--previous_wgrad]

``--model`` profiles another zoo model in the same configuration (e.g. ``resnet18_gn``).  ``--bn_reps`` sets the launches per call
of the BatchNorm isolation and copy-reference measurements.  ``--previous_tiles`` profiles the step without the one-wave conv tiles
(``set_conv_one_wave(False)``), for an A/B in one session.
``--previous_wgrad`` profiles it with the weight-gradient kernels the filter-row kernel replaces (``set_wgrad_rows(False)``).

Builds the engine exactly as ``bench.py`` does, runs one warm-up round (which captures the training-step CUDA graph), then
replays the captured full-batch step ``--replays`` times under ``torch.profiler`` with CUDA activities.  The kernels inside the
graph are listed one by one; the script writes DIR/profile_step.md (and .json) with one row per kernel name: calls and
microseconds per step, share of the step and, for the implicit-GEMM conv / GEMM kernel, its FLOP, L2 operand bytes and achieved
TFLOP/s per launch shape.  FLOP and bytes come from the launch shapes (``launch_record`` below), recorded by wrapping the
extension's conv / GEMM entry points during the warm-up round.  The card's name, power limit and maximum SM clock are read in
the same run (read-only nvidia-smi query).

The BatchNorm family (statistics, apply, backward reduction, backward apply and the ordered sums of their partials) gets a table
of its own, per launch shape: M, C, mode, the HBM bytes each pass must move and the achieved TB/s in the step; then the same calls
replayed one at a time outside the graph (no concurrent side-stream kernels), and a device-to-device copy of the same bytes in the
same session as the attainable bandwidth on that card at its power limit.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BM, BK = 128, 64        # gemm.cu tile rows / k-block depth
KERNEL = "umma_conv_gemm_kernel"


def _pow2_ceil(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def conv_tiles(NB, Ho, Wo):
    """m-tiles of launch_conv_bf16: TW x TH x TN = 128-pixel boxes."""
    TW = min(_pow2_ceil(Wo), BM)
    TH = _pow2_ceil(Ho)
    if TW * TH > BM:
        TH = BM // TW
    TN = BM // (TW * TH)
    return -(-Wo // TW) * -(-Ho // TH) * -(-NB // TN)


ONE_WAVE = True        # False: the tiles of set_conv_one_wave(False)


def pick_bn(N, K, m_tiles, sms, conv, one_wave=None):
    """Tile width launch_conv_bf16 (pick_conv_tile in gemm.cu) / launch_gemm_bf16 choose: 128 when it divides N, else 64; a 128-wide
    conv grid smaller than the SMs goes to the 64-wide tile, unless it fills one wave (0.9 of the SMs) over at least 24 k-blocks."""
    if conv and (ONE_WAVE if one_wave is None else one_wave) and N % 128 == 0 and -(-K // BK) >= 24:
        ctas = m_tiles * (N // 128)
        if ctas <= sms and 10 * ctas >= 9 * sms:
            return 128
    bn = 128 if N % 128 == 0 else 64
    if conv and bn == 128 and m_tiles * (N // 128) < sms:
        bn = 64
    return bn


def launch_record(kind, M, N, K, m_tiles, sms, conv, bmn=False, cluster=(1, 1), one_wave=None):
    """One implicit-GEMM launch: FLOP = 2 M N K (useful work, masked rows excluded) and L2 operand bytes = what the CTAs' TMA
    loads read, every CTA its own A and B tile per 64-deep k-block; an operand shared by the CTAs of a cluster is fetched once
    per cluster (``cluster`` = CTAs along M sharing B, along N sharing A)."""
    bn = pick_bn(N, K, m_tiles, sms, conv, one_wave)
    n_tiles = -(-N // bn)
    kb = -(-K // BK)
    ctas = m_tiles * n_tiles
    cm, cn = cluster
    a_bytes = ctas * kb * BM * BK * 2 / cn
    b_bytes = ctas * kb * bn * BK * 2 / cm
    return {"kind": kind, "M": M, "N": N, "K": K, "bn": bn, "grid": (m_tiles, n_tiles), "bmn": bmn,
            "flop": 2.0 * M * N * K, "l2_bytes": a_bytes + b_bytes}


def install_recorder(ext, sms, log):
    """Wrap the extension's conv / GEMM entry points so every call appends its launch record to ``log``; ``advance_cursor``
    (called once at the end of every training step) appends a step delimiter."""
    orig = {n: getattr(ext, n) for n in ("conv_bf16", "conv_bf16_strided", "gemm_bf16", "stem_gemm_bf16", "advance_cursor")}

    def conv_bf16(x, w, out, NB, planes, dh, *a):
        wtap = a[-2]
        Ho, Wo, Cout, Cin = out.shape[1], out.shape[2], out.shape[3], x.shape[3]
        log.append(launch_record("dgrad" if wtap else "fwd", NB * Ho * Wo, Cout, len(dh) * Cin, conv_tiles(NB, Ho, Wo), sms, True,
                                 bool(wtap)))
        return orig["conv_bf16"](x, w, out, NB, planes, dh, *a)

    def conv_bf16_strided(x, w, out, dh, dw, bias, relu, acc, wtap, T, in_s, out_s, ph, pw):
        NB, Cin, Cout = x.shape[0], x.shape[3], out.shape[3]
        Ho, Wo = out.shape[1] // out_s, out.shape[2] // out_s
        log.append(launch_record("dgrad-s2-plane" if wtap else "fwd-s2", NB * Ho * Wo, Cout, len(dh) * Cin, conv_tiles(NB, Ho, Wo),
                                 sms, True, bool(wtap)))
        return orig["conv_bf16_strided"](x, w, out, dh, dw, bias, relu, acc, wtap, T, in_s, out_s, ph, pw)

    def gemm_bf16(A, B, out, *a, **k):
        M, K, N = A.shape[0], A.shape[1], B.shape[0]
        log.append(launch_record("gemm", M, N, K, -(-M // BM), sms, False))
        return orig["gemm_bf16"](A, B, out, *a, **k)

    def stem_gemm_bf16(A, W, out, *a, **k):
        M, N = A.shape[0], W.shape[0]
        log.append(launch_record("stem", M, N, W.shape[1], -(-M // BM), sms, False))
        return orig["stem_gemm_bf16"](A, W, out, *a, **k)

    def advance_cursor(*a, **k):
        log.append(None)
        return orig["advance_cursor"](*a, **k)

    for n, f in (("conv_bf16", conv_bf16), ("conv_bf16_strided", conv_bf16_strided), ("gemm_bf16", gemm_bf16),
                 ("stem_gemm_bf16", stem_gemm_bf16), ("advance_cursor", advance_cursor)):
        setattr(ext, n, f)
    return orig


ROWS = True            # False: the weight-gradient kernels of set_wgrad_rows(False)
WG_KERNELS = ("umma_wgrad_kernel", "umma_wgrad_halo_kernel", "umma_wgrad_rows_kernel")


def wg_splits(base, num_kb, sms, low_waves=1):
    """Split-K count of the weight-gradient launchers (wg_splits in wgrad.cu)."""
    waves = -(-base // sms) if base >= sms else low_waves
    splits = min(max((waves * sms) // base, 1), num_kb)
    per = -(-num_kb // splits)
    return -(-num_kb // per)


def wgrad_launch(NB, Hin, Win, Cin, Ho, Wo, Cout, k, stride, pad, sms, cin_valid=None, rows=None):
    """Kernel, grid, FLOP and L2 operand bytes of one conv weight-gradient launch (launch_conv_wgrad_bf16 / _halo_bf16 in wgrad.cu):
    L2 operand bytes = every CTA's TMA boxes per k-block (dY tiles and input boxes or halos) over its split-K range."""
    rows = ROWS if rows is None else rows
    cin_valid = Cin if cin_valid is None else cin_valid
    flop = 2.0 * NB * Ho * Wo * Cout * k * k * cin_valid
    co128 = -(-Cout // 128)
    std3 = k == 3 and stride == 1 and pad == 1
    if std3 and Cin == 64 and Hin % 16 == 0 and Win % 8 == 0:                 # 16 x 8 tiles of 128 pixels
        num_kb = NB * (Hin // 16) * (Win // 8)
        splits = wg_splits(co128 * 3, num_kb, sms)
        a_groups = 2 if Cout % 128 == 0 else 1
        return {"kernel": "umma_wgrad_halo_kernel", "grid": (co128, 3, splits), "ctas": co128 * 3 * splits, "splits": splits,
                "flop": flop, "l2_bytes": co128 * 3 * num_kb * (a_groups * 16384 + 18 * 16 * 128)}
    TW = min(_pow2_ceil(Wo), 64)
    TH = _pow2_ceil(Ho)
    if TW * TH > 64:
        TH = 64 // TW
    TN = 64 // (TW * TH)
    num_kb = -(-Wo // TW) * -(-Ho // TH) * -(-NB // TN)
    ci_tiles = Cin // 64
    if rows and std3 and TN == 1 and TW == Wo and TW % 8 == 0 and cin_valid == Cin:
        splits = wg_splits(co128 * ci_tiles * 3, num_kb, sms)
        tiles = -(-Cout // 64) * ci_tiles
        return {"kernel": "umma_wgrad_rows_kernel", "grid": (tiles, 1, splits), "ctas": tiles * splits, "splits": splits,
                "flop": flop, "l2_bytes": tiles * num_kb * (8192 + (TW + 2) * (TH + 2) * 128)}
    wide = Cin % 128 == 0 and cin_valid == Cin and k == 1
    taps = 3 if k == 3 else 1
    groups = 2 if wide else 1
    ci_tiles = Cin // (64 * groups)
    a_groups = 2 if Cout > 64 else 1
    splits = wg_splits(co128 * ci_tiles * (k * k // taps), num_kb, sms)
    grid = (co128 * ci_tiles, k * k // taps, splits)
    return {"kernel": f"umma_wgrad_kernel<{64 * groups}, {taps}>", "grid": grid, "ctas": grid[0] * grid[1] * splits, "splits": splits,
            "flop": flop, "l2_bytes": grid[0] * grid[1] * num_kb * (a_groups * 8192 + taps * groups * 8192)}


def install_wgrad_recorder(ext, sms, log):
    """Wrap the extension's conv weight-gradient entry points so every call appends its ``wgrad_launch`` record to ``log``, with a
    step delimiter at every ``advance_cursor``."""
    orig = {n: getattr(ext, n) for n in ("conv_wgrad_bf16", "conv_wgrad_halo_bf16", "conv_wgrad_bf16_strided", "advance_cursor")}

    def rec(dy, x, dW, stride, cin_valid, planes=1):
        NB, Ho, Wo, Cout = dy.shape
        k = dW.shape[1] if dW.dim() == 4 else 3
        Hin, Win, Cin = x.shape[1], x.shape[2], x.shape[3]
        if planes == 4:                                      # parity-split copy: each plane is one stride-2 phase
            Hin, Win = 2 * Hin, 2 * Win
        pad = (k - 1) // 2
        r = wgrad_launch(NB, Hin, Win, Cin, Ho, Wo, Cout, k, stride, pad, sms, cin_valid)
        r["shape"] = f"{k}x{k}/s{stride} {Hin}x{Win} {Cin}->{Cout}"
        log.append(r)

    def conv_wgrad_bf16(dy, x, dW, NB, planes, cin_valid, dh, dw, pl):
        rec(dy, x, dW, 2 if planes == 4 else 1, cin_valid, planes)
        return orig["conv_wgrad_bf16"](dy, x, dW, NB, planes, cin_valid, dh, dw, pl)

    def conv_wgrad_halo_bf16(dy, x, dW, cin_valid):
        rec(dy, x, dW, 1, cin_valid)
        return orig["conv_wgrad_halo_bf16"](dy, x, dW, cin_valid)

    def conv_wgrad_bf16_strided(dy, x, dW, cin_valid, dh, dw, in_stride):
        rec(dy, x, dW, in_stride, cin_valid)
        return orig["conv_wgrad_bf16_strided"](dy, x, dW, cin_valid, dh, dw, in_stride)

    def advance_cursor(*a, **k):
        log.append(None)
        return orig["advance_cursor"](*a, **k)

    for n, f in (("conv_wgrad_bf16", conv_wgrad_bf16), ("conv_wgrad_halo_bf16", conv_wgrad_halo_bf16),
                 ("conv_wgrad_bf16_strided", conv_wgrad_bf16_strided), ("advance_cursor", advance_cursor)):
        setattr(ext, n, f)
    return orig


def wgrad_table(wg_launches, kernels, replays):
    """Rows of the weight-gradient table: traced weight-gradient kernels keyed by (kernel, grid), matched to the step's launch
    records; the ordered split-K sums that follow them are in the kernel table (``ordered_sum``)."""
    per = collections.defaultdict(lambda: [0, 0.0])
    for e in kernels:
        nm = short_name(e["name"])
        if nm.startswith(WG_KERNELS):
            g = tuple(e.get("args", {}).get("grid", [0, 0, 0])[:3])
            per[(nm, g)][0] += 1
            per[(nm, g)][1] += float(e["dur"])
    by_key = collections.defaultdict(list)
    for r in wg_launches:
        by_key[(r["kernel"].replace(" ", ""), tuple(r["grid"]))].append(r)
    out = []
    for (nm, g), (cnt, us) in sorted(per.items(), key=lambda kv: -kv[1][1]):
        calls = cnt / replays
        us_step = us / replays
        recs = by_key.get((nm.replace(" ", ""), g), [])
        ok = bool(recs) and len(recs) == round(calls) and us_step > 0
        flop = sum(r["flop"] for r in recs)
        l2 = sum(r["l2_bytes"] for r in recs)
        out.append({"kernel": nm, "grid": list(g), "calls_per_step": calls, "us_per_step": us_step,
                    "launches": sorted({r["shape"] for r in recs}), "gflop": flop / 1e9, "l2_mb": l2 / 1e6,
                    "tflops": flop / (us_step * 1e-6) / 1e12 if ok else None, "l2_tb_s": l2 / (us_step * 1e-6) / 1e12 if ok else None})
    return out


BN_KERNELS = ("channel_reduce_kernel", "bn_apply_kernel", "bn_bwd_apply_kernel", "ordered_sum")


def bn_record(kind, x, C, relu=False, res=False, dres=False, recompute=False):
    """One BatchNorm entry-point call: kind 'stats' | 'apply' | 'bwd' (reduction + apply), its shape, mode and HBM bytes per pass
    (bf16 activations, E bytes each): statistics read x; apply reads x (and the residual) and writes y; the backward reduction reads
    dy, x (and y for the mask unless it is recomputed from x); the backward apply reads the same and writes dx (and the residual
    gradient)."""
    M = x.numel() // C
    E = 2 * M * C
    mode = "+".join(m for m, on in (("relu", relu), ("res", res or dres), ("recompute", recompute)) if on) or "plain"
    if kind == "stats":
        passes = {"stats": E}
    elif kind == "apply":
        passes = {"apply": E * (3 if res else 2)}
    else:
        reads = E * (2 if recompute or not relu else 3)
        passes = {"bwd_reduce": reads, "bwd_apply": reads + E * (2 if dres else 1)}
    return {"kind": "bn-" + kind, "M": M, "C": C, "mode": mode, "relu": relu, "res": res, "dres": dres, "recompute": recompute,
            "passes": passes}


def install_bn_recorder(ext, log):
    """Wrap the BatchNorm entry points like install_recorder does the GEMMs; ``advance_cursor`` appends a step delimiter."""
    orig = {n: getattr(ext, n) for n in ("channel_stats", "bn_apply", "bn_bwd", "bn_bwd_recompute", "advance_cursor")}

    def channel_stats(x, stats):
        log.append(bn_record("stats", x, x.shape[-1]))
        return orig["channel_stats"](x, stats)

    def bn_apply(x, res, y, *a):
        if a[4] == 1:                                                    # training (fin_mode 1); evaluation is not in the step
            log.append(bn_record("apply", x, x.shape[-1], relu=bool(a[3]), res=res is not None))
        return orig["bn_apply"](x, res, y, *a)

    def bn_bwd(dy, y, x, gamma, mr, dsum, dx, dres, *a):
        log.append(bn_record("bwd", x, x.shape[-1], relu=bool(a[2]), dres=dres is not None))
        return orig["bn_bwd"](dy, y, x, gamma, mr, dsum, dx, dres, *a)

    def bn_bwd_recompute(dy, x, *a):
        log.append(bn_record("bwd", x, x.shape[-1], relu=True, recompute=True))
        return orig["bn_bwd_recompute"](dy, x, *a)

    def advance_cursor(*a, **k):
        log.append(None)
        return orig["advance_cursor"](*a, **k)

    for n, f in (("channel_stats", channel_stats), ("bn_apply", bn_apply), ("bn_bwd", bn_bwd), ("bn_bwd_recompute", bn_bwd_recompute),
                 ("advance_cursor", advance_cursor)):
        setattr(ext, n, f)
    return orig


def bn_signature(r):
    return (r["kind"], r["M"], r["C"], r["mode"])


def _replay_bn_call(ext, r, dev, torch):
    """Fresh tensors of the recorded shape; returns a closure that issues that one call (the same launches as in the step)."""
    M, C = r["M"], r["C"]
    g = torch.Generator(dev).manual_seed(M + C)
    t = lambda: torch.randn(M, C, device=dev, generator=g).to(torch.bfloat16)  # noqa: E731
    gamma, beta = torch.rand(C, device=dev) + 0.5, torch.randn(C, device=dev) * 0.1
    mr = torch.stack([torch.zeros(C, device=dev), torch.ones(C, device=dev)])
    if r["kind"] == "bn-stats":
        x, stats = t(), torch.zeros(1, 2, C, device=dev)
        return lambda: ext.channel_stats(x, stats)
    if r["kind"] == "bn-apply":
        x, res, y = t(), (t() if r["res"] else None), t()
        stats = torch.stack([torch.zeros(C, device=dev), torch.full((C,), float(M), device=dev)])[None] * 1.0
        rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
        return lambda: ext.bn_apply(x, res, y, gamma, beta, mr, r["relu"], 1, stats, float(M), 1e-5, 0.1, rm, rv)
    dy, x, y, dx = t(), t(), t(), t()
    dres = t() if r["dres"] else None
    dsum, dg, db = torch.zeros(1, 2, C, device=dev), torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    if r["recompute"]:
        return lambda: ext.bn_bwd_recompute(dy, x, gamma, beta, mr, dsum, dx, dg, db, True)
    return lambda: ext.bn_bwd(dy, y, x, gamma, mr, dsum, dx, dres, dg, db, r["relu"], True)


def _trace_kernels(prof):
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
    return [e for e in trace.get("traceEvents", []) if e.get("cat") == "kernel"]


def _pass_of(name):
    if name.startswith("bn_apply_kernel"):
        return "apply"
    if name.startswith("bn_bwd_apply_kernel"):
        return "bwd_apply"
    if name.startswith("channel_reduce_kernel"):
        return "stats" if name.startswith("channel_reduce_kernel<0") else "bwd_reduce"
    return "sum"


def isolate_bn(ext, sigs, reps, dev):
    """Every distinct BatchNorm call of the step replayed alone (no concurrent side-stream kernels), ``reps`` times under the
    profiler: per kernel (name, grid) its microseconds per call.  The same (name, grid) keys identify the launches in the step trace."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for sig, r in sigs.items():
        call = _replay_bn_call(ext, r, dev, torch)
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call()
            torch.cuda.synchronize()
        per = collections.defaultdict(float)
        for e in _trace_kernels(prof):
            nm = short_name(e["name"])
            if nm.startswith(BN_KERNELS):
                per[(nm, tuple(e.get("args", {}).get("grid", [0, 0, 0])[:1]))] += float(e["dur"]) / reps
        out[sig] = dict(per)
    return out


def copy_reference(nbytes_list, reps, dev):
    """Device-to-device copy moving the same bytes (half read, half written): microseconds per copy, CUDA events."""
    import torch
    res = {}
    for nb in sorted(set(nbytes_list)):
        n = max(1, nb // 4)                                      # bf16 elements per side: nb / 2 bytes read + nb / 2 written
        src, dst = torch.ones(n, device=dev, dtype=torch.bfloat16), torch.empty(n, device=dev, dtype=torch.bfloat16)
        for _ in range(3):
            dst.copy_(src)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        ev0.record()
        for _ in range(reps):
            dst.copy_(src)
        ev1.record()
        torch.cuda.synchronize()
        res[nb] = ev0.elapsed_time(ev1) * 1e3 / reps
    return res


def bn_tables(bn_launches, kernels, replays, ext, dev, reps):
    """Per launch shape of the BatchNorm family: bytes, in-step microseconds and TB/s, the same launch alone, and a copy of the same
    bytes.  Rows are (kernel, grid) keys, as for the GEMM table; a key's launches are the step's calls that produce it."""
    counts = collections.Counter(bn_signature(r) for r in bn_launches)
    sigs = {bn_signature(r): r for r in bn_launches}
    iso = isolate_bn(ext, sigs, reps, dev)
    step = collections.defaultdict(lambda: [0, 0.0])
    for e in kernels:
        nm = short_name(e["name"])
        if nm.startswith(BN_KERNELS):
            k = (nm, tuple(e.get("args", {}).get("grid", [0, 0, 0])[:1]))
            step[k][0] += 1
            step[k][1] += float(e["dur"])
    rows = []
    for key, (cnt, us) in sorted(step.items(), key=lambda kv: -kv[1][1]):
        owners = [(s, n) for s, n in counts.items() if key in iso.get(s, {})]
        if not owners:                                           # an ordered sum of a non-BatchNorm user (weight gradients, loss)
            continue
        p = _pass_of(key[0])
        per_launch = [(n, sigs[s]["passes"].get(p, 0)) for s, n in owners]       # the ordered sums: microseconds only
        nbytes = sum(n * b for n, b in per_launch)
        iso_us = sum(n * iso[s][key] for s, n in owners)
        calls, us_step = cnt / replays, us / replays
        matched = round(calls) == sum(n for _, n in owners)
        rows.append({"kernel": key[0], "grid": key[1][0], "pass": p, "calls_per_step": calls, "us_per_step": us_step,
                     "launches": sorted(f"{s[0][3:]} M{s[1]} C{s[2]} {s[3]} x{n}" for s, n in owners), "mb": nbytes / 1e6,
                     "tb_s": nbytes / (us_step * 1e-6) / 1e12 if (matched and nbytes and us_step) else None,
                     "iso_us": iso_us, "iso_tb_s": nbytes / (iso_us * 1e-6) / 1e12 if (nbytes and iso_us) else None,
                     "_per_launch": per_launch})
    cref = copy_reference([b for r in rows for _, b in r["_per_launch"] if b], reps, dev)
    for r in rows:
        cu = sum(n * cref[b] for n, b in r.pop("_per_launch") if b)
        r["copy_us"] = cu or None
        r["copy_tb_s"] = r["mb"] * 1e6 / (cu * 1e-6) / 1e12 if cu else None
    return rows


def one_step_launches(log):
    """Launch records of the first complete full-batch step in the log (an eager warm-up step before the graph is captured):
    the first step whose first launch has the most rows."""
    steps, cur = [], []
    for r in log:
        if r is None:
            steps.append(cur)
            cur = []
        else:
            cur.append(r)
    steps = [s for s in steps if s]
    if not steps:
        raise RuntimeError("no training step was recorded")
    top = max(s[0]["M"] for s in steps)
    return next(s for s in steps if s[0]["M"] == top)


def one_step_launches_any(log):
    """Launch records of the longest step in a log with ``None`` step delimiters (the full-batch eager warm-up step)."""
    steps, cur = [], []
    for r in log:
        if r is None:
            steps.append(cur)
            cur = []
        else:
            cur.append(r)
    return max(steps, key=len) if steps else []


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({type(e).__name__})"


def short_name(name):
    n = name.split("(")[0].replace("void ", "").strip()
    return n.split("rlr::")[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profile_out")
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--bs", type=int, default=256)
    ap.add_argument("--train_size", type=int, default=50000)
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--crop_pad", type=int, default=0, help="training augmentation of the profiled step (engine flag --crop_pad)")
    ap.add_argument("--hflip", action="store_true", help="training augmentation of the profiled step (engine flag --hflip)")
    ap.add_argument("--previous_tiles", action="store_true", help="profile without the one-wave conv tiles (set_conv_one_wave(False))")
    ap.add_argument("--previous_wgrad", action="store_true",
                    help="profile with the weight-gradient kernels the filter-row kernel replaces (set_wgrad_rows(False))")
    ap.add_argument("--bn_reps", type=int, default=20, help="launches per BatchNorm call in the isolation and copy measurements")
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from rlr_b200 import ops
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    from rlr_b200.parallel import init_distributed

    if not torch.cuda.is_available():
        raise SystemExit("profile_step.py measures on the GPU; no CUDA device is visible")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if a.previous_tiles:
        global ONE_WAVE
        ONE_WAVE = False
        ops.ext().set_conv_one_wave(False)
    if a.previous_wgrad:
        global ROWS
        ROWS = False
        ops.ext().set_wgrad_rows(False)
    log = []
    install_recorder(ops.ext(), sms, log)
    wg_log = []
    install_wgrad_recorder(ops.ext(), sms, wg_log)
    bn_log = []
    install_bn_recorder(ops.ext(), bn_log)
    ctx = init_distributed(None, None)
    args = make_args(data="cifar10", model=a.model, num_agents=1, agents_in_flight=0, local_ep=2, bs=a.bs, aggr="avg",
                     robustLR_threshold=0, num_corrupt=0, poison_frac=0.0, agent_frac=1.0, pattern_type="plus",
                     synthetic=a.train_size, synthetic_val=1000, snap=10 ** 9, rounds=10 ** 9, log_dir="", trainer="auto",
                     backend="auto", dtype="bf16", seed=0, crop_pad=a.crop_pad, hflip=a.hflip)
    eng = FLEngine(args, ctx=ctx, verbose=False)
    eng.run_round(1)                                   # captures the step graphs (and records one eager step's launches)
    eng.run_round(2)
    torch.cuda.synchronize()
    launches = one_step_launches(log)
    tr = eng.trainer
    graphs = [g for k, g in tr._graphs.items() if k[0] == a.bs and not k[3]]
    if not graphs:
        raise RuntimeError("no captured full-batch step graph")
    graph = graphs[0]
    for _ in range(3):
        tr.cursor.zero_()
        graph.replay()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(a.replays):
        tr.cursor.zero_()                              # every replay reads the same valid sample indices
        graph.replay()
    ev1.record()
    torch.cuda.synchronize()
    step_ms_unprofiled = ev0.elapsed_time(ev1) / a.replays
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.replays):
            tr.cursor.zero_()
            graph.replay()
        torch.cuda.synchronize()
    kernels = _trace_kernels(prof)
    gpu = gpu_info()
    bn_launches = [r for r in one_step_launches(bn_log)] if any(bn_log) else []
    wg_rows = wgrad_table(one_step_launches_any(wg_log), kernels, a.replays)
    bn_rows = bn_tables(bn_launches, kernels, a.replays, ops.ext(), torch.device("cuda", 0), a.bn_reps) if bn_launches else []
    eng.close()

    per_name = collections.defaultdict(lambda: [0, 0.0])
    per_shape = collections.defaultdict(lambda: [0, 0.0])       # (name, grid) of the GEMM kernel
    for e in kernels:
        nm = short_name(e["name"])
        per_name[nm][0] += 1
        per_name[nm][1] += float(e["dur"])
        if nm.startswith(KERNEL):
            g = tuple(e.get("args", {}).get("grid", [0, 0, 0])[:2])
            per_shape[(nm, g)][0] += 1
            per_shape[(nm, g)][1] += float(e["dur"])
    total_us = sum(v[1] for v in per_name.values()) / a.replays

    # launch records -> traced GEMM kernels, matched by tile width, B layout (template arguments 1 and 3) and grid
    by_grid = collections.defaultdict(list)
    for r in launches:
        by_grid[(r["bn"], r["bmn"], tuple(r["grid"]))].append(r)
    shape_rows = []
    for (nm, g), (cnt, us) in sorted(per_shape.items(), key=lambda kv: -kv[1][1]):
        calls = cnt / a.replays
        targs = [t.strip() for t in nm.split("<", 1)[1].rstrip(">").split(",")]
        recs = by_grid.get((int(targs[0]), targs[2] == "true", g), [])
        flop = sum(r["flop"] for r in recs)
        l2 = sum(r["l2_bytes"] for r in recs)
        kinds = sorted({f'{r["kind"]} M{r["M"]} N{r["N"]} K{r["K"]}' for r in recs})
        us_step = us / a.replays
        shape_rows.append({"kernel": nm, "grid": list(g), "calls_per_step": calls, "us_per_step": us_step,
                           "matched_launches": len(recs), "launches": kinds, "gflop": flop / 1e9, "l2_mb": l2 / 1e6,
                           "tflops": (flop / (us_step * 1e-6) / 1e12) if (recs and us_step and len(recs) == round(calls)) else None,
                           "l2_tb_s": (l2 / (us_step * 1e-6) / 1e12) if (recs and us_step and len(recs) == round(calls)) else None})
    rows = []
    for nm, (cnt, us) in sorted(per_name.items(), key=lambda kv: -kv[1][1]):
        us_step = us / a.replays
        rows.append({"kernel": nm, "calls_per_step": cnt / a.replays, "us_per_step": us_step, "share": us_step / total_us})
    gemm_us = sum(r["us_per_step"] for r in rows if r["kernel"].startswith(KERNEL))
    gemm_flop = sum(r["flop"] for r in launches)
    res = {"gpu": gpu, "model": a.model, "crop_pad": a.crop_pad, "hflip": a.hflip, "replays": a.replays, "batch": a.bs, "step_ms_unprofiled": step_ms_unprofiled,
           "kernel_us_per_step": total_us, "gemm_kernel_us_per_step": gemm_us, "gemm_kernel_share": gemm_us / total_us,
           "gemm_gflop_per_step": gemm_flop / 1e9, "gemm_tflops": gemm_flop / (gemm_us * 1e-6) / 1e12 if gemm_us else None,
           "conv_cluster": os.environ.get("RLR_CONV_CLUSTER", "default"), "one_wave_tiles": ONE_WAVE, "kernels": rows, "gemm_shapes": shape_rows,
           "bn_shapes": bn_rows, "wgrad_rows_kernel": ROWS, "wgrad_shapes": wg_rows}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "profile_step.json"), "w") as f:
        json.dump(res, f, indent=1)
    md = [f"GPU: {gpu} (name, power limit, max SM clock)  ",
          f"Model: {a.model}, crop pad {a.crop_pad}, hflip {a.hflip}, one-wave conv tiles {'on' if ONE_WAVE else 'off'}  ",
          f"Step (batch {a.bs}, graph replay, profiler off): {step_ms_unprofiled:.3f} ms; summed kernel time {total_us / 1e3:.3f} ms.  ",
          f"`{KERNEL}` (all instantiations): {gemm_us:.0f} us/step = {100 * gemm_us / total_us:.1f} % of kernel time, "
          f"{gemm_flop / 1e9:.0f} GFLOP/step, {res['gemm_tflops'] or 0:.0f} TFLOP/s.",
          "", "| kernel | calls/step | us/step | share |", "|---|---:|---:|---:|"]
    md += [f'| `{r["kernel"]}` | {r["calls_per_step"]:.0f} | {r["us_per_step"]:.1f} | {100 * r["share"]:.1f} % |' for r in rows]
    md += ["", f"`{KERNEL}` by launch grid (m-tiles x n-tiles):", "",
           "| instantiation | grid | calls/step | us/step | launches | GFLOP | L2 operand MB | TFLOP/s | L2 TB/s |",
           "|---|---|---:|---:|---|---:|---:|---:|---:|"]
    for r in shape_rows:
        tf = f'{r["tflops"]:.0f}' if r["tflops"] else "-"
        bw = f'{r["l2_tb_s"]:.1f}' if r["l2_tb_s"] else "-"
        md.append(f'| `{r["kernel"].replace(KERNEL, "")}` | {r["grid"][0]}x{r["grid"][1]} | {r["calls_per_step"]:.0f} | '
                  f'{r["us_per_step"]:.1f} | {"; ".join(r["launches"]) or "-"} | {r["gflop"]:.1f} | {r["l2_mb"]:.0f} | {tf} | {bw} |')
    if wg_rows:
        md += ["", f"Weight gradients by launch grid ({'filter-row kernel' if ROWS else 'set_wgrad_rows(False)'}); GFLOP and L2 operand MB "
               "from the launch shapes (every CTA's TMA boxes per k-block):", "",
               "| kernel | grid | calls/step | us/step | launches | GFLOP | L2 operand MB | TFLOP/s | L2 TB/s |",
               "|---|---|---:|---:|---|---:|---:|---:|---:|"]
        for r in wg_rows:
            tf = f'{r["tflops"]:.0f}' if r["tflops"] else "-"
            bw = f'{r["l2_tb_s"]:.1f}' if r["l2_tb_s"] else "-"
            md.append(f'| `{r["kernel"]}` | {"x".join(map(str, r["grid"]))} | {r["calls_per_step"]:.0f} | {r["us_per_step"]:.1f} | '
                      f'{"; ".join(r["launches"]) or "-"} | {r["gflop"]:.1f} | {r["l2_mb"]:.0f} | {tf} | {bw} |')
    if bn_rows:
        fam = sum(r["us_per_step"] for r in bn_rows)
        md += ["", f"BatchNorm family by launch shape (kernel, grid): {fam:.1f} us/step in the step. MB = HBM bytes the pass must move "
               "(bf16 activations; the ordered sums of the partials: time only). *alone* = the same launches replayed one at a time "
               "outside the graph; *copy* = a device-to-device copy of the same bytes in this session.", "",
               "| kernel | grid | pass | calls/step | us/step | launches | MB | TB/s | alone us | alone TB/s | copy us | copy TB/s |",
               "|---|---:|---|---:|---:|---|---:|---:|---:|---:|---:|---:|"]
        f1 = lambda v, d=1: f"{v:.{d}f}" if v else "-"  # noqa: E731
        for r in bn_rows:
            md.append(f'| `{r["kernel"]}` | {r["grid"]} | {r["pass"]} | {r["calls_per_step"]:.0f} | {r["us_per_step"]:.1f} | '
                      f'{"; ".join(r["launches"])} | {f1(r["mb"], 0)} | {f1(r["tb_s"], 2)} | {r["iso_us"]:.1f} | {f1(r["iso_tb_s"], 2)} | '
                      f'{f1(r["copy_us"])} | {f1(r["copy_tb_s"], 2)} |')
        by_pass = collections.defaultdict(lambda: [0.0, 0.0, 0.0])
        for r in bn_rows:
            by_pass[r["pass"]][0] += r["us_per_step"]
            by_pass[r["pass"]][1] += r["iso_us"]
            by_pass[r["pass"]][2] += r["mb"]
        md += ["", "| pass | us/step in the step | us/step alone | MB/step | TB/s in the step | TB/s alone |", "|---|---:|---:|---:|---:|---:|"]
        for p, (us, iso_us, mb) in by_pass.items():
            md.append(f"| {p} | {us:.1f} | {iso_us:.1f} | {mb:.0f} | {f1(mb / us if mb else 0, 2)} | {f1(mb / iso_us if mb else 0, 2)} |")
    with open(os.path.join(a.out, "profile_step.md"), "w") as f:
        f.write("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
