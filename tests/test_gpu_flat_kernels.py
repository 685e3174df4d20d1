"""GPU: the flat-vector kernels against fp64 statements at sizes that make every grid-stride loop take several sweeps of its capped grid.

* the fused server step (``fused_aggregate_kernel`` / ``fused_aggregate_median_kernel``) on every path against ``ops.aggregate_oracle``,
* the local optimizer (``sqnorm`` / ``sgd_step`` / ``pgd_project`` behind ``ops.FlatSGD``) against an fp64 statement of src/agent.py,
* the loss and evaluation reductions (``softmax_xent`` / ``eval_metrics``) against fp64 ``log_softmax``.

Each launcher caps its grid at a few CTAs per SM, so a coordinate past the first ``sweep(...)`` coordinates is handled by a second trip
through the loop.  Sizes are derived from the device's SM count and the launcher rules, not from one GPU model."""
import math

import numpy as np
import pytest
import torch

import rlr_b200  # noqa: F401
from rlr_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24                 # unit roundoff of fp32
ULP = 2.0 ** -23               # one fp32 ulp, relative to the value


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def agg_sweep(mode, K):
    """Coordinates one sweep of ``launch_fused_aggregate``'s capped grid covers (ops/csrc/aggregate.cu)."""
    sms = _sms()
    if mode != "comed" or K <= 8:
        return sms * 8 * 256 * 4        # vector path: 8 CTAs / SM x 256 threads x 4 coordinates
    if K <= 64:
        return sms * 2 * 256            # Batcher networks: 2 CTAs / SM x 256 threads, one coordinate each
    if K <= 320:
        return sms * 128                # shared-memory bisection: 1 CTA / SM x 128 threads
    return sms * 2 * 128                # re-read bisection: 2 CTAs / SM x 128 threads


def flat_sweep():
    """Coordinates one sweep of ``sqnorm`` / ``sgd_step`` / ``pgd_project`` covers (ops/csrc/elementwise.cu: 4 CTAs / SM x 256 x 4)."""
    return _sms() * 4 * 256 * 4


def _sizes(S, sweeps):
    """``sweeps`` full sweeps plus a remainder that is a multiple of 4 but not of 32, and a split point (n_vote / n_pgd) that is a
    multiple of 4 inside the last full sweep and inside a 32-coordinate group."""
    n = sweeps * S + (S // 2) // 8 * 8 + 4
    split = (sweeps - 1) * S + (S // 3) // 32 * 32 + 12
    assert n % 4 == 0 and n % 32 and split % 4 == 0 and split % 32 and (sweeps - 1) * S < split < sweeps * S
    return n, split


# =====================================================================================================================================
# A. server step
# =====================================================================================================================================
def _agents(g, K, seed):
    """K participants' parameters on the device: g plus a 0.1-scale update with ~20% exact zeros (sign votes of 0, median ties)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    W = torch.empty(K, g.numel(), device=DEV)
    for k in range(K):
        W[k] = g + 0.1 * torch.randn(g.numel(), generator=gen, device=DEV) * (torch.rand(g.numel(), generator=gen, device=DEV) > 0.2)
    return list(W)


def _oracle(g, ws, wt, mode, theta, lr, n_vote, opt=None):
    """``ops.aggregate_oracle`` over coordinate chunks on the CPU (the statement is per coordinate; n_vote is shifted per chunk), so
    K x n fp64 values never exist at once.  ``opt``: a full-length CPU ``ServerOptState``, updated in place through per-chunk views."""
    n, K = g.numel(), len(ws)
    step = max(1024, (1 << 22) // K) // 4 * 4
    out = torch.empty(n, dtype=torch.float32)
    flips = 0
    for lo in range(0, n, step):
        hi = min(n, lo + step)
        part = None
        if opt is not None:
            part = ops.ServerOptState(opt.kind, 0, opt.beta1, opt.beta2, opt.tau)
            part.m = opt.m[lo:hi]
            part.v = opt.v[lo:hi] if opt.v is not None else None
        rows = torch.stack([w[lo:hi] for w in ws]).cpu()
        o, f = ops.aggregate_oracle(g[lo:hi].cpu(), list(rows), wt, mode, theta, lr, None, min(max(n_vote - lo, 0), hi - lo),
                                    opt=part)
        out[lo:hi] = o
        flips += f
    return out, flips


def _theta(K):
    return max(1, (K + 2) // 3)


def _lr(mode):
    return 0.5 if mode == "sign" else 1.0


# avg / sign: always the vector path.  comed: vector path (K <= 8), Batcher networks (8 < K <= 64), shared-memory bisection
# (64 < K <= 320), re-read bisection (K > 320) -- each at its two ends.
AGG_CASES = [("avg", 1), ("avg", 5), ("avg", 40), ("sign", 1), ("sign", 5), ("sign", 40),
             ("comed", 3), ("comed", 8), ("comed", 12), ("comed", 64), ("comed", 100), ("comed", 320), ("comed", 321), ("comed", 1024)]
IN_PLACE = [("avg", 5), ("sign", 40), ("comed", 8), ("comed", 64), ("comed", 100), ("comed", 1024)]   # one per kernel path


@pytest.mark.parametrize("mode,K,in_place", [(m, K, False) for m, K in AGG_CASES] + [(m, K, True) for m, K in IN_PLACE])
def test_server_step_over_several_sweeps_matches_oracle(mode, K, in_place):
    n, n_vote = _sizes(agg_sweep(mode, K), 3)
    assert K * n * 4 <= 1.6e9
    seed = 1000 * K + len(mode) + in_place
    g = torch.randn(n, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)
    ws = _agents(g, K, seed + 1)
    wt = [float(100 + 13 * k) for k in range(K)]
    ref, nflip = _oracle(g, ws, wt, mode, _theta(K), _lr(mode), n_vote)
    flipped = torch.zeros(1, dtype=torch.int64, device=DEV)
    shadow = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    out = None if in_place else torch.empty_like(g)
    res = ops.fused_aggregate(g, ws, wt, mode, _theta(K), _lr(mode), n_vote=n_vote, out=out, out_bf16=shadow, flipped=flipped)
    assert (res.data_ptr() == g.data_ptr()) == in_place
    torch.testing.assert_close(res.cpu(), ref, atol=1e-6, rtol=1e-6)
    assert int(flipped.item()) == nflip and nflip > 0
    assert torch.equal(shadow, res.bfloat16())


@pytest.mark.parametrize("mode,K", [("avg", 5), ("comed", 12), ("comed", 100), ("comed", 321)])
def test_server_adam_state_over_several_sweeps_matches_oracle(mode, K):
    """Three rounds of FedAdam on each path family: the weights and the carried fp32 state m, v beyond the first sweep."""
    n, n_vote = _sizes(agg_sweep(mode, K), 3)
    seed = 77 * K
    g = torch.randn(n, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)
    wt = [float(100 + 13 * k) for k in range(K)]
    ref_opt = ops.ServerOptState("adam", n, 0.9, 0.99, 1e-3)
    dev_opt = ops.ServerOptState("adam", n, 0.9, 0.99, 1e-3, device=DEV)
    for rnd in range(3):
        ws = _agents(g, K, seed + 1 + rnd)
        ref, nflip = _oracle(g, ws, wt, mode, _theta(K), 0.5, n_vote, ref_opt)
        flipped = torch.zeros(1, dtype=torch.int64, device=DEV)
        shadow = torch.empty(n, dtype=torch.bfloat16, device=DEV)
        out = torch.empty_like(g)
        ops.fused_aggregate(g, ws, wt, mode, _theta(K), 0.5, n_vote=n_vote, out=out, out_bf16=shadow, flipped=flipped, opt=dev_opt)
        torch.testing.assert_close(out.cpu(), ref, atol=1e-6, rtol=1e-6)
        torch.testing.assert_close(dev_opt.m.cpu(), ref_opt.m, atol=1e-6, rtol=1e-6)
        torch.testing.assert_close(dev_opt.v.cpu(), ref_opt.v, atol=1e-6, rtol=1e-6)
        assert int(flipped.item()) == nflip
        assert torch.equal(shadow, out.bfloat16())
        assert torch.all(dev_opt.m[n_vote:] == 0)
        g = out
        del ws


# =====================================================================================================================================
# B. local optimizer
# =====================================================================================================================================
def _f32(x):
    return float(np.float32(x))


# hyper-parameters at their fp32 values: the precision the kernels receive them in, so the statement and the kernel share operands
LR, MU, MAX_NORM = _f32(0.1), _f32(0.9), 10.0
PGD_CLIP = {"off": 0.0, "inside": 64.0, "projected": 0.0625}


def _sgd_statement(w, g, m, w0, clip, k, w_in=None):
    """One ``FlatSGD`` step in fp64 (src/agent.py:41-60), from the kernel's own previous state, and a per-coordinate bound on the error of
    the fp32 kernels.  Returns ``(w', m', ||g||^2, ||w' - w0||^2 or None, bound_w, bound_m, rho)``.

    Error bound, first order in U = 2^-24 (each fp32 rounding moves a result by at most U of its magnitude):
      coef = min(1, c / (||g|| + 1e-6)): ||g||^2 from fp32 squares and pair sums (<= 2U relative), sqrt rounded to fp32, + 1e-6f, one
        division: <= 4U relative.
      m' = mu m + coef g: two products and a sum (or one fma): |dm| <= U|mu m| + 5U|coef g| + U|m'|      <= 8U (|mu m| + |coef g|) = Em
      w' = w - lr m': lr Em, plus the product and the difference:                                     Ew = lr Em + U (lr|m'| + |w'|)
      PGD, d = w' - w0 over [0, k), r = ||d||: the kernel sums its own d, so |dr| <= ||Ew|| (triangle inequality) + U r (difference)
        + U r (fp32 squares and pair sums: 2U on r^2) + U r (sqrt to fp32):  rho = ||Ew|| / r + 3U relative.
      projected: inv = 1 / (r / clip) adds two roundings; w'' = w0 + d inv rounds the difference, the product and the sum:
        Ep = inv (Ew + U|d|) + (rho + 2U) inv |d| + U (inv |d| + |w''|).
    The first-step variant (``w_in``) reads w_in and zero momentum on [0, k) and leaves w[k:] alone (bound 0 there)."""
    w, g, m = w.double(), g.double(), m.double()
    gsq = float((g * g).sum())
    coef = min(1.0, MAX_NORM / (math.sqrt(gsq) + 1e-6))
    if w_in is None:
        a, b = MU * m, coef * g
        m1 = a + b
        w1 = w - LR * m1
    else:
        a, b = torch.zeros_like(g), coef * g
        b[k:] = 0
        m1 = b.clone()
        w1 = w.clone()
        w1[:k] = w_in[:k].double() - LR * m1[:k]
    em = 8 * U * (a.abs() + b.abs())
    ew = LR * em + U * (LR * m1.abs() + w1.abs())
    if w_in is not None:
        ew[k:] = 0
    dsq, rho = None, 0.0
    if clip > 0:
        d = w1[:k] - w0[:k].double()
        dsq = float((d * d).sum())
        r = math.sqrt(dsq)
        rho = float(ew[:k].norm()) / r + 3 * U
        assert r > 1.1 * clip or r < clip / 1.1, "keep the projection decision far from its edge"
        denom = max(1.0, r / clip)
        if denom > 1.0:
            inv = 1.0 / denom
            w1[:k] = w0[:k].double() + d * inv
            ew[:k] = inv * (ew[:k] + U * d.abs()) + (rho + 2 * U) * inv * d.abs() + U * (inv * d.abs() + w1[:k].abs())
    return w1, m1, gsq, dsq, ew, em, rho


def _check_step(opt, w, m, shadow, ref, n, k, shadow_upto=None):
    w1, m1, gsq, dsq, ew, em, rho = ref
    err_w = (w.cpu().double() - w1).abs()
    err_m = (m.cpu().double() - m1).abs()
    assert bool((err_w <= ew).all()), f"w: worst excess {float((err_w - ew).max()):.3e} at {int((err_w - ew).argmax())}"
    assert bool((err_m <= em).all()), f"m: worst excess {float((err_m - em).max()):.3e} at {int((err_m - em).argmax())}"
    # ||g||^2: fp32 squares and pair sums (2U relative), fp64 accumulation over n / 4 terms
    n0 = float(opt.norms[0])
    assert abs(n0 - gsq) <= (2 * U + n * 2.0 ** -53) * gsq, (n0, gsq)
    if dsq is not None:
        n1 = float(opt.norms[1])
        assert abs(n1 - dsq) <= (2 * rho + rho * rho) * dsq, (n1, dsq)
    s = n if shadow_upto is None else shadow_upto
    assert torch.equal(shadow[:s], w[:s].bfloat16())


@pytest.mark.parametrize("pgd", ["off", "inside", "projected"])
@pytest.mark.parametrize("clipped", [True, False])
def test_flat_sgd_over_several_sweeps_matches_fp64_statement(clipped, pgd):
    n, k = _sizes(flat_sweep(), 2)
    gen = torch.Generator(device=DEV).manual_seed(11 + 2 * clipped + len(pgd))
    w0 = torch.randn(n, generator=gen, device=DEV)
    w = w0.clone()
    m = 1e-3 * torch.randn(n, generator=gen, device=DEV)           # momentum carried from earlier steps of the round
    shadow = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
    opt = ops.FlatSGD(n, DEV, LR, MU, MAX_NORM, PGD_CLIP[pgd], n_pgd=k)
    for _ in range(3):
        # ||g|| ~ 30 sqrt(n) >> 10 (clipped) or ~ 1e-3 sqrt(n) << 10 (not clipped): the clip decision is the same in fp32 and fp64
        g = torch.randn(n, generator=gen, device=DEV) * (30.0 if clipped else 1e-3)
        ref = _sgd_statement(w.cpu(), g.cpu(), m.cpu(), w0.cpu(), PGD_CLIP[pgd], k)
        opt.step(w, g, m, w0=w0 if pgd != "off" else None, w_bf16=shadow)
        _check_step(opt, w, m, shadow, ref, n, k)


@pytest.mark.parametrize("pgd", ["off", "projected"])
def test_flat_sgd_first_step_variant_matches_fp64_statement(pgd):
    """``FlatSGD.step(..., w_in=...)``: parameters come from w_in and the momentum counts as 0 on [0, n_pgd) -- the buffers' old
    contents there are NaN and must never be read -- while w[n_pgd:] (BatchNorm running statistics) is kept bit for bit."""
    n, k = _sizes(flat_sweep(), 2)
    gen = torch.Generator(device=DEV).manual_seed(5 + len(pgd))
    w_in = torch.randn(n, generator=gen, device=DEV)
    w = torch.full((n,), float("nan"), device=DEV)
    w[k:] = 7.0 + torch.arange(n - k, device=DEV, dtype=torch.float32) * 1e-3
    tail = w[k:].clone()
    m = torch.full((n,), float("nan"), device=DEV)
    shadow = torch.full((n,), float("nan"), dtype=torch.bfloat16, device=DEV)
    g = torch.randn(n, generator=gen, device=DEV) * 30.0
    opt = ops.FlatSGD(n, DEV, LR, MU, MAX_NORM, PGD_CLIP[pgd], n_pgd=k)
    ref = _sgd_statement(w.cpu(), g.cpu(), torch.zeros(n), w_in.cpu(), PGD_CLIP[pgd], k, w_in=w_in.cpu())
    opt.step(w, g, m, w0=w_in if pgd != "off" else None, w_bf16=shadow, w_in=w_in)
    assert torch.equal(w[k:], tail)
    assert bool((m[k:] == 0).all())
    # the shadow is written where the step writes w: everywhere by the projection pass, on [0, n_pgd) by the step alone
    _check_step(opt, w, m, shadow, ref, n, k, shadow_upto=None if pgd != "off" else k)


def test_pgd_step_is_bitwise_reproducible():
    """The PGD radius is a fixed-order sum: identical steps give identical bits in w, m, the shadow and both norms."""
    n, k = _sizes(flat_sweep(), 2)
    gen = torch.Generator(device=DEV).manual_seed(3)
    w0 = torch.randn(n, generator=gen, device=DEV)
    w_start = w0 + 1e-3 * torch.randn(n, generator=gen, device=DEV)
    m_start = 1e-3 * torch.randn(n, generator=gen, device=DEV)
    g = torch.randn(n, generator=gen, device=DEV) * 30.0
    runs = []
    for _ in range(4):
        w, m = w_start.clone(), m_start.clone()
        shadow = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
        opt = ops.FlatSGD(n, DEV, LR, MU, MAX_NORM, PGD_CLIP["projected"], n_pgd=k)
        opt.step(w, g, m, w0=w0, w_bf16=shadow)
        runs.append((w, m, shadow, opt.norms.clone()))
    assert float(runs[0][3][1]) > PGD_CLIP["projected"] ** 2
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)


# =====================================================================================================================================
# C. loss and evaluation
# =====================================================================================================================================
def _logits(B, C, dtype, seed):
    """``randn * 3`` logits with, by row, the label logit 20 / 80 / 200 below the largest other logit, the label tied with another
    class at the top, or (C > 2) two other classes tied at the top."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, generator=gen) * 3
    y = torch.randint(0, C, (B,), generator=gen)
    r = torch.arange(B)
    kind = (5 * r + 2) % 6
    others = x.clone()
    others[r, y] = -math.inf
    top = others.max(1).values
    for kd, gap in ((1, 20.0), (2, 80.0), (3, 200.0)):
        s = kind == kd
        x[r[s], y[s]] = top[s] - gap
    t = x.max(1).values + 1.0
    c1 = (y + 1 + r % max(1, C - 1)) % C                              # != y
    s = kind == 4
    x[r[s], y[s]] = t[s]
    x[r[s], c1[s]] = t[s]
    if C > 2:
        c2 = (c1 + 1) % C
        c2 = torch.where(c2 == y, (c2 + 1) % C, c2)
        s = kind == 5
        x[r[s], c1[s]] = t[s]
        x[r[s], c2[s]] = t[s]
    return x.to(dtype), y


P_SWITCH = 2.0 ** -64         # softmax_xent: -log p_y at or above this label probability, log(se) - (x_y - mx) below it


def _row_stats(x, y, train):
    """fp64 per-row statement (loss, softmax) and a bound on the error of one row's fp32 loss.
    exp(x_c - mx): the fp32 difference is rounded (U |a_c| relative on the exponential), then __expf (training: 2 + floor(1.173 |a_c|)
    ulps) or expf (evaluation: 2 ulps); flushed results are off by < 2^-126.  A sequential fp32 sum of C terms adds (C - 1) U.
    log(se) - (x_y - mx) (evaluation; training below P_SWITCH): logf adds 1 ulp of log(se), then the label's gap (U |gap|) and the
    final difference (U |loss|) round.  -log(p_y + 1e-30) (training at or above P_SWITCH): p_y = t_y * fp32(1 / se) is off by
    e_y + rel_se + 2U relative, the 1e-30 guard adds 1e-30 / p_y and a rounding, and __logf adds 2^-21.41 absolute on [0.5, 2] and
    3 ulps elsewhere."""
    xd = x.double()
    B, C = xd.shape
    r = torch.arange(B)
    mx = xd.max(1).values
    a = (xd - mx[:, None]).abs()
    lse = torch.logsumexp(xd, 1)
    p = torch.exp(xd - lse[:, None])
    nll = lse - xd[r, y]
    e = U * a + ((2 + 1.173 * a) if train else 2.0) * ULP
    rel_se = (p * e).sum(1) + (C - 1) * U + C * 2.0 ** -126
    row = rel_se + ULP * (lse - mx) + U * (mx - xd[r, y]) + U * nll
    if train:
        py = p[r, y]
        assert not bool(((py > P_SWITCH / 4) & (py < P_SWITCH * 4)).any()), "keep every row's branch clear of the switch"
        direct = e[r, y] + rel_se + 3 * U + 1e-30 / py + torch.where(py >= 0.5, torch.full_like(py, 2.0 ** -21.41), 3 * ULP * nll)
        row = torch.where(py >= P_SWITCH, direct, row)
    return nll, p, e, rel_se, row


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("B", [1, 127, 128, 129, 1000, 4097])
@pytest.mark.parametrize("C", [2, 10, 32])
def test_softmax_xent_and_eval_metrics_match_fp64_log_softmax(C, B, dtype):
    x, y = _logits(B, C, dtype, seed=C * 10007 + B)
    xd_, yd = x.to(DEV), y.to(DEV)
    pred = x.double().argmax(1)                                       # the first maximal index, as the kernels pick it
    nblocks = (B + 127) // 128

    # training loss: fp32 per-row losses summed in fp32 (128-row block trees, then the blocks in order)
    nll, p, e, rel_se, row = _row_stats(x, y, train=True)
    loss_sum = torch.zeros(1, dtype=torch.float32, device=DEV)
    correct = torch.zeros(1, dtype=torch.int32, device=DEV)
    _, dl = ops.softmax_xent(xd_, yd, True, loss_sum, correct)
    tol = float(row.sum()) + (10 + nblocks) * U * float(nll.sum())
    assert abs(float(loss_sum) - float(nll.sum())) <= tol, (float(loss_sum), float(nll.sum()), tol)
    assert int(correct) == int((pred == y).sum())

    # dlogits = (softmax - onehot) / B: p_c = fl(t_c * fl(1 / se)) is off by p_c (e_c + rel_se + 2U) (+ 2^-126 when flushed); then the
    # difference, the scale (itself fp32(1 / B)) and the product round; a bf16 output rounds once more (2^-8 relative); results below
    # the smallest normal (2^-126) may lose that much absolutely
    onehot = torch.nn.functional.one_hot(y, C).double()
    dl_ref = (p - onehot) / B
    dp = p * (e + rel_se[:, None] + 2 * U) + 2.0 ** -126
    err = (dp + U * (p - onehot).abs()) / B * (1 + U) + 2 * U * dl_ref.abs()
    r_out = 2.0 ** -8 if dtype == torch.bfloat16 else 0.0
    bound = err * (1 + r_out) + r_out * dl_ref.abs() + 2.0 ** -126
    diff = (dl.cpu().double() - dl_ref).abs()
    assert dl.dtype == dtype and bool((diff <= bound).all()), f"dlogits: worst excess {float((diff - bound).max()):.3e}"

    # evaluation: fp32 per-row losses (expf / logf) summed in fp64; confusion[true, pred] exact
    nll_e, _, _, _, row_e = _row_stats(x, y, train=False)
    ls = torch.zeros(1, dtype=torch.float64, device=DEV)
    conf = torch.zeros(C, C, dtype=torch.int64, device=DEV)
    ops.eval_metrics(xd_, yd, ls, conf)
    tol_e = float(row_e.sum()) + B * 2.0 ** -52 * float(nll_e.sum())
    assert abs(float(ls) - float(nll_e.sum())) <= tol_e, (float(ls), float(nll_e.sum()), tol_e)
    conf_ref = torch.zeros(C, C, dtype=torch.int64).index_put_((y, pred), torch.ones(B, dtype=torch.int64), accumulate=True)
    assert torch.equal(conf.cpu(), conf_ref)


def test_softmax_xent_rejects_more_than_32_classes():
    with pytest.raises(RuntimeError):
        ops.softmax_xent(torch.zeros(4, 33, device=DEV), torch.zeros(4, dtype=torch.int64, device=DEV))


def test_eval_metrics_loss_is_bitwise_reproducible():
    """33 blocks of 128 rows: their loss partials are added in block order, so repeated calls give the same bits."""
    x, y = _logits(4097, 10, torch.float32, seed=9)
    x, y = x.to(DEV), y.to(DEV)
    sums = []
    for _ in range(4):
        ls = torch.zeros(1, dtype=torch.float64, device=DEV)
        ops.eval_metrics(x, y, ls, torch.zeros(10, 10, dtype=torch.int64, device=DEV))
        sums.append(ls)
    for s in sums[1:]:
        assert torch.equal(s, sums[0])
