"""fp64 statements of the memory-bound layer kernels (BatchNorm, GroupNorm, ReLU backward, max / average pooling, dropout, and the
dropout fused into the pooling kernel and the linear-layer epilogues) and a checker that judges each output element against them.

Each kernel is judged in two stages, so that the error of a statistic cannot hide an error in the per-element arithmetic:

* **Statistics against fp64 truth.**  Stored sums (BatchNorm ``stats`` / ``dsum``, GroupNorm ``dgamma`` / ``dbeta``) are compared
  with the exact sums of their terms under the fp32 summation bound of ``gemm_oracle.check_stats``,
  ``KAPPA_STATS * 2^-24 * sqrt(M) * sum |v|`` (plus a few roundings per term where a term is itself a product).  The finalised
  statistics (``mean_rstd``, the running mean and the unbiased running variance with its ``count > 1`` guard) are compared with
  the fp64 function of sums known to within ``d1`` / ``d2``: once of the kernel's OWN stored sums (``d`` = their slot-summation
  error: a few ulps, sharp enough to see a biased variance at 262,144 rows) and once of the exact sums (``d`` = the summation
  bound).  The bound is propagated through ``var = s2/M - mean^2`` with the cancellation term ``2 |mean| d1 / M`` stated explicitly,
  and through ``rsqrt`` as the exact image of the interval ``var +- dvar``.
* **Per-element outputs given the kernel's own stored statistics.**  ``y``, ``dx`` and the average-pool output are the fp64 value
  of the stated expression, pushed through the kernel's monotone epilogue (ReLU, bf16 round-to-nearest-even); the interval allows
  ``KAPPA_EW`` fp32 roundings of every term's magnitude (the kernels are built without fast-math, with FMA contraction).  GroupNorm's
  ``dx`` uses in-kernel group sums that are not stored: its interval also carries their summation bound.  As in
  ``gemm_oracle``, the fraction of bf16 outputs that differ from the rounded statement must not exceed ``RHO`` (catches rounding-
  mode faults that stay within one ulp).
* **Exact statements** (``torch.equal``): the max-pool forward (value and arg-max: the first maximum in window order, floor mode)
  and backward (odd last row / column zeroed, the producer's ReLU read off the pooled output, fused dropout), ``relu_bwd``
  (``rn_bf16(fp32(dy * scale))`` where ``y > 0``), ``dres`` (the masked ``dy``), the average-pool backward (``rn_bf16(dy / HW)``),
  the stand-alone dropout kernels and their mask tensor, and the keep-mask of every fused-dropout output.

The dropout keep-mask (common.cuh ``dropout_keep8``) is a pure function of the flat index ``e`` of the OUTPUT element (the pooled
element for the max-pool, ``row * ldc + col`` for the GEMM epilogue, the flat index for split-K and stand-alone dropout)::

    u = philox4x32(ctr = e // 8, stream = ((step << 20) mod 2^64) ^ node, key = seed)
    keep = ((u[(e % 8) // 2] >> (16 * (e % 2))) & 0xFFFF) >= uint32(float32(p) * 65536)

Calibration (H100 80GB HBM3 at 700 W; the 177 distinct layer-kernel calls of one training step of the ten zoo models at batch 256 / 96 /
80 with dropout on, each replayed alone, plus the edge cases of tests/test_gpu_layer_oracle.py).  Largest kappa needed: elementwise
outputs 1.94 (BatchNorm dx at 6144 x 256; BatchNorm y 0.87, GroupNorm y 0.94, GroupNorm dx 0.23, BatchNorm dgamma / dbeta 0.75);
finalised statistics 1.24 against the kernel's own sums, 0.87 against the exact ones, GroupNorm mean / rstd 0.44; BatchNorm statistics
sums 0.84 of the check_stats bound (the 256-slot chain of channel_stats at 257 rows), backward sums 0.18, GroupNorm dgamma / dbeta
0.18; linear layers with fused dropout 0.012 of gemm_oracle's bound.  Largest mismatch fraction 0.71 % (BatchNorm dx).  Every exact
statement held bit for bit.  ``KAPPA_EW``, ``KAPPA_FIN``, ``KAPPA_CSTATS`` and ``RHO`` keep a margin of 4x over these.

BatchNorm's one-pass variance far from zero mean, measured on the same card (65,536 rows): the output stays within 0.5 bf16 ulp of the
fp64 truth up to |mean| / std = 8, and within 0.512 ulp at 32, so no kernel change is needed at any ratio up to 32.
"""
from __future__ import annotations

import math
from typing import NamedTuple

import numpy as np
import torch

from gemm_oracle import GUARD, KAPPA_STATS, U, Result, Statement, check, check_stats, gemm_statement, guard_intact, guarded, rn_bf16  # noqa: F401

KAPPA_EW = 8.0          # fp32 roundings allowed per term magnitude of an elementwise expression (see the calibration above)
KAPPA_FIN = 5.0         # the same for the finalised statistics (mean / rstd / running statistics)
KAPPA_CSTATS = 3.5      # check_stats constant of the BatchNorm statistics pass (channel_stats: a 256-long fp32 chain over row slots)
RHO = 0.03              # largest fraction of bf16 outputs allowed to differ from the rounded statement
RHO_MIN = 4096          # ... judged on outputs of at least this many elements
_M64 = 2 ** 64 - 1


def _d(t):
    return t.double()


# =====================================================================================================================
# dropout keep-mask
# =====================================================================================================================
class Drop(NamedTuple):
    """A dropout layer's parameters: rate, Philox key, value of the device step counter, node id."""
    p: float
    seed: int
    step: int
    node: int

    @property
    def thr(self) -> int:
        return int(np.float32(self.p) * np.float32(65536.0))

    def scale(self, kind="f32") -> float:
        """1/(1-p) as the kernel computes it: in fp32 (pooling and stand-alone dropout kernels), or in fp64 rounded to fp32 (the GEMM
        epilogues and relu_bwd, which receive it from the host)."""
        if kind == "f32":
            return float(np.float32(1.0) / (np.float32(1.0) - np.float32(self.p)))
        return float(np.float32(1.0 / (1.0 - self.p)))


def dropout_bits(n: int, d: Drop) -> np.ndarray:
    """The 16 random bits of flat elements 0 .. n-1."""
    q = np.arange((n + 7) // 8, dtype=np.uint64)
    stream = ((int(d.step) << 20) & _M64) ^ int(d.node)
    u = np.stack(ops_philox()(q, stream, d.seed))          # [4, n/8] uint32
    e = np.arange(n)
    w = u[(e % 8) // 2, e // 8].astype(np.uint32)
    return (w >> (16 * (e % 2)).astype(np.uint32)) & np.uint32(0xFFFF)


def dropout_keep(shape, d: Drop, device="cpu") -> torch.Tensor:
    """Boolean keep-mask of a tensor of ``shape`` (flat element index = the kernel's output index)."""
    n = math.prod(shape)
    return torch.from_numpy(dropout_bits(n, d) >= d.thr).reshape(shape).to(device)


def ops_philox():
    from rlr_b200 import ops
    return ops.philox4x32


# =====================================================================================================================
# stage 1: sums against fp64 truth
# =====================================================================================================================
def check_sums(name, got, terms, extra=None, kappa=KAPPA_STATS, rounding=0.0) -> Result:
    """``got`` ([slots, k, C] fp32 partials, or [k, C]) against the exact column sums of ``terms`` ([k, M, C] fp64) (+ ``extra`` [k, C],
    an old value the kernel added into).  Bound: fp32 summation of M terms, ``kappa * 2^-24 * sqrt(M) * sum |v|``, plus ``rounding``
    fp32 roundings of every term (terms that are products computed in fp32)."""
    k, M, C = terms.shape
    want = terms.sum(1)
    mag = terms.abs().sum(1)
    if extra is not None:
        want, mag = want + _d(extra), mag + _d(extra).abs()
    g = _d(got).reshape(-1, k, C).sum(0)
    bound = U * (math.sqrt(M) + 1) * mag                 # + 1: the add of the slot partials / of the old value
    err = ((g - want).abs() - rounding * U * mag).clamp_min(0)      # the per-term roundings are a fixed allowance
    r = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
    r = torch.where(torch.isnan(g), torch.full_like(r, math.inf), r)
    kmax = float(r.max()) if r.numel() else 0.0
    worst = tuple(int(i) for i in torch.unravel_index(r.argmax(), r.shape)) if r.numel() else ()
    return Result(name, kmax, 0.0, worst, kmax <= kappa)


def check_value(name, got, want, unit, phi=lambda a: a, kappa=KAPPA_EW, rho=RHO) -> Result:
    """Per element, the smallest kappa with ``phi(want - kappa unit) <= got <= phi(want + kappa unit)`` (``phi`` monotone; an element
    with ``unit == 0`` must equal ``phi(want)``); bf16 outputs of at least ``RHO_MIN`` elements also face the mismatch fraction ``rho``
    (below that one element is more than the fraction).  Elements whose statement is within 2^10 units of zero are left out of the
    fraction: there the result is cancellation, rounding noise by construction."""
    want, unit = _d(want), _d(unit).expand_as(want)
    r = check(name, got, Statement(want, (unit / U) ** 2, 1), phi, kappa, 1.0)
    if got.dtype != torch.bfloat16:
        return r
    sharp = want.abs() > 1024 * unit
    mism = float(((got.float() != phi(want.float())) & sharp).double().sum() / sharp.double().sum().clamp_min(1))
    ok = r.ok and (mism <= rho or int(sharp.sum()) < RHO_MIN)
    return Result(name, r.kappa, mism, r.worst, ok)


# =====================================================================================================================
# BatchNorm
# =====================================================================================================================
class Fin(NamedTuple):
    mean: torch.Tensor
    rstd: torch.Tensor
    rm: torch.Tensor
    rv: torch.Tensor
    u_mean: torch.Tensor
    u_rstd: torch.Tensor
    u_rm: torch.Tensor
    u_rv: torch.Tensor


def f32(v: float) -> float:
    return float(np.float32(v))


def rsqrt_interval(v, dv, eps):
    """(rstd, unit): rsqrt(v + eps) and the largest distance to rsqrt(v' + eps) for v' in [v - dv, v + dv] (v' >= 0)."""
    r = (v + eps).rsqrt()
    lo = (v + dv + eps).rsqrt()
    hi = ((v - dv).clamp_min(0) + eps).rsqrt()
    return r, torch.maximum(hi - r, r - lo)


def bn_finalize(s1, s2, count, eps, momentum, rm, rv, d1, d2) -> Fin:
    """fp64 statement of the training finalize of bn_apply (fin.mode 1) from sums ``s1`` / ``s2`` known to within ``d1`` / ``d2``:
    mean = s1/M, var = max(s2/M - mean^2, 0) (biased, one pass), rstd = rsqrt(var + eps), running mean / variance updated with
    momentum, the variance unbiased by M/(M-1) when M > 1.  Units: the propagated sum errors plus KAPPA_FIN-scaled fp32 roundings."""
    M = float(count)
    eps, mom = f32(eps), f32(momentum)
    s1, s2, rm, rv = _d(s1), _d(s2), _d(rm), _d(rv)
    mean = s1 / M
    ex2 = s2 / M
    var = (ex2 - mean * mean).clamp_min(0)
    u_mean = _d(d1) / M + U * mean.abs()
    # var = s2/M - mean^2: the sum errors, the cancellation term 2 |mean| d1 / M, and the roundings of s2/M, mean^2 and the difference
    dvar = _d(d2) / M + 2 * mean.abs() * _d(d1) / M + (_d(d1) / M) ** 2 + U * (ex2 + mean * mean + var)
    rstd, u_r = rsqrt_interval(var, dvar, eps)
    u_rstd = u_r + U * rstd                                    # the add of eps and rsqrtf (2 ulp) are in the KAPPA_FIN roundings
    unb = var * M / (M - 1) if M > 1 else var
    f = M / (M - 1) if M > 1 else 1.0
    rm1 = (1 - mom) * rm + mom * mean
    rv1 = (1 - mom) * rv + mom * unb
    u_rm = mom * u_mean + U * ((1 - mom) * rm.abs() + mom * mean.abs())
    u_rv = mom * dvar * f + U * ((1 - mom) * rv.abs() + mom * unb)
    return Fin(mean, rstd, rm1, rv1, u_mean, u_rstd, u_rm, u_rv)


def bn_eval(rm, rv, eps) -> Fin:
    """Evaluation (fin.mode 2): mean = running mean, rstd = rsqrt(running var + eps); nothing is updated."""
    rm, rv = _d(rm), _d(rv)
    rstd = (rv + f32(eps)).rsqrt()
    z = torch.zeros_like(rm)
    return Fin(rm, rstd, rm, rv, z, U * rstd, z, z)


def check_fin(name, fin: Fin, mean_rstd=None, rm=None, rv=None, kappa=KAPPA_FIN):
    """Results for the stored mean / rstd and running statistics (any of them None: not judged)."""
    out = []
    if mean_rstd is not None:
        out.append(check_value(name + " mean", mean_rstd[0], fin.mean, fin.u_mean, kappa=kappa))
        out.append(check_value(name + " rstd", mean_rstd[1], fin.rstd, fin.u_rstd, kappa=kappa))
    if rm is not None:
        out.append(check_value(name + " running_mean", rm, fin.rm, fin.u_rm, kappa=kappa))
    if rv is not None:
        out.append(check_value(name + " running_var", rv, fin.rv, fin.u_rv, kappa=kappa))
    return out


def stat_slots_bound(stats):
    """Error of adding the [slots, 2, C] fp32 partials in order: (d1, d2)."""
    s = _d(stats).reshape(-1, 2, stats.shape[-1])
    mag = s.abs().sum(0) * U * max(0, s.shape[0] - 1)
    return mag[0], mag[1]


def affine_statement(x, mean, rstd, gamma, beta, res=None, u_rstd=None):
    """(value, unit) of ``(x - mean) * rstd * gamma + beta [+ res]`` as the kernels evaluate it: scale = gamma * rstd, shift =
    beta - mean * scale, x * scale + shift [+ res] -- every term's magnitude may carry a few fp32 roundings; ``u_rstd``: an uncertainty
    of rstd itself (evaluation mode: rstd is not stored)."""
    x, mean, rstd, gamma, beta = _d(x), _d(mean), _d(rstd), _d(gamma), _d(beta)
    sc = gamma * rstd
    v = x * sc + (beta - mean * sc)
    mag = (x * sc).abs() + (mean * sc).abs() + beta.abs()
    if res is not None:
        v = v + _d(res)
        mag = mag + _d(res).abs() + v.abs()
    unit = U * mag
    if u_rstd is not None:
        unit = unit + ((x - mean) * gamma).abs() * _d(u_rstd)
    return v, unit


def epi_relu(relu):
    return (lambda a: rn_bf16(a.clamp_min(0))) if relu else rn_bf16


def bn_bwd_terms(dy, x, mask, mean_rstd):
    """[2, M, C] fp64 terms of the backward sums: dz = dy * mask and dz * xhat, xhat = (x - mean) * rstd."""
    C = x.shape[-1]
    dz = _d(dy).reshape(-1, C) * mask.reshape(-1, C)
    xhat = (_d(x).reshape(-1, C) - _d(mean_rstd[0])) * _d(mean_rstd[1])
    return torch.stack([dz, dz * xhat]), xhat


def bn_dx_statement(dz, xhat, gamma, mean_rstd, dsum):
    """(value, unit) of dx = gamma rstd (dz - S0/M - xhat S1/M) given the kernel's stored sums ``dsum`` ([slots, 2, C])."""
    M = dz.shape[0]
    S = _d(dsum).reshape(-1, 2, dz.shape[-1]).sum(0)
    k1, k2 = S[0] / M, S[1] / M
    g = _d(gamma) * _d(mean_rstd[1])
    v = g * (dz - k1 - xhat * k2)
    unit = U * g.abs() * (dz.abs() + k1.abs() + (xhat * k2).abs())
    return v, unit


def bn_param_grads(dsum):
    """(dgamma, dbeta, unit) from the kernel's own stored sums: dbeta = (S0 / M) * M, dgamma = (S1 / M) * M in fp32."""
    s = _d(dsum).reshape(-1, 2, dsum.shape[-1])
    S = s.sum(0)
    unit = U * (s.abs().sum(0) * max(1, s.shape[0]) + S.abs())
    return S[1], S[0], unit[1], unit[0]


# =====================================================================================================================
# GroupNorm
# =====================================================================================================================
def gn_groups(x, groups):
    """[B, G, n] fp64 view of x [B, H, W, C] by (sample, group): group g = channels [g C/G, (g+1) C/G)."""
    B, C = x.shape[0], x.shape[-1]
    return _d(x).reshape(B, -1, groups, C // groups).permute(0, 2, 1, 3).reshape(B, groups, -1)


def gn_stats(x, groups, mean_k, eps, kappa=KAPPA_STATS):
    """Statements of the stored per-(sample, group) mean and rstd: the mean against the exact one (its in-kernel sum within the
    summation bound), the centred variance against the exact sum of squares about the kernel's OWN mean."""
    xg = gn_groups(x, groups)
    n = xg.shape[-1]
    mean = xg.mean(-1)
    u_mean = U * (kappa * math.sqrt(n) + 1) * xg.abs().sum(-1) / n + U * mean.abs()
    var_k = ((xg - _d(mean_k)[..., None]) ** 2).mean(-1)                   # about the kernel's own mean
    dvar = U * (kappa * math.sqrt(n) + 2) * var_k
    rstd, u_r = rsqrt_interval(var_k, dvar, f32(eps))
    return mean, u_mean, rstd, u_r + U * rstd


def per_channel(t, C):
    """[B, G] -> [B, 1, 1, C]: the value of each channel's group."""
    B, G = t.shape
    return t.repeat_interleave(C // G, dim=1).reshape(B, 1, 1, C)


def gn_dx_statement(dz, x, gamma, mean_rstd, groups, kappa=KAPPA_STATS):
    """(value, unit) of dx = rstd (dz gamma - s_a/M - xhat s_b/M), s_a = sum dz gamma, s_b = sum dz gamma xhat per (sample, group), with
    the summation bound of the in-kernel sums s_a, s_b (they are not stored)."""
    B, H, W, C = x.shape
    G = groups
    m = per_channel(_d(mean_rstd[:, 0]), C)
    r = per_channel(_d(mean_rstd[:, 1]), C)
    xhat = (_d(x) - m) * r
    a = dz * _d(gamma)
    b = a * xhat
    M = H * W * (C // G)

    def gsum(t):
        return t.reshape(B, H * W, G, C // G).sum((1, 3))

    sa, sb = gsum(a), gsum(b)
    ua = U * (kappa * math.sqrt(M) + 2) * gsum(a.abs())
    ub = U * (kappa * math.sqrt(M) + 2) * gsum(b.abs())
    ka, kb = per_channel(sa, C) / M, per_channel(sb, C) / M
    v = r * (a - ka - xhat * kb)
    unit = r.abs() * ((per_channel(ua, C) + xhat.abs() * per_channel(ub, C)) / M + U * (a.abs() + ka.abs() + (xhat * kb).abs()))
    return v, unit, xhat


# =====================================================================================================================
# pooling
# =====================================================================================================================
def maxpool_statement(x, drop: Drop | None = None):
    """(y, idx) of the 2x2 / stride-2 max-pool (floor mode): the FIRST maximum in window order (0,0), (0,1), (1,0), (1,1), ties
    included; fused dropout: y = keep ? rn_bf16(fp32(y * scale)) : 0 with the keep-mask of the pooled element."""
    B, H, W, C = x.shape
    Ho, Wo = H // 2, W // 2
    xc = x[:, :2 * Ho, :2 * Wo].float()
    cands = [xc[:, dy::2, dx::2] for dy in (0, 1) for dx in (0, 1)]
    best, idx = cands[0].clone(), torch.zeros(B, Ho, Wo, C, dtype=torch.uint8, device=x.device)
    for k in (1, 2, 3):
        up = cands[k] > best
        best = torch.where(up, cands[k], best)
        idx = torch.where(up, torch.full_like(idx, k), idx)
    if drop is not None:
        keep = dropout_keep(best.shape, drop, x.device)
        best = torch.where(keep, rn_bf16(best * drop.scale("f32")), torch.zeros_like(best))
    return best.to(torch.bfloat16), idx


def maxpool_bwd_statement(dy, idx, in_shape, drop: Drop | None = None, zmask=None):
    """dx of the max-pool: g = dy [* keep * scale, rounded once] [* (pooled output > 0)] at each window's arg-max, zeros elsewhere,
    including the last row / column of an odd-sized input."""
    B, H, W, C = in_shape
    Ho, Wo = H // 2, W // 2
    g = dy.float()
    if drop is not None:
        keep = dropout_keep(g.shape, drop, dy.device)
        g = torch.where(keep, g * drop.scale("f32"), torch.zeros_like(g))
    if zmask is not None:
        g = torch.where(zmask.float() > 0, g, torch.zeros_like(g))
    g = rn_bf16(g)
    dx = torch.zeros(B, H, W, C, device=dy.device)
    for k in range(4):
        dx[:, (k >> 1):2 * Ho:2, (k & 1):2 * Wo:2] = torch.where(idx == k, g, torch.zeros_like(g))
    return dx.to(torch.bfloat16)


def avgpool_statement(x):
    """(Statement, phi) of the global average pool: s = sum over H x W, one fp32 chain of HW terms, then rn_bf16(s / HW)."""
    B, H, W, C = x.shape
    xd = _d(x).reshape(B, H * W, C)
    HW = H * W
    return Statement(xd.sum(1), (xd * xd).sum(1), HW), (lambda a: rn_bf16(a.float() / HW))


def avgpool_bwd_statement(dy, in_shape):
    B, H, W, C = in_shape
    return rn_bf16(dy.float().reshape(B, 1, 1, C) / (H * W)).expand(B, H, W, C).to(torch.bfloat16)


# =====================================================================================================================
# ReLU backward and dropout
# =====================================================================================================================
def relu_bwd_statement(dy, y, scale=1.0):
    """dy <- rn_bf16(fp32(dy * scale)) where y > 0, else 0 (scale: fp32 of the host value)."""
    s = f32(scale)
    return torch.where(y.float() > 0, rn_bf16(dy.float() * s), torch.zeros_like(dy, dtype=torch.float32)).to(torch.bfloat16)


def dropout_statement(x, drop: Drop):
    """(y, mask) of the stand-alone dropout kernel over the flat tensor: y = keep ? rn_bf16(x * scale) : 0, mask = keep (uint8)."""
    keep = dropout_keep(x.shape, drop, x.device)
    y = torch.where(keep, rn_bf16(x.float() * drop.scale("f32")), torch.zeros_like(x, dtype=torch.float32))
    return y.to(torch.bfloat16), keep.to(torch.uint8)


def dropout_bwd_statement(dy, mask, p):
    s = Drop(p, 0, 0, 0).scale("f32")
    return torch.where(mask != 0, rn_bf16(dy.float() * s), torch.zeros_like(dy, dtype=torch.float32)).to(torch.bfloat16)


def epi_linear_drop(bias, relu, keep, scale):
    """Epilogue of a linear layer with fused dropout (wgmma GEMM epilogue and split-K finishing pass): rn_bf16(relu(acc + b) * keep *
    scale), computed in fp32; monotone in acc."""
    b = bias.float() if bias is not None else None
    kf = keep.float()

    def phi(a):
        if b is not None:
            a = a + b
        if relu:
            a = a.clamp_min(0)
        return rn_bf16(torch.where(kf > 0, a * scale, torch.zeros_like(a)))
    return phi
