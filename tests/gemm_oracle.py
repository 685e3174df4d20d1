"""fp64 statements of the tensor-core GEMM / convolution kernels and a checker that judges each output element against them.

A *statement* of an entry point is the exact result of its reduction, computed in fp64 from the same bf16 operands (every bf16
product and every partial sum of up to 2^20 of them is exact or within 2^-40 relative in fp64):

* ``s``  -- the sum of products of every output element,
* ``sq`` -- the sum of the squared products, which sizes the fp32 accumulation error,
* ``K``  -- the reduction length.

The kernels accumulate in fp32 and then apply an *epilogue* ``phi`` in fp32: bias, ReLU, the bf16 pack with round-to-nearest-even,
and for accumulating outputs the read-modify-write of the old value.  Each epilogue is monotone in the accumulator, so an output that
came from an accumulator within ``delta`` of ``s`` lies in ``[phi(s - delta), phi(s + delta)]``, with::

    delta = KAPPA * 2^-24 * L * sqrt(sq),    L = K (bf16 outputs),  L = min(K, CHAIN) (fp32 outputs)

``L`` is the length of one fp32 accumulation chain.  The bf16-output kernels run the whole reduction as one chain.  The fp32 outputs
are the weight and bias gradients: their kernels split a long pixel range over CTAs, each CTA accumulating at most a few thousand
products, and add the split partials in a fixed order.  Errors of different splits are independent, so the total stays that of
one chain of ``CHAIN`` products.

The checker reports, per element, the smallest ``kappa`` for which the element is inside its interval, and fails if any exceeds
``KAPPA`` (an element whose statement has ``sq == 0`` -- no tap reached it -- must equal ``phi(s)`` exactly).  A second criterion
catches rounding-mode errors that stay within one ulp: the fraction of bf16 elements that differ from ``phi(s)`` must not exceed
``RHO``.

Calibration (H100 80GB HBM3 at 700 W; 219 distinct conv / linear problems harvested from one training step of every zoo model at
batch 256 / 96 / 80, the edge shapes and the knob matrix of tests/test_gpu_gemm_oracle.py).  The unbiased random-walk model
``2^-24 sqrt(K) sqrt(sq)`` of fp32 accumulation does NOT fit the wgmma accumulation: the kappa it needs grows like sqrt(K) along
one accumulation chain -- 1.5 at K = 576, 2.2 at 1152, 2.9 at 2304, 4.9 at 4608 for the forward convolutions, 6.6 for the layer-4
weight gradient (K = 256 x 4 x 4) -- so the error grows like K, as a biased (truncating) accumulation does.  The bound is therefore
linear in K.  Largest kappa needed under it: 0.079 forward convolutions (layer 4, K = 4608), 0.079 data gradients, 0.11 conv weight
gradients (layer 4; the split-K weight gradients of the large layers need far less, their chains are short), 0.057 linear layers;
the largest, 0.49, at the tiniest reductions that add into an existing gradient (a conv weight gradient over one 2 x 2 image,
K = 4 + the old value; the head weight gradient at batch 7: 0.24); statistics 0.19 of their bound; largest mismatch fraction
0.29 % (fc1 without split-K, K = 9216).  The split fp32 weight gradients need kappa * K <= 455 at every K up to 262144 (the layer-1
3x3 weight gradient at batch 256; 421 for the unsplit layer-4 one at K = 4096), so ``CHAIN = 4096`` puts them at kappa <= 0.11,
where the whole length K would have allowed the layer-1 gradient 64x more error.  ``KAPPA``, ``KAPPA_STATS`` and ``RHO`` keep a
margin of 4x over these.
"""
from __future__ import annotations

import math
from typing import Callable, NamedTuple

import torch
import torch.nn.functional as F

U = 2.0 ** -24          # unit roundoff of fp32 round-to-nearest
KAPPA = 2.0             # accumulation-error constant of ``delta`` (see the calibration above)
CHAIN = 4096            # longest fp32 accumulation chain counted for the split-K fp32 outputs
KAPPA_STATS = 0.8       # the same for the per-channel statistics sums (``delta = KAPPA_STATS * U * sqrt(M) * sum |v|``)
RHO = 0.012             # largest fraction of bf16 outputs allowed to differ from phi(s)
GUARD = 64              # guard elements placed after every output buffer


class Statement(NamedTuple):
    s: torch.Tensor      # fp64 exact sum of products
    sq: torch.Tensor     # fp64 sum of squared products
    K: int               # reduction length (an upper bound where padding drops terms)


def _d(t):
    return t.double()


# =====================================================================================================================
# statements
# =====================================================================================================================
def gemm_statement(a, b) -> Statement:
    """out[m, n] = sum_k a[m, k] b[n, k]."""
    a, b = _d(a), _d(b)
    return Statement(a @ b.t(), (a * a) @ (b * b).t(), a.shape[1])


def conv_statement(x, w, stride, pad) -> Statement:
    """Forward convolution, NHWC: y[b, i, j, co] = sum_{dy, dx, ci} x[b, s i + dy - p, s j + dx - p, ci] w[co, dy, dx, ci] (zero padding)."""
    xd, wd = _d(x).permute(0, 3, 1, 2), _d(w).permute(0, 3, 1, 2)
    s = F.conv2d(xd, wd, None, stride, pad).permute(0, 2, 3, 1)
    sq = F.conv2d(xd * xd, wd * wd, None, stride, pad).permute(0, 2, 3, 1)
    return Statement(s, sq, w.shape[1] * w.shape[2] * w.shape[3])


def _conv_bwd(dy, x_shape, x, w, stride, pad, mask):
    dyd = _d(dy).permute(0, 3, 1, 2)
    xd = _d(x).permute(0, 3, 1, 2) if x is not None else torch.zeros(x_shape, dtype=torch.float64, device=dy.device).permute(0, 3, 1, 2)
    wd = _d(w).permute(0, 3, 1, 2)
    return torch.ops.aten.convolution_backward(dyd, xd, wd, None, [stride, stride], [pad, pad], [1, 1], False, [0, 0], 1, mask)


def dgrad_statement(dy, w, x_shape, stride, pad) -> Statement:
    """Data gradient: dx = d(sum dy * conv(x, w)) / dx, NHWC [B, H, W, Cin]."""
    s = _conv_bwd(dy, x_shape, None, w, stride, pad, [True, False, False])[0]
    sq = _conv_bwd(dy * dy, x_shape, None, w * w, stride, pad, [True, False, False])[0]
    return Statement(s.permute(0, 2, 3, 1), sq.permute(0, 2, 3, 1), w.shape[0] * w.shape[1] * w.shape[2])


def wgrad_statement(x, dy, k, stride, pad) -> Statement:
    """Weight gradient: gw[co, dy, dx, ci] = sum over batch and output pixels of dy[.., co] x[.., tap, ci], [Cout, k, k, Cin]."""
    w0 = torch.zeros(dy.shape[-1], k, k, x.shape[-1], dtype=torch.float64, device=x.device)
    s = _conv_bwd(dy, None, x, w0, stride, pad, [False, True, False])[1]
    sq = _conv_bwd(dy * dy, None, x * x, w0, stride, pad, [False, True, False])[1]
    return Statement(s.permute(0, 2, 3, 1), sq.permute(0, 2, 3, 1), dy.shape[0] * dy.shape[1] * dy.shape[2])


def colsum_statement(v) -> Statement:
    """Bias gradient: gb[c] = sum over every other index of v[..., c]."""
    vd = _d(v).reshape(-1, v.shape[-1])
    return Statement(vd.sum(0), (vd * vd).sum(0), vd.shape[0])


def plus_old(st: Statement, old) -> Statement:
    """An fp32 output that adds into an existing value: the old value is one more term of the sum."""
    o = _d(old)
    return Statement(st.s + o, st.sq + o * o, st.K + 1)


# =====================================================================================================================
# epilogues, evaluated in the kernels' own precision (fp32 arithmetic, bf16 round-to-nearest-even)
# =====================================================================================================================
def rn_bf16(t):
    return t.float().to(torch.bfloat16).float()


def epi_store(bias=None, relu=False) -> Callable:
    """bf16(relu?(acc + bias)): forward convolutions, GEMMs, split-K, the head kernels, overwriting data gradients."""
    def phi(a):
        if bias is not None:
            a = a + bias.float()
        if relu:
            a = a.clamp_min(0)
        return rn_bf16(a)
    return phi


def epi_acc_twice(old) -> Callable:
    """bf16(bf16(acc) + old): accumulating conv / GEMM epilogues (gemm.cu, gemm_persistent.cu, conv_halo*.cu) and the accumulating
    depth_to_space merge of the parity planes -- the accumulator is packed to bf16 before the old value is added."""
    o = old.float()
    return lambda a: rn_bf16(rn_bf16(a) + o)


def epi_acc_once(old) -> Callable:
    """bf16(acc + old): the CUDA-core head kernels add the old data gradient to the fp32 accumulator and round once."""
    o = old.float()
    return lambda a: rn_bf16(a + o)


def epi_f32(a):
    """fp32 outputs (weight and bias gradients): the accumulator itself."""
    return a


# =====================================================================================================================
# checker
# =====================================================================================================================
class Result(NamedTuple):
    name: str
    kappa: float         # largest per-element kappa needed (inf: an element no accumulation error explains)
    mismatch: float      # fraction of elements != phi(s) (bf16 outputs)
    worst: tuple         # index of the worst element
    ok: bool


def needed_kappa(out, st: Statement, phi, L, kmax=1e6, iters=48):
    """Per element, the smallest kappa with phi(s - kappa du) <= out <= phi(s + kappa du), du = 2^-24 L sqrt(sq); inf if none
    up to ``kmax`` (also for NaN)."""
    o = out.float()
    du = U * L * st.sq.sqrt()

    def inside(k):
        return (o >= phi((st.s - k * du).float())) & (o <= phi((st.s + k * du).float()))

    hi = torch.full_like(st.s, kmax)
    reach = inside(hi)
    lo = torch.zeros_like(st.s)
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        m = inside(mid)
        hi = torch.where(m, mid, hi)
        lo = torch.where(m, lo, mid)
    k = torch.where(inside(lo.new_zeros(())), torch.zeros_like(hi), hi)
    return torch.where(reach, k, torch.full_like(k, math.inf))


def check(name, out, st: Statement, phi, kappa=KAPPA, rho=RHO) -> Result:
    """Judge ``out`` against statement ``st`` under epilogue ``phi``; bf16 outputs also face the mismatch-fraction criterion."""
    assert out.shape == st.s.shape, (name, tuple(out.shape), tuple(st.s.shape))
    k = needed_kappa(out, st, phi, min(st.K, CHAIN) if out.dtype == torch.float32 else st.K)
    kmax = float(k.max()) if k.numel() else 0.0
    worst = tuple(int(i) for i in torch.unravel_index(k.argmax(), k.shape)) if k.numel() else ()
    mism = float((out.float() != phi(st.s.float())).double().mean()) if out.dtype == torch.bfloat16 and out.numel() else 0.0
    ok = kmax <= kappa and (out.dtype != torch.bfloat16 or mism <= rho)
    return Result(name, kmax, mism, worst, ok)


def check_stats(name, stats, out, kappa=KAPPA_STATS) -> Result:
    """Per-channel BatchNorm statistics ``stats`` ([slots, 2, C] fp32 partials, or [2, C]) against the sums of the STORED bf16 output
    ``out`` (masked rows are not in ``out``, so they count as zero), computed in fp64.  Bound: fp32 summation of M terms,
    ``kappa * 2^-24 * sqrt(M) * sum |v|``."""
    y = _d(out).reshape(-1, out.shape[-1])
    want = torch.stack([y.sum(0), (y * y).sum(0)])
    mag = torch.stack([y.abs().sum(0), (y * y).sum(0)])
    got = _d(stats).reshape(-1, 2, out.shape[-1]).sum(0)
    bound = U * math.sqrt(y.shape[0]) * mag
    r = (got - want).abs() / bound.clamp_min(1e-300)
    r = torch.where((got - want).abs() == 0, torch.zeros_like(r), r)
    r = torch.where(torch.isnan(got), torch.full_like(r, math.inf), r)
    kmax = float(r.max())
    worst = tuple(int(i) for i in torch.unravel_index(r.argmax(), r.shape))
    return Result(name, kmax, 0.0, worst, kmax <= kappa)


# =====================================================================================================================
# output buffers with guard bands
# =====================================================================================================================
def guarded(shape, dtype, device, fill=float("nan")):
    """(view, buffer): a contiguous output of ``shape`` followed by GUARD elements in one allocation; the view is prefilled with
    ``fill`` (NaN: any element the kernel does not write fails the check), the guard band with a sentinel."""
    n = math.prod(shape)
    buf = torch.empty(n + GUARD, dtype=dtype, device=device)
    buf[:n] = fill
    buf[n:] = -1232.0
    return buf[:n].view(shape), buf


def guard_intact(buf) -> bool:
    return bool((buf[-GUARD:].float() == -1232.0).all())
