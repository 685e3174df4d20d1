"""Layer primitives of the native executor (models/native.py), each with an ``sm100`` back-end (hand-written kernels
of ops/csrc: gemm.cu = wgmma/TMA implicit-GEMM convolution + GEMM, norm.cu = NHWC bf16 layer kernels) and an
``aten`` back-end (the same math through PyTorch library calls on the same buffers: CPU path + in-place oracle).

Reference call sites these primitives replace (SURVEY.md 2.4 rows K2-K8): the ``nn.Conv2d`` / ``nn.Linear`` / ``max_pool2d`` /
``Dropout2d`` layers of src/models.py:11-58 and their autograd backward inside ``loss.backward()`` (src/agent.py:47-48); the
BatchNorm / residual / average-pool primitives serve ResNet-18 and VGG-11, which the reference does not have."""
from __future__ import annotations

import math
import os

import torch
import torch.nn.functional as F

_scratch = {}
_s2d_done = {}
STAT_SLOTS = 16         # conv epilogues spread their BatchNorm statistics over this many partial buffers (gemm.h kStatSlots)
USE_WGRAD_HALO = True   # 3x3/s1/p1, 64 input channels: halo-reuse weight-gradient kernel (wgrad.cu)
# Stride-2 convolutions without parity-split copies: the forward conv and the weight gradient read the original input through a
# TMA box with element strides 2, and the four parity planes of the data gradient are stored straight into dX (strided epilogue
# rows) -- no space_to_depth / depth_to_space passes.  RLR_STRIDED_TMA=0 restores the copies.
USE_STRIDED_TMA = bool(int(os.environ.get("RLR_STRIDED_TMA", "1")))
# Stem convolutions (Cin * k * k <= 64, stride 1): gather the k x k x Cin patch of every output pixel into ONE 64-wide K block
# (im2col_small, or -- in the training step -- directly by the batch-assembly kernel gather_im2col) and run the plain wgmma GEMM on
# it, instead of k*k k-blocks of a 64-channel zero-padded input; the weight gradient is a [Cout x 64] GEMM over the same matrix.
# Tested by tests/test_gpu_variants.py::test_im2col_stem_conv_and_wgrad and tests/test_gpu_native.py::test_stem_gemm_*;
# RLR_IM2COL_STEM=0 restores the padded conv.
USE_IM2COL_STEM = bool(int(os.environ.get("RLR_IM2COL_STEM", "1")))
# BatchNorm(+ReLU, no residual) backward without reading the layer output: the mask is recomputed from x with the forward's own
# scale/shift expression: one activation read less per backward pass; default on (RLR_BN_RECOMPUTE=0 reads the stored output instead).
USE_BN_RECOMPUTE = bool(int(os.environ.get("RLR_BN_RECOMPUTE", "1")))
# 3x3/s1/p1 convs with 64 input channels: three filter taps per N = 192 MMA with a lane shift-add epilogue (conv_halo3.cu) instead of
# nine N = 64 MMAs per k-step (33 % more tiles, shuffles in the epilogue): opt-in (RLR_HALO3=1).
USE_HALO3 = bool(int(os.environ.get("RLR_HALO3", "0")))
# halo-reuse kernel also for valid / full 3x3 convs and sizes that are not whole 16x8 tiles (reference CNNs: conv2 and its data gradient)
USE_HALO_ANY = bool(int(os.environ.get("RLR_HALO_ANY", "1")))
# Dense layers with few output tiles and a deep reduction (FMNIST CNN fc1: 256 x 128 x 9216): split-K GEMM with an fp32 workspace
# (gemm_splitk.cu).  Verified and default on (RLR_SPLITK=0 runs the single-pass GEMM).
USE_SPLITK = bool(int(os.environ.get("RLR_SPLITK", "1")))
# Classifier-head kernels v2 (weights staged in shared memory, weight gradient spread over K/64 x B/16 blocks, partials summed in a fixed order).
# Default on (RLR_HEAD_V2=0 restores the first kernels).
USE_HEAD_V2 = bool(int(os.environ.get("RLR_HEAD_V2", "1")))


def _stem_ok(k, stride, cin, cout):
    return USE_IM2COL_STEM and stride == 1 and cin * k * k <= 64 and cout % 8 == 0 and (cout <= 64 or cout % 128 == 0)


def stem_geometry(in_shape, a):
    """(k, pad, Ho, Wo) if the conv with attributes ``a`` on an (H, W, C) input takes the im2col stem path, else None.  The native
    trainer asks this for its first layer and, if so, lets the batch-assembly kernel write the im2col matrix directly."""
    h, w, c = in_shape
    k, s, p = a["k"], a.get("stride", 1), a.get("pad", 0)
    if not _stem_ok(k, s, c, a["cout"]):
        return None
    return k, p, h + 2 * p - k + 1, w + 2 * p - k + 1


def _ext():
    from . import ext
    return ext()


def _zero(t):
    from . import zero_
    return zero_(t)


def _fallback(site, detail=""):
    from . import note_fallback
    note_fallback(site, detail)


def scratch(tag, shape, dtype, device):
    """Persistent scratch tensor (stable address: safe to bake into CUDA graphs)."""
    key = (tag, tuple(shape), dtype, str(device))
    t = _scratch.get(key)
    if t is None:
        t = _scratch[key] = torch.zeros(shape, dtype=dtype, device=device)
    return t


# =====================================================================================================================
# convolution
# =====================================================================================================================
def conv_supported(in_shape, a, kind):
    """Can the wgmma implicit-GEMM kernel run this conv?  ``in_shape`` = (H, W, Cin)."""
    h, w, cin = in_shape
    k, s, p, cout = a["k"], a.get("stride", 1), a.get("pad", 0), a["cout"]
    if k not in (1, 3) or s not in (1, 2) or cout % 8:
        return False
    even = s == 1 or (h % 2 == 0 and w % 2 == 0)
    if kind == "fwd":
        return even and (cin % 64 == 0 or cin < 64)
    if kind == "dgrad":      # reduction over Cout (padded to 64 by the TMA zero fill is NOT available here: K must be exact)
        return even and cin % 8 == 0 and cout % 64 == 0
    if kind == "wgrad":
        return even and (cin % 64 == 0 or cin < 64) and (cout <= 64 or cout % 128 == 0)
    return False


def _halo_ok(k, stride, pad, cin, h, w, stats=False):
    """Can the persistent halo-reuse kernel (conv_halo.cu) take this 3x3 / stride-1 conv of a 64-channel [h, w] input?  Padding 0 / 1 / 2
    (valid, same, full = the data gradient of a valid conv); any output size -- the image is covered by 16 x 8 pixel tiles and pixels
    beyond it are masked -- as long as at least half of the tile area is real output (below that the generic implicit GEMM, which
    packs the pixels of several images into one 128-row tile, wastes fewer MMAs).  BatchNorm statistics need whole tiles."""
    if not (k == 3 and stride == 1 and cin == 64 and pad in (0, 1, 2)):
        return False
    if not USE_HALO_ANY:                                     # round-1 predicate: 'same' convs on whole tiles only
        return pad == 1 and h % 16 == 0 and w % 8 == 0
    ho, wo = h + 2 * pad - 2, w + 2 * pad - 2
    if ho < 1 or wo < 1:
        return False
    if stats and (ho % 16 or wo % 8):
        return False
    return 2 * ho * wo >= (-(-ho // 16) * 16) * (-(-wo // 8) * 8)


def _wgrad_halo_ok(k, stride, pad, cin, h, w):
    return k == 3 and stride == 1 and pad == 1 and cin == 64 and h % 16 == 0 and w % 8 == 0


def _taps(k, stride, pad):
    dh, dw, pl = [], [], []
    for dy in range(k):
        for dx in range(k):
            oy, ox = dy - pad, dx - pad
            if stride == 1:
                dh.append(oy); dw.append(ox); pl.append(0)
            else:  # input index 2*o + off  ->  parity plane (off mod 2), shifted by floor(off / 2)
                dh.append(oy // 2); dw.append(ox // 2); pl.append((oy % 2) * 2 + (ox % 2))
    return dh, dw, pl


def conv2d_fwd_sm100(x, w, bias, y, stride, pad, relu, stats, tag="fwd", zero_stats=True, s2d_epoch=None, wait=None):
    """y[B,Ho,Wo,Cout] = conv(x[B,H,W,Cin], w[Cout,k,k,Cin]) (+bias)(ReLU); ``stats`` [STAT_SLOTS,2,Cout] accumulates per-channel
    sum / sum^2 partials (sum over dim 0 for the totals).  ``wait`` = (ready_ptr, lo, hi, epoch_tensor): stem path only -- the GEMM's
    producer warp acquires the broadcast-ready words [lo, hi] before it reads the filter (``w`` then lives in the multicast shadow)."""
    e = _ext()
    Cout, k = w.shape[0], w.shape[1]
    if x.dim() == 2:      # the batch-assembly kernel already produced the im2col matrix A[B*Ho*Wo][64] (gather_im2col)
        B, Ho, Wo, Cin = y.shape[0], y.shape[1], y.shape[2], w.shape[3]
        assert x.shape == (B * Ho * Wo, 64) and _stem_ok(k, stride, Cin, Cout)
        if stats is not None and zero_stats:
            _zero(stats)
        rp, lo, hi, ep = wait if wait is not None else (0, 0, 0, None)
        # the un-padded filter [Cout][k*k*Cin] is gathered (and zero-padded to K = 64) by the GEMM's producer warp: no padded copy
        e.stem_gemm_bf16(x, w.reshape(Cout, k * k * Cin), y.view(B * Ho * Wo, Cout), bias, bool(relu), stats, int(rp), int(lo), int(hi), ep)
        return y
    B, H, W, Cin = x.shape
    if _stem_ok(k, stride, Cin, Cout):
        Ho, Wo = y.shape[1], y.shape[2]
        A = scratch(("im2col", tag), (B * Ho * Wo, 64), x.dtype, x.device)
        e.im2col_small(x.contiguous(), A, k, pad)
        if stats is not None and zero_stats:
            _zero(stats)
        e.stem_gemm_bf16(A, w.reshape(Cout, k * k * Cin), y.view(B * Ho * Wo, Cout), bias, bool(relu), stats, 0, 0, 0, None)
        return y
    if Cin % 64:
        cp = (Cin + 63) // 64 * 64
        xp = scratch(("xpad", tag), (B, H, W, cp), x.dtype, x.device)
        e.pad_rows(x.reshape(B * H * W, Cin), xp.view(B * H * W, cp))                   # channel padding: rows = pixels
        wp = scratch(("wpad", tag, w.data_ptr()), (Cout, k, k, cp), w.dtype, w.device)
        e.pad_rows(w.reshape(Cout * k * k, Cin), wp.view(Cout * k * k, cp))
        x, w, Cin = xp, wp, cp
    if _halo_ok(k, stride, pad, Cin, H, W, stats is not None):
        # persistent halo-reuse kernel (conv_halo.cu): 36 KB of L2 traffic per 128-pixel tile instead of 216 KB
        if USE_HALO3 and stats is None and pad == 1 and H % 16 == 0:
            e.conv3x3_halo3_bf16(x, w.reshape(Cout, 9 * 64), y, bias, bool(relu), False)
            return y
        if stats is not None and zero_stats:
            _zero(stats)
        e.conv3x3_halo_bf16(x, w.reshape(Cout, 9 * 64), y, bias, bool(relu), False, stats, 0, None)
        return y
    if stride == 2 and USE_STRIDED_TMA and stats is None:
        e.conv_bf16_strided(x, w.reshape(Cout, k * k * Cin), y, [dy_ - pad for dy_ in range(k) for _ in range(k)],
                            [dx_ - pad for _ in range(k) for dx_ in range(k)], bias, bool(relu), False, [], 0, 2, 1, 0, 0)
        return y
    planes = 1
    if stride == 2:
        # parity-split copy keyed by the INPUT tensor: the 3x3/s2 conv and the 1x1/s2 shortcut of a ResNet block read the same
        # input, so within one forward pass (same `s2d_epoch`) the copy is made once and shared (also with both weight gradients)
        key = ("s2d", x.data_ptr(), Cin)
        x4 = scratch(key, (4 * B, H // 2, W // 2, Cin), x.dtype, x.device)
        if s2d_epoch is None or _s2d_done.get(key + (B,)) != s2d_epoch:
            e.space_to_depth(x, x4)
            _s2d_done[key + (B,)] = s2d_epoch
        x, planes = x4, 4
    dh, dw, pl = _taps(k, stride, pad)
    if stats is not None and zero_stats:
        _zero(stats)
    e.conv_bf16(x, w.reshape(Cout, k * k * Cin), y, B, planes, dh, dw, pl, bias, bool(relu), False, stats, [], 0)
    return y


def conv2d_dgrad_sm100(dy, w, dx, stride, pad, accumulate):
    """dx[B,H,W,Cin] (+)= conv_transpose(dy[B,Ho,Wo,Cout], w[Cout,k,k,Cin]) for stride 1: a convolution of dy with
    the tap-flipped, transposed filter and padding k-1-pad."""
    e = _ext()
    Cout, k, _, Cin = w.shape
    B = dy.shape[0]
    if stride == 2:
        return _conv2d_dgrad_s2(e, dy, w, dx, pad, accumulate)
    if _halo_ok(k, 1, k - 1 - pad, Cout, dy.shape[1], dy.shape[2]) and dx.shape[-1] % 8 == 0:
        wt = scratch(("wt", w.data_ptr(), dx.data_ptr()), (Cin, k * k * Cout), w.dtype, w.device)   # resident-filter kernel wants K-major taps
        e.filter_transpose(w, wt, Cout, k * k, Cin)
        if USE_HALO3 and pad == 1 and dy.shape[1] % 16 == 0:
            e.conv3x3_halo3_bf16(dy, wt, dx, None, False, bool(accumulate))
        else:
            e.conv3x3_halo_bf16(dy, wt, dx, None, False, bool(accumulate), None, 0, None)
        return dx
    dh, dw, pl = _taps(k, 1, k - 1 - pad)
    if Cin % 64 == 0:
        # read the forward filter W[co][tap][ci] directly as an MN-major B operand; k-block tap t' multiplies filter tap T-1-t'
        T = k * k
        e.conv_bf16(dy, w.reshape(Cout, T * Cin), dx, B, 1, dh, dw, pl, None, False, bool(accumulate), None,
                    [T - 1 - t for t in range(T)], T)
        return dx
    wt = scratch(("wt", w.data_ptr(), dx.data_ptr()), (Cin, k * k * Cout), w.dtype, w.device)
    e.filter_transpose(w, wt, Cout, k * k, Cin)
    e.conv_bf16(dy, wt, dx, B, 1, dh, dw, pl, None, False, bool(accumulate), None, [], 0)
    return dx


def _conv2d_dgrad_s2(e, dy, w, dx, pad, accumulate):
    """Stride-2 data gradient by input parity: input pixel (2a+pi, 2b+pj) only receives the taps with
    (pi + pad - dy) and (pj + pad - dx) even, from output pixel (a + (pi+pad-dy)/2, b + (pj+pad-dx)/2).  Each parity
    plane is therefore a small stride-1 convolution of dY with a sub-filter (1/2/2/4 taps for 3x3, pad 1); the four
    planes are computed by the wgmma conv kernel into a parity-split buffer and interleaved by depth_to_space, or (strided
    mode) stored directly at their pixels of dX."""
    Cout, k, _, Cin = w.shape
    B, Ho, Wo, _ = dy.shape
    plan = []
    for pi in range(2):
        for pj in range(2):
            taps, dh, dw = [], [], []
            for fy in range(k):
                for fx in range(k):
                    if (pi + pad - fy) % 2 == 0 and (pj + pad - fx) % 2 == 0:
                        taps.append(fy * k + fx); dh.append((pi + pad - fy) // 2); dw.append((pj + pad - fx) // 2)
            if taps:
                plan.append((pi, pj, taps, dh, dw))
    if USE_STRIDED_TMA and Cin % 64 == 0 and dx.shape[1] == 2 * Ho and dx.shape[2] == 2 * Wo:
        # each parity plane is stored straight into dX by the conv epilogue (row index = strided pixel): no parity buffer, no merge
        if not accumulate and len(plan) < 4:
            _zero(dx)                      # planes that receive no tap (1x1 shortcut: three of four)
        for pi, pj, taps, dh, dw in plan:
            e.conv_bf16_strided(dy, w.reshape(Cout, k * k * Cin), dx, dh, dw, None, False, bool(accumulate), taps, k * k, 1, 2, pi, pj)
        return dx
    dx4 = scratch(("dx4", w.data_ptr(), dx.data_ptr()), (4 * B, Ho, Wo, Cin), dy.dtype, dy.device)
    mask = 0
    for pi, pj, taps, dh, dw in plan:
        plane = pi * 2 + pj
        mask |= 1 << plane
        if Cin % 64 == 0:   # forward filter read MN-major: the plane's sub-filter is just a tap list
            e.conv_bf16(dy, w.reshape(Cout, k * k * Cin), dx4[plane * B:(plane + 1) * B], B, 1, dh, dw, [0] * len(taps), None,
                        False, False, None, taps, k * k)
            continue
        wt = scratch(("wt_s2", w.data_ptr(), dx.data_ptr(), plane), (Cin, len(taps) * Cout), w.dtype, w.device)
        e.filter_gather_transpose(w, wt, Cout, k * k, Cin, taps)
        e.conv_bf16(dy, wt, dx4[plane * B:(plane + 1) * B], B, 1, dh, dw, [0] * len(taps), None, False, False, None, [], 0)
    e.depth_to_space(dx4, dx, bool(accumulate), mask)
    return dx


def conv2d_wgrad_sm100(x, dy, gw, gb, stride, pad, tag="fwd", zero=True):
    """gw[Cout,k,k,Cin] (fp32) = sum over pixels of dy (x) x  (+ gb = sum dy).  Reuses the channel-padded / parity-split
    copies of ``x`` that ``conv2d_fwd_sm100`` left in the scratch buffers of the same ``tag``."""
    e = _ext()
    Cout, k = gw.shape[0], gw.shape[1]
    pre = x.dim() == 2                                      # x is already the im2col matrix (gather_im2col)
    B, H, W, Cin = (dy.shape[0], 0, 0, gw.shape[3]) if pre else x.shape
    cin_valid = Cin
    if pre or _stem_ok(k, stride, Cin, Cout):
        Ho, Wo = dy.shape[1], dy.shape[2]
        A = x if pre else scratch(("im2col", tag), (B * Ho * Wo, 64), x.dtype, x.device)   # filled by the forward pass
        dW = scratch(("dwstem", tag), (Cout, 64), torch.float32, x.device)
        _zero(dW)
        e.linear_wgrad_bf16(dy.view(B * Ho * Wo, Cout), A, dW)
        if zero:
            _zero(gw)
        e.unpad_add(dW, gw.view(Cout, k * k * Cin))                                      # valid K columns into the flat gradient
        if gb is not None:
            _bias_grad(e, dy, gb, zero)
        return
    if Cin % 64:
        cp = (Cin + 63) // 64 * 64
        x = scratch(("xpad", tag), (B, H, W, cp), x.dtype, x.device)      # filled by the forward pass
        Cin = cp
    planes = 1
    strided = stride == 2 and USE_STRIDED_TMA
    if stride == 2 and not strided:
        x = scratch(("s2d", x.data_ptr(), Cin), (4 * B, H // 2, W // 2, Cin), x.dtype, x.device)  # filled by the forward pass
        planes = 4
    dh, dw, pl = _taps(k, stride, pad)
    if zero:
        _zero(gw)
    if strided:
        e.conv_wgrad_bf16_strided(dy, x, gw, cin_valid, [dy_ - pad for dy_ in range(k) for _ in range(k)],
                                  [dx_ - pad for _ in range(k) for dx_ in range(k)], 2)
    elif USE_WGRAD_HALO and _wgrad_halo_ok(k, stride, pad, Cin, H, W) and (Cout <= 64 or Cout % 128 == 0):
        e.conv_wgrad_halo_bf16(dy, x, gw, cin_valid)
    else:
        e.conv_wgrad_bf16(dy, x, gw, B, planes, cin_valid, dh, dw, pl)
    if gb is not None:
        _bias_grad(e, dy, gb, zero)


def _bias_ok(C):
    return C >= 8 and C <= 2048 and C % 8 == 0 and 256 % (C // 8) == 0       # norm.cu chan_ok


def _bias_grad(e, dy, gb, zero):
    """gb[C] = column sums of dy[..., C], written straight into the flat gradient (one reduction kernel, no staging copy)."""
    C = dy.shape[-1]
    if zero:
        _zero(gb)
    if _bias_ok(C):
        e.bias_grad(dy.contiguous(), gb)
    else:
        _fallback("bias_grad", f"C={C}")
        gb.add_(dy.float().reshape(-1, C).sum(0))


# =====================================================================================================================
# batch norm (+ residual + relu)
# =====================================================================================================================
def bn_fwd(x, y, res, gamma, beta, rm, rv, stats, mean_rstd, count, eps, momentum, train, relu, impl, stats_buf=None):
    """``stats``: per-channel sum / sum^2 partials already produced by the conv epilogue, or None -> one streaming pass over
    ``x`` computes them here (into ``stats_buf`` [1,2,C], assumed zeroed, or a scratch buffer)."""
    C = x.shape[-1]
    if impl == "sm100":
        e = _ext()
        if train and stats is None:
            if stats_buf is not None:
                stats = stats_buf
            else:
                stats = scratch(("bnstats", mean_rstd.data_ptr()), (1, 2, C), torch.float32, x.device)
                _zero(stats)
            e.channel_stats(x, stats)
        # mean / rstd are derived inside bn_apply from the raw sums (training) or the running statistics (evaluation): no
        # separate finalize launch; CTA 0 stores mean/rstd for the backward pass and updates the running statistics
        e.bn_apply(x, res, y, gamma, beta, mean_rstd, bool(relu), 1 if train else 2, stats if train else None, float(count), float(eps),
                   float(momentum), rm, rv)
        return
    xf = x.float().reshape(-1, C)
    if train:
        if stats is not None:
            tot = stats.reshape(-1, 2, C).sum(0)
            mean = tot[0] / count
            var = (tot[1] / count - mean * mean).clamp_min(0)
        else:
            mean = xf.mean(0)
            var = xf.var(0, unbiased=False)
        rm.mul_(1 - momentum).add_(momentum * mean)
        rv.mul_(1 - momentum).add_(momentum * var * (count / max(1, count - 1)))
        mean_rstd[0].copy_(mean); mean_rstd[1].copy_(torch.rsqrt(var + eps))
    else:
        mean_rstd[0].copy_(rm); mean_rstd[1].copy_(torch.rsqrt(rv + eps))
    out = (xf - mean_rstd[0]) * (mean_rstd[1] * gamma) + beta
    if res is not None:
        out = out + res.float().reshape(-1, C)
    if relu:
        out = out.clamp_min(0)
    y.copy_(out.reshape(y.shape))


def bn_bwd(dy, y, x, gamma, mean_rstd, dsum, dx, dres, dgamma, dbeta, relu, impl, zero_dsum=True, beta=None):
    C = x.shape[-1]
    if impl == "sm100":
        if USE_BN_RECOMPUTE and relu and dres is None and beta is not None:
            # BN + ReLU without a residual: recompute the ReLU mask from x (needed anyway for xhat) instead of reading y -- one
            # activation-sized read less in each of the two backward passes
            _ext().bn_bwd_recompute(dy, x, gamma, beta, mean_rstd, dsum, dx, dgamma, dbeta, bool(zero_dsum))
            return
        _ext().bn_bwd(dy, y, x, gamma, mean_rstd, dsum, dx, dres, dgamma, dbeta, bool(relu), bool(zero_dsum))
        return
    dz = dy.float().reshape(-1, C)
    if relu:
        dz = dz * (y.float().reshape(-1, C) > 0)
    if dres is not None:
        dres.copy_(dz.reshape(dres.shape))
    xhat = (x.float().reshape(-1, C) - mean_rstd[0]) * mean_rstd[1]
    s0, s1 = dz.sum(0), (dz * xhat).sum(0)
    M = dz.shape[0]
    dbeta.copy_(s0); dgamma.copy_(s1)
    dx.copy_((gamma * mean_rstd[1] * (dz - s0 / M - xhat * s1 / M)).reshape(dx.shape))


# =====================================================================================================================
# group norm (+ residual + relu)
# =====================================================================================================================
def gn_supported(x, groups):
    """Shapes the GroupNorm kernels (groupnorm.cu) take: NHWC, C % 8 == 0, ``groups`` divides C, at most 2048 channels per group
    rounded up to whole 8-channel vectors."""
    C = x.shape[-1]
    cpg = C // groups if groups > 0 and C % groups == 0 else 0
    return x.dim() == 4 and C % 8 == 0 and cpg > 0 and (8 // math.gcd(8, cpg)) * cpg <= 2048


def gn_fwd(x, y, res, gamma, beta, mean_rstd, groups, eps, relu, impl):
    """y[B,H,W,C] = [ReLU]((x - mean_ng) * rstd_ng * gamma_c + beta_c [+ res]) with torch.nn.GroupNorm(groups, C, eps) statistics
    (per sample and group over H x W x C/groups, biased variance); ``mean_rstd`` [B,2,groups] fp32 receives mean / rstd for
    ``gn_bwd``.  Training and evaluation compute the same thing (no running state)."""
    if impl == "sm100":
        if gn_supported(x, groups):
            _ext().gn_fwd(x, res, y, gamma, beta, mean_rstd, int(groups), float(eps), bool(relu))
            return
        _fallback("gn_fwd", f"shape={tuple(x.shape)} groups={groups}")
    B, C = x.shape[0], x.shape[-1]
    xg = x.float().reshape(B, -1, groups, C // groups)                               # [B, HW, G, C/G]
    mean = xg.mean((1, 3))
    var = xg.var((1, 3), unbiased=False)
    rstd = torch.rsqrt(var + eps)
    mean_rstd[:, 0].copy_(mean); mean_rstd[:, 1].copy_(rstd)
    out = ((xg - mean[:, None, :, None]) * rstd[:, None, :, None]).reshape(B, -1, C) * gamma + beta
    if res is not None:
        out = out + res.float().reshape(B, -1, C)
    if relu:
        out = out.clamp_min(0)
    y.copy_(out.reshape(y.shape))


def gn_bwd(dy, y, x, gamma, mean_rstd, dx, dres, dgamma, dbeta, groups, relu, impl, zero=True):
    """Backward of ``gn_fwd``: dz = dy * [y > 0] (relu) ; dres = dz (residual) ; dx = rstd * (dz*gamma - s_a/M - xhat * s_b/M) with
    s_a = sum dz*gamma, s_b = sum dz*gamma*xhat per (sample, group) and M = H*W*C/groups ; dgamma = sum dz*xhat, dbeta = sum dz.
    ``zero=False``: dgamma / dbeta are added into (the native plan's flat gradient is zeroed once per step)."""
    if zero:
        _zero(dgamma)
        _zero(dbeta)
    if impl == "sm100":
        if gn_supported(x, groups):
            _ext().gn_bwd(dy, y if relu else None, x, gamma, mean_rstd, dx, dres, dgamma, dbeta, int(groups), bool(relu))
            return
        _fallback("gn_bwd", f"shape={tuple(x.shape)} groups={groups}")
    B, C = x.shape[0], x.shape[-1]
    G, cpg = groups, C // groups
    dz = dy.float().reshape(B, -1, C)
    if relu:
        dz = dz * (y.float().reshape(B, -1, C) > 0)
    if dres is not None:
        dres.copy_(dz.reshape(dres.shape))
    mean, rstd = mean_rstd[:, 0], mean_rstd[:, 1]                                    # [B, G]
    xhat = ((x.float().reshape(B, -1, G, cpg) - mean[:, None, :, None]) * rstd[:, None, :, None]).reshape(B, -1, C)
    dgamma.add_((dz * xhat).sum((0, 1)))
    dbeta.add_(dz.sum((0, 1)))
    dzg = (dz * gamma).reshape(B, -1, G, cpg)
    M = dzg.shape[1] * cpg
    s_a = dzg.sum((1, 3))[:, None, :, None]
    s_b = (dzg * xhat.reshape(B, -1, G, cpg)).sum((1, 3))[:, None, :, None]
    d = rstd[:, None, :, None] * (dzg - s_a / M - xhat.reshape(B, -1, G, cpg) * s_b / M)
    dx.copy_(d.reshape(dx.shape))


def relu_bwd_(dy, y, impl, scale=1.0):
    """dy <- dy * (y > 0) * scale.  ``scale`` = 1/(1-p) when dropout was fused into the producer of ``y`` (y = relu(z) * keep / (1-p)):
    y > 0 exactly where the element was kept and z > 0, so one mask read off the output covers ReLU and dropout."""
    if impl == "sm100" and dy.numel() % 8 == 0:
        _ext().relu_bwd(dy, y, float(scale))
    else:
        if impl == "sm100":
            _fallback("relu_bwd", f"numel={dy.numel()}")
        dy.mul_((y > 0).to(dy.dtype) * scale)


# =====================================================================================================================
# pooling / dropout
# =====================================================================================================================
def maxpool2_fwd(x, y, idx, impl, drop=None, mask=None):
    """2x2 max-pool; ``drop`` = (p, seed, step counter tensor, node id): dropout fused into the pooling kernel (Philox keep-mask of the
    pooled element, recomputed by ``maxpool2_bwd`` -- no mask tensor).  The aten back-end draws a torch mask into ``mask`` instead."""
    if impl == "sm100" and x.shape[-1] % 8 == 0:
        if drop is not None:
            _ext().maxpool2_fwd(x, y, idx, float(drop[0]), int(drop[1]), drop[2], int(drop[3]))
        else:
            _ext().maxpool2_fwd(x, y, idx)
        return
    if impl == "sm100":
        _fallback("maxpool2_fwd", f"C={x.shape[-1]}")
    B, H, W, C = x.shape
    Ho, Wo = H // 2, W // 2
    win = x[:, :Ho * 2, :Wo * 2].reshape(B, Ho, 2, Wo, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(B, Ho, Wo, C, 4)
    v, i = win.float().max(-1)
    if drop is not None:
        keep = torch.rand(v.shape, device=v.device) >= drop[0]
        mask.copy_(keep)
        v = v * keep / (1 - drop[0])
    y.copy_(v); idx.copy_(i)


def maxpool2_bwd(dy, idx, dx, impl, drop=None, mask=None, relu_out=None):
    """dx[B,H,W,C] = gradient of the 2x2 max-pool (zeros except at each window's arg-max).  ``drop`` = the dropout fused into the pooling
    forward (mask recomputed); ``relu_out`` = the pooled forward output when the ReLU fused into the PRODUCER of the pooled tensor is
    back-propagated here as well: the arg-max is positive iff the pooled value is, so no separate pass over the 4x larger tensor."""
    if impl == "sm100" and dx.shape[-1] % 8 == 0:
        kw = dict(relu_out=relu_out.contiguous()) if relu_out is not None else {}
        if drop is not None:
            _ext().maxpool2_bwd(dy, idx, dx, float(drop[0]), int(drop[1]), drop[2], int(drop[3]), **kw)
        else:
            _ext().maxpool2_bwd(dy, idx, dx, **kw)
        return
    if impl == "sm100":
        _fallback("maxpool2_bwd", f"C={dx.shape[-1]}")
    if relu_out is not None:
        dy = dy * (relu_out > 0).to(dy.dtype)
    B, H, W, C = dx.shape
    Ho, Wo = H // 2, W // 2
    dx.zero_()
    if drop is not None:
        dy = dy * mask.to(dy.dtype) / (1 - drop[0])
    oh = F.one_hot(idx.long(), 4).to(dy.dtype) * dy.unsqueeze(-1)                   # [B,Ho,Wo,C,4]
    dx[:, :Ho * 2, :Wo * 2].copy_(oh.reshape(B, Ho, Wo, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(B, Ho * 2, Wo * 2, C))


def avgpool_fwd(x, y, impl):
    if impl == "sm100":
        _ext().avgpool_fwd(x, y)
    else:
        y.copy_(x.float().mean((1, 2), keepdim=True))


def avgpool_bwd(dy, dx, impl):
    if impl == "sm100":
        _ext().avgpool_bwd(dy, dx)
    else:
        dx.copy_((dy.float() / (dx.shape[1] * dx.shape[2])).expand_as(dx))


def dropout_fwd(x, y, mask, p, seed, step, stream, impl):
    if impl == "sm100" and x.numel() % 8 == 0:
        _ext().dropout_fwd(x, y, mask, float(p), int(seed), step, int(stream))
        return
    if impl == "sm100":
        _fallback("dropout_fwd", f"numel={x.numel()}")
    keep = torch.rand(x.shape, device=x.device) >= p
    mask.copy_(keep)
    y.copy_(x * keep / (1 - p))


def dropout_bwd(dy, mask, dx, p, impl):
    if impl == "sm100" and dx.numel() % 8 == 0:
        _ext().dropout_bwd(dy, mask, dx, float(p))
    else:
        if impl == "sm100":
            _fallback("dropout_bwd", f"numel={dx.numel()}")
        dx.copy_(dy * mask / (1 - p))


# =====================================================================================================================
# linear
# =====================================================================================================================
def linear_fused_dropout_ok(N, K):
    """Can dropout be fused into this linear layer's GEMM epilogue (wgmma GEMM / split-K finishing pass)?"""
    return N > 32 and K % 64 == 0 and N % 64 == 0


def linear_fwd(x, w, bias, y, relu, impl, drop=None):
    """y[B,N] = x[B,K] w[N,K]^T + b (ReLU).  N <= 32: CUDA-core head kernel; otherwise the wgmma GEMM.  ``drop`` = (p, seed, step
    counter tensor, node id): dropout fused into the GEMM epilogue after bias / ReLU (SURVEY.md K5); the backward pass reads the
    combined ReLU-and-dropout mask off the output (``relu_bwd_(..., scale=1/(1-p))``)."""
    N, K = w.shape
    dk = dict(drop_p=float(drop[0]), drop_seed=int(drop[1]), drop_step=drop[2], drop_stream=int(drop[3])) if drop is not None else {}
    if impl == "sm100":
        if N <= 32:
            if USE_HEAD_V2 and K % 2 == 0 and (N * K) % 8 == 0 and N * K * 2 <= 48 * 1024:
                _ext().linear_small_fwd2(x.contiguous(), w, bias, y, bool(relu))
                return
            _ext().linear_small_fwd(x.contiguous(), w, bias, y, bool(relu))
            return
        if K % 64 == 0 and N % 64 == 0:
            M = x.shape[0]
            if USE_SPLITK and K >= 1024 and ((M + 127) // 128) * ((N + 127) // 128) <= 16:
                ws = scratch(("splitk_ws", y.data_ptr()), (M, N), torch.float32, x.device)     # zero at creation, left zero by the kernel
                _ext().gemm_splitk_bf16(x.contiguous(), w, y, ws, bias, bool(relu), **dk)
                return
            _ext().gemm_bf16(x.contiguous(), w, y, bias, bool(relu), False, None, **dk)
            return
        _fallback("linear_fwd", f"N={N} K={K}")
    out = F.linear(x, w.to(x.dtype), bias.to(x.dtype) if bias is not None else None)
    if relu:
        out = F.relu(out)
    if drop is not None:       # aten back-end: torch's own RNG; the backward still reads the mask off y (relu + dropout)
        out = out * (torch.rand(out.shape, device=out.device) >= drop[0]) / (1 - drop[0])
    y.copy_(out)


def linear_bwd(x, dy, w, dx, dw, db, acc_dx, impl, zero=True):
    N, K = w.shape
    if impl == "sm100" and N <= 32:
        if USE_HEAD_V2 and K % 2 == 0:
            if zero:                  # v2 accumulates with atomics (the native plan passes zero=False: the flat gradient is pre-zeroed)
                _zero(dw)
                if db is not None:
                    _zero(db)
            _ext().linear_small_bwd2(x.contiguous(), dy.contiguous(), w, dx, dw, db, bool(acc_dx))
            return
        _ext().linear_small_bwd(x.contiguous(), dy.contiguous(), w, dx, dw, db, bool(acc_dx))
        return
    dyf = dy.to(x.dtype)
    sm = impl == "sm100" and K % 64 == 0 and N % 64 == 0
    if sm and (N <= 64 or N % 128 == 0):
        if zero:
            _zero(dw)
        _ext().linear_wgrad_bf16(dy.contiguous(), x.contiguous(), dw)
    else:
        if impl == "sm100":
            _fallback("linear_wgrad", f"N={N} K={K}")
        dw.copy_(dyf.t() @ x)
    if db is not None:
        if sm and _bias_ok(N):
            _bias_grad(_ext(), dy, db, zero)
        else:
            if impl == "sm100":
                _fallback("linear_bias_grad", f"N={N}")
            db.copy_(dyf.float().sum(0))
    if dx is not None:
        if sm:   # dx = dy @ W  ==  GEMM with the transposed weight as the K-major B operand
            wt = scratch(("wt_lin", w.data_ptr(), dx.data_ptr()), (K, N), w.dtype, w.device)   # per consumer: trainers in flight may share w (broadcast buffer)
            _ext().filter_transpose(w, wt, N, 1, K)
            _ext().gemm_bf16(dy.contiguous(), wt, dx, None, False, bool(acc_dx), None)
            return
        if impl == "sm100":
            _fallback("linear_dgrad", f"N={N} K={K}")
        d = dyf @ w.to(x.dtype)
        if acc_dx:
            dx.add_(d)
        else:
            dx.copy_(d)
