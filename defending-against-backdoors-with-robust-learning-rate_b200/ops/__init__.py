"""Operator layer.

Every op has two implementations behind one Python signature:

* **native** -- a hand-written sm_90a kernel from ``ops/_C.so`` (sources in ``ops/csrc``), used whenever the tensors
  live on a CUDA device.  If the extension is missing on a GPU box the op raises -- there is no silent eager fallback.
* **oracle** -- a plain fp32/fp64 PyTorch re-statement of the same semantics, used on CPU (the plumbing config and the
  CPU test-suite) and as the numerical reference the GPU tests compare the kernels against.

The reference has no operator layer at all (SURVEY.md 2.4): each row of that table maps to one function here.
"""
from __future__ import annotations

import importlib.util
import math
import os
import threading
from typing import NamedTuple

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_C.so")
_ext = None
_ext_err = None
_lock = threading.Lock()

MODE_IDS = {"avg": 0, "comed": 1, "sign": 2}
MAX_FUSED_AGENTS = 1024   # kMaxAgents of ops/csrc/aggregate.cu (participant tables of the fused kernel)
SERVER_OPTS = {"sgd": 0, "momentum": 1, "adagrad": 2, "adam": 3, "yogi": 4}   # AggParams::opt of ops/csrc/aggregate.cu


class _Counter:
    """Counts calls into the native extension (each call launches >= 1 of our kernels); used for ``gpu_launches``."""
    calls = 0


class _CountingExt:
    def __init__(self, mod):
        self._mod = mod
        self._cache = {}

    def __getattr__(self, name):
        fn = self._cache.get(name)
        if fn is None:
            real = getattr(self._mod, name)
            if not callable(real):
                return real

            def fn(*a, _real=real, **k):
                _Counter.calls += 1
                return _real(*a, **k)
            self._cache[name] = fn
        return fn


def launch_calls() -> int:
    return _Counter.calls


# ---- library fall-throughs ---------------------------------------------------------------------------------------------
# The sm100 back-end of a layer primitive may meet a shape no kernel of ours covers and fall through to a PyTorch library call
# (cuBLAS / cuDNN / ATen).  Every such fall-through is recorded here by call site; ``RLR_STRICT=1`` turns it into an error.  The
# bench prints the counters (``library_fallbacks``) and tests/test_gpu_native.py asserts they stay empty for every zoo model.
_fallbacks: dict = {}


def note_fallback(site: str, detail: str = ""):
    _fallbacks[site] = _fallbacks.get(site, 0) + 1
    if os.environ.get("RLR_STRICT", "0") == "1":
        raise RuntimeError(f"RLR_STRICT=1: sm100 back-end fell through to a library call at {site} {detail}")


def fallback_calls() -> dict:
    """{call site: count} of library fall-throughs of the sm100 back-end since the last reset (empty = none)."""
    return dict(_fallbacks)


def reset_fallbacks():
    _fallbacks.clear()


def zero_(t):
    """Zero a tensor: a memset node on CUDA (no ATen fill kernel inside captured steps), ``zero_()`` on CPU."""
    if t.is_cuda and t.is_contiguous():
        ext().memset_zero(t)
    else:
        t.zero_()
    return t


def native_available() -> bool:
    """True if the compiled extension can be imported (it may still be unusable without a GPU)."""
    try:
        ext()
        return True
    except Exception:  # noqa: BLE001
        return False


def ext():
    """The compiled extension module; raises with build instructions if it is missing."""
    global _ext, _ext_err
    if _ext is not None:
        return _ext
    with _lock:
        if _ext is not None:
            return _ext
        if not os.path.exists(_SO):
            raise RuntimeError(f"native extension {_SO} not built; run `python -m rlr_b200.ops.build` "
                               "(or __graft_entry__.build())")
        spec = importlib.util.spec_from_file_location("rlr_b200.ops._C", _SO)
        mod = importlib.util.module_from_spec(spec)
        try:
            spec.loader.exec_module(mod)
        except Exception as e:  # noqa: BLE001
            _ext_err = e
            raise
        _ext = _CountingExt(mod)
    return _ext


def _i32(x, device):
    return torch.as_tensor(x, dtype=torch.int32, device=device)


# =====================================================================================================================
# data path
# =====================================================================================================================
_M32, _M64 = 2 ** 32 - 1, 2 ** 64 - 1


def philox4x32(ctr, stream, key):
    """Philox4x32-10 (Salmon et al., SC'11) with the packing of ``struct Philox`` in ops/csrc/common.cuh: counter words
    ``(ctr lo, ctr hi, stream lo, stream hi)``, key words ``(key lo, key hi)``.  ``ctr``: an integer or an integer array (uint64
    values); ``stream`` / ``key``: integers.  Returns the four output words as uint32 arrays of ``ctr``'s shape."""
    ctr = np.asarray(ctr).astype(np.uint64)
    stream, key = int(stream) & _M64, int(key) & _M64
    m32 = np.uint64(_M32)
    c0, c1 = ctr & m32, ctr >> np.uint64(32)
    c2, c3 = np.full_like(ctr, stream & _M32), np.full_like(ctr, stream >> 32)
    a, b = np.uint64(key & _M32), np.uint64(key >> 32)
    for _ in range(10):
        p0, p1 = c0 * np.uint64(0xD2511F53), c2 * np.uint64(0xCD9E8D57)       # 32 x 32 -> 64 bit, exact in uint64
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ a, p1 & m32, (p0 >> np.uint64(32)) ^ c3 ^ b, p0 & m32
        a, b = (a + np.uint64(0x9E3779B9)) & m32, (b + np.uint64(0xBB67AE85)) & m32
    return tuple(w.astype(np.uint32) for w in (c0, c1, c2, c3))


_AUGMENT_TAG = 0x6A09E667F3BCC908       # domain tag: keeps augmentation streams apart from every other Philox stream


def augment_stream(seed: int, agent_id: int, rnd: int, epoch: int) -> int:
    """Philox stream word of the training augmentation of (agent, round, local epoch): a splitmix64 hash in the style of
    ``models.native.dropout_stream_base``.  It does not depend on the rank, trainer or world size, so an agent draws the same
    crops wherever and alongside whatever it is trained.  Kept below 2^63 so it fits the device int64 word."""
    z = (int(seed) * 0x9E3779B97F4A7C15 + (int(agent_id) + 1) * 0xBF58476D1CE4E5B9 + (int(rnd) + 1) * 0x94D049BB133111EB
         + (int(epoch) + 1) * 0xD6E8FEB86659FD93 + _AUGMENT_TAG) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return (z ^ (z >> 31)) & (2 ** 63 - 1)


class Augment(NamedTuple):
    """Training augmentation of a gathered batch: ``RandomCrop(H x W, padding=pad, fill=0)`` then ``RandomHorizontalFlip()`` (when
    ``flip``) of the raw images, before normalisation.  Sample b of a batch is at position p = (cursor, or ``start`` without a
    cursor) + b of the epoch order and draws ``u = philox4x32(p, stream, seed)``: crop offsets ``u.x % (2 pad + 1)``,
    ``u.y % (2 pad + 1)``, flip ``u.z & 1``.  ``stream``: one-element int64 tensor on the data's device holding the epoch's
    ``augment_stream`` (the kernels read it at run time, so captured graphs follow it from epoch to epoch)."""
    pad: int
    flip: bool
    seed: int
    stream: torch.Tensor
    start: int = 0


def training_augment(args, stream):
    """The ``Augment`` of the engine flags ``--crop_pad`` / ``--hflip`` over the trainer's stream word; None when both are off."""
    pad, flip = int(getattr(args, "crop_pad", 0)), bool(getattr(args, "hflip", False))
    return Augment(pad, flip, int(args.seed), stream) if (pad or flip) else None


def augment_draws(aug: Augment, positions):
    """``(oy, ox, flip)`` int64 tensors of the samples at ``positions`` (the host statement of ``augment_draw``, common.cuh)."""
    u = philox4x32(np.asarray(positions, dtype=np.int64), int(aug.stream), aug.seed)
    n = 2 * int(aug.pad) + 1
    flip = (u[2] & 1).astype(np.int64) if aug.flip else np.zeros(len(u[2]), dtype=np.int64)
    return (torch.from_numpy((u[0] % n).astype(np.int64)), torch.from_numpy((u[1] % n).astype(np.int64)), torch.from_numpy(flip))


def augment_raw(x, aug: Augment, pos0: int):
    """Cropped / flipped raw images ``[B,H,W,C]`` of the batch at positions ``pos0 ..`` (the CPU path of the augmented gathers):
    ``aug[b,h,w] = x[b, h + oy - pad, w' + ox - pad]`` with ``w' = W-1-w`` when flipped, and 0 outside the image."""
    B, H, W, _ = x.shape
    oy, ox, fl = augment_draws(aug, pos0 + np.arange(B))
    P = int(aug.pad)
    xp = torch.nn.functional.pad(x, (0, 0, P, P, P, P))
    w = torch.arange(W)
    rows = torch.arange(H)[None, :] + oy[:, None]                                             # [B,H] in padded coordinates
    cols = torch.where(fl[:, None].bool(), W - 1 - w[None, :], w[None, :]) + ox[:, None]      # [B,W]
    return xp[torch.arange(B)[:, None, None], rows[:, :, None], cols[:, None, :]]


def _augment_args(aug):
    """Trailing (crop pad, flip, seed, stream word, start) arguments of the gather bindings."""
    if aug is None:
        return 0, False, 0, None, 0
    seed = int(aug.seed) & _M64
    return int(aug.pad), bool(aug.flip), seed - 2 ** 64 if seed >= 2 ** 63 else seed, aug.stream, int(aug.start)


def gather_normalize(data, idxs, mean, std, dtype=torch.float32, nhwc=False, c_pad=None, out=None,
                     cursor=None, targets=None, out_labels=None, batch=None, augment=None):
    """``normalize(data[idxs])``: raw NHWC uint8/float pixels -> fp32/bf16 batch (SURVEY.md K1).

    ``data`` [N,H,W,C]; ``idxs`` int64 sample indices (with ``cursor``: a device int32 offset into ``idxs`` so a CUDA
    graph can replay the launch over successive batches; ``batch`` = batch size then).  Output NCHW, or NHWC padded to
    ``c_pad`` channels when ``nhwc``.  Same arithmetic as ``ToTensor`` + ``Normalize`` (src/utils.py:101,112-115).
    ``augment``: an ``Augment`` -- the raw images are randomly cropped / flipped before normalisation.
    """
    N, H, W, C = data.shape
    B = int(batch if batch is not None else idxs.shape[0])
    c_pad = int(c_pad or C)
    if out is None:
        shape = (B, H, W, c_pad) if nhwc else (B, C, H, W)
        out = torch.empty(shape, dtype=dtype, device=data.device)
    if data.is_cuda:
        ext().gather_normalize(data, idxs, cursor, targets, out, out_labels, B, c_pad, not nhwc,
                               [float(m) for m in mean], [float(s) for s in std], *_augment_args(augment))
        return out
    off = int(cursor.item()) if cursor is not None else 0
    sel = idxs[off:off + B]
    x = data[sel].to(torch.float32)
    if augment is not None:
        x = augment_raw(x, augment, off if cursor is not None else augment.start)
    if data.dtype == torch.uint8:
        x = x / 255.0
    x = (x - torch.tensor(mean, dtype=torch.float32)) / torch.tensor(std, dtype=torch.float32)
    if nhwc:
        if c_pad > C:
            x = torch.nn.functional.pad(x, (0, c_pad - C))
        out.copy_(x.to(out.dtype))
    else:
        out.copy_(x.permute(0, 3, 1, 2).to(out.dtype))
    if out_labels is not None and targets is not None:
        out_labels[:B] = targets[sel]
    return out


def gather_im2col(data, idxs, mean, std, k, pad, out, cursor=None, targets=None, out_labels=None, batch=None, augment=None):
    """Batch assembly fused with the first layer's im2col (SURVEY.md K1+K2, tiny-K stems: C*k*k <= 64): row (b, ho, wo) of ``out``
    [B*Ho*Wo, 64] (bf16) is the k x k x C patch of the normalised image around that output pixel in (tap, channel) order, zero
    padded -- the A operand of the stem convolution as a single-k-block wgmma GEMM.  Same cursor / label / ``augment`` contract as
    ``gather_normalize``; the convolution's zero padding lies outside the augmented image and stays 0."""
    N, H, W, C = data.shape
    B = int(batch if batch is not None else idxs.shape[0])
    Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
    if data.is_cuda:
        ext().gather_im2col(data, idxs, cursor, targets, out, out_labels, B, int(k), int(pad), [float(m) for m in mean], [float(s) for s in std],
                            *_augment_args(augment))
        return out
    off = int(cursor.item()) if cursor is not None else 0
    sel = idxs[off:off + B]
    x = data[sel].to(torch.float32)
    if augment is not None:
        x = augment_raw(x, augment, off if cursor is not None else augment.start)
    if data.dtype == torch.uint8:
        x = x / 255.0
    x = (x - torch.tensor(mean, dtype=torch.float32)) / torch.tensor(std, dtype=torch.float32)          # [B,H,W,C]
    xp = torch.nn.functional.pad(x, (0, 0, pad, pad, pad, pad))
    cols = [xp[:, dy:dy + Ho, dx:dx + Wo, :] for dy in range(k) for dx in range(k)]                       # (tap, channel) order
    A = torch.cat(cols, dim=-1).reshape(B * Ho * Wo, k * k * C)
    out[:B * Ho * Wo].zero_()
    out[:B * Ho * Wo, :k * k * C] = A.to(out.dtype)
    if out_labels is not None and targets is not None:
        out_labels[:B] = targets[sel]
    return out


def stamp_pixels(data, sel, rows, cols, vals, mode):
    """Apply a compiled trojan pixel program to images ``sel`` of ``data`` [N,H,W,C] in place (SURVEY.md 2.2)."""
    if len(rows) == 0 or sel.numel() == 0:
        return data
    if data.is_cuda:
        dev = data.device
        ext().stamp_pixels(data, sel.to(dev, torch.int64).contiguous(), _i32(rows, dev), _i32(cols, dev),
                           torch.as_tensor(vals, dtype=torch.float32, device=dev), int(mode))
        return data
    r = torch.as_tensor(rows, dtype=torch.int64)
    c = torch.as_tensor(cols, dtype=torch.int64)
    v = torch.as_tensor(vals, dtype=torch.float32)
    s = sel.to(torch.int64)[:, None]
    cur = data[s, r[None, :], c[None, :], :]                      # [S,P,C]
    if mode == 0:
        new = v[None, :, None].expand_as(cur).to(data.dtype)
    elif mode == 1:  # uint8 wrap-around add
        new = ((cur.to(torch.int64) + v[None, :, None].to(torch.int64)) % 256).to(data.dtype)
    else:
        new = (cur.to(torch.float32) - v[None, :, None]).to(data.dtype)
    data[s, r[None, :], c[None, :], :] = new
    return data


# =====================================================================================================================
# server step
# =====================================================================================================================
class ServerOptState:
    """Server optimizer (``--server_opt``) and its state over coordinates ``[base, base + n)`` of the flat vector.

    ``m`` (every kind but sgd) starts at 0 and ``v`` (adagrad / adam / yogi) at ``tau**2``; both are fp32 and rounded once per round.
    sgd holds no state.  The update rules are in ``server_opt_step``."""

    def __init__(self, kind="sgd", n=0, beta1=0.9, beta2=0.99, tau=1e-3, device="cpu", base=0):
        if kind not in SERVER_OPTS:
            raise ValueError(f"unknown server optimizer {kind!r}; expected one of {tuple(SERVER_OPTS)}")
        self.kind, self.beta1, self.beta2, self.tau, self.base = kind, float(beta1), float(beta2), float(tau), int(base)
        self.m = torch.zeros(n, dtype=torch.float32, device=device) if kind != "sgd" else None
        self.v = torch.full((n,), self.tau * self.tau, dtype=torch.float32, device=device) if kind in ("adagrad", "adam", "yogi") else None

    @property
    def hparams(self):
        return {"server_opt": self.kind, "beta1": self.beta1, "beta2": self.beta2, "tau": self.tau}


def server_opt_step(d, opt):
    """fp64 server optimizer on the pseudo-gradient ``d`` of coordinates ``[opt.base, opt.base + len(d))`` (Reddi et al., Adaptive
    Federated Optimization, Algorithm 2, without bias correction; FedAvgM for momentum).  Returns the step that the server lr
    scales; the new state is rounded into ``opt.m`` / ``opt.v`` while the step uses the unrounded fp64 values.  Also the statement
    of the kernel's epilogue (``server_step`` in ops/csrc/aggregate.cu)."""
    b1, b2 = opt.beta1, opt.beta2
    m0 = opt.m[: d.numel()]
    if opt.kind == "momentum":
        m1 = b1 * m0.double() + d
        m0.copy_(m1)
        return m1
    m1 = b1 * m0.double() + (1.0 - b1) * d
    v0, d2 = opt.v[: d.numel()].double(), d * d
    if opt.kind == "adagrad":
        v1 = v0 + d2
    elif opt.kind == "adam":
        v1 = b2 * v0 + (1.0 - b2) * d2
    elif opt.kind == "yogi":
        v1 = v0 - (1.0 - b2) * d2 * torch.sign(v0 - d2)
    else:
        raise ValueError(opt.kind)
    m0.copy_(m1)
    opt.v[: d.numel()].copy_(v1)
    return m1 / (v1.sqrt() + opt.tau)


def _server_update(g, agg, signs, mean_tail, theta, server_lr, n_vote, opt):
    """RLR flip + server step (sgd, or ``opt``'s optimizer) on the voted coordinates, plain weighted mean behind ``n_vote``."""
    n = g.numel()
    lr = torch.full_like(g, float(server_lr))
    flipped = 0
    neg = None
    if theta > 0:
        neg = signs.abs() < theta
        neg[n_vote:] = False
        lr[neg] = -float(server_lr)
        flipped = int(neg.sum())
    if opt is None or opt.kind == "sgd":
        new = g + lr * agg
    else:
        if opt.base != 0:
            raise ValueError("the fp64 server step needs the full-length optimizer state (base 0)")
        d = agg[:n_vote] if neg is None else torch.where(neg[:n_vote], -agg[:n_vote], agg[:n_vote])
        new = g.clone()
        new[:n_vote] = g[:n_vote] + float(server_lr) * server_opt_step(d, opt)
    if n_vote < n:
        new[n_vote:] = g[n_vote:] + mean_tail[n_vote:]
    return new.float(), flipped


def aggregate_oracle(w_global, w_agents, weights, mode="avg", theta=0, server_lr=1.0, noise=None, n_vote=None,
                     scales=None, opt=None, total_weight=None):
    """fp64 PyTorch statement of the server step (reference src/aggregation.py:19-75).

    ``w_agents``: list of local parameter vectors; updates are ``w_k - w_global``.  ``noise``: optional pre-sampled
    noise vector (added to the aggregate BEFORE the lr multiply).  Coordinates ``>= n_vote`` get a plain weighted mean.
    ``opt``: optional ``ServerOptState`` (full length); its state is updated in place.  ``total_weight``: the weighted mean's
    denominator (default ``sum(weights)``).
    Returns ``(new_global_fp32, n_flipped)``.
    """
    g = w_global.double()
    n = g.numel()
    n_vote = n if n_vote is None else int(n_vote)
    ups = [(w.double() - g) for w in w_agents]
    wt = torch.as_tensor(weights, dtype=torch.float64, device=g.device)
    tot = wt.sum() if total_weight is None else float(total_weight)
    mean_raw = sum(w_ * u for w_, u in zip(wt, ups)) / tot     # tail coordinates (BatchNorm statistics) are never clip-scaled
    if scales is not None:
        ups = [u * float(s) for u, s in zip(ups, scales)]
    mean = sum(w_ * u for w_, u in zip(wt, ups)) / tot
    signs = sum(torch.sign(u) for u in ups)
    if mode == "avg":
        agg = mean.clone()
    elif mode == "comed":
        agg = torch.median(torch.stack(ups, dim=1), dim=1).values
    elif mode == "sign":
        agg = torch.sign(signs)
    else:
        raise ValueError(mode)
    if noise is not None:
        agg = agg + noise.double()
    return _server_update(g, agg, signs, mean_raw, theta, server_lr, n_vote, opt)


def aggregate_partials(w_global, w_local_agents, local_weights, n_vote=None, scales=None):
    """This rank's share of the server step for the additive aggregators: ``(vote, wsum)`` with
    ``vote = sum_k sign(w_k - w_g)`` (float32: small integers) and ``wsum = sum_k n_k (w_k - w_g)`` (float64) over the LOCAL
    participants.  Summed over ranks (all_reduce) they are exactly the ``signs`` and ``mean * sum(n)`` of ``aggregate_oracle``."""
    g = w_global.double()
    vote = torch.zeros_like(w_global, dtype=torch.float32)
    wsum = torch.zeros_like(g)
    nv = g.numel() if n_vote is None else int(n_vote)
    for i, (w, nk) in enumerate(zip(w_local_agents, local_weights)):
        u = w.double() - g
        if scales is not None:
            u = u.clone()
            u[:nv] *= float(scales[i])           # server clipping scales the voted coordinates only
        vote += torch.sign(u).float()
        wsum += float(nk) * u
    return vote, wsum


def aggregate_from_partials(w_global, vote, wsum, total_weight, mode="avg", theta=0, server_lr=1.0, noise=None, n_vote=None,
                            opt=None):
    """Finish the server step from globally reduced partials (same formulas and order as ``aggregate_oracle``; avg / sign only)."""
    if mode not in ("avg", "sign"):
        raise ValueError(f"aggregate_from_partials: mode {mode!r} is not additive (coordinate median needs every update)")
    g = w_global.double()
    n = g.numel()
    n_vote = n if n_vote is None else int(n_vote)
    mean = wsum / float(total_weight)
    signs = vote.double()
    agg = mean.clone() if mode == "avg" else torch.sign(signs)
    if noise is not None:
        agg = agg + noise.double()
    return _server_update(g, agg, signs, mean, theta, server_lr, n_vote, opt)


class PtrTable:
    """Device int64 table of raw pointers (kept with the tensors it points into, so they stay alive)."""

    def __init__(self, ptrs, device, keep=()):
        self.tensor = torch.tensor([int(p) for p in ptrs], dtype=torch.int64, device=device)
        self.keep = tuple(keep)


def fused_aggregate(w_global, w_agents, weights, mode="avg", theta=0, server_lr=1.0, noise_std=0.0, seed=0,
                    noise_stream=0, n_vote=None, scales=None, out=None, out_bf16=None, flipped=None, opt=None, total_weight=None):
    """Single-process fused server step: ``out <- w_global + lr ⊙ agg({w_k - w_global})`` in one kernel.

    On CUDA this launches ``fused_aggregate_kernel`` (ops/csrc/aggregate.cu); on CPU it runs the fp64 oracle (with
    torch-sampled noise).  ``out`` may alias ``w_global``.  ``opt``: optional full-length ``ServerOptState``, updated in place.
    ``total_weight``: the weighted mean's denominator (default ``sum(weights)``; FLTrust passes 1 when every weight is 0).
    Returns the tensor written.  The multi-GPU variant (peer pointers, multicast stores, in-kernel barriers) is driven by
    ``parallel.fused_agg.FusedAggregator``.
    """
    n = w_global.numel()
    n_vote = n if n_vote is None else int(n_vote)
    out = w_global if out is None else out
    dev = w_global.device
    if not w_global.is_cuda or len(w_agents) > MAX_FUSED_AGENTS:
        if w_global.is_cuda:
            # more participants than the kernel's pointer / weight tables hold (1024): exact torch evaluation on the device (fp64,
            # same semantics) -- recorded as a library fall-through
            note_fallback("fused_aggregate", f"K={len(w_agents)} > {MAX_FUSED_AGENTS}")
        noise = None
        if noise_std > 0:     # a torch generator on the data's device: the CPU and the device fall-through draw different streams
            gen = torch.Generator(device=dev).manual_seed(int(seed) * 1000003 + int(noise_stream))
            noise = torch.randn(n, generator=gen, dtype=torch.float64, device=dev) * noise_std
            noise[n_vote:] = 0
        new, nflip = aggregate_oracle(w_global, w_agents, weights, mode, theta, server_lr, noise, n_vote, scales, opt,
                                      total_weight)
        out.copy_(new)
        if out_bf16 is not None:
            out_bf16.copy_(new.to(torch.bfloat16))
        if flipped is not None:
            flipped += nflip
        return out
    assert n % 4 == 0 and n_vote % 4 == 0, "flat buffers are padded to multiples of 4"
    for w in w_agents:
        assert w.is_cuda and w.dtype == torch.float32 and w.is_contiguous() and w.numel() == n
    agents = PtrTable([w.data_ptr() for w in w_agents], dev, w_agents)
    outs = PtrTable([out.data_ptr()], dev)
    outs_b = PtrTable([out_bf16.data_ptr()], dev) if out_bf16 is not None else None
    wt = torch.as_tensor(weights, dtype=torch.float64).to(dev)
    sc = torch.as_tensor(scales, dtype=torch.float32).to(dev) if scales is not None else None
    tot = float(sum(float(x) for x in weights)) if total_weight is None else float(total_weight)
    ext().fused_aggregate(agents.tensor, wt, sc, tot, w_global.data_ptr(), outs.tensor,
                          outs_b.tensor if outs_b else None, False, 0, n, n_vote, MODE_IDS[mode], int(theta),
                          float(server_lr), float(noise_std), int(seed), int(noise_stream), flipped, None, None, 0, 1, 0,
                          False, *opt_launch_args(opt))
    return out


def opt_launch_args(opt):
    """The server optimizer arguments of the ``fused_aggregate`` binding: (opt, beta1, beta2, tau, opt_m, opt_v, state_base)."""
    if opt is None or opt.kind == "sgd":
        return 0, 0.0, 0.0, 0.0, None, None, 0
    return SERVER_OPTS[opt.kind], opt.beta1, opt.beta2, opt.tau, opt.m, opt.v, opt.base


def update_norms(w_global, w_agents, n=None):
    """L2 norms of the agents' updates ``||w_k - w_global||`` (server clipping, src/aggregation.py:77-81, and the
    Norms/* diagnostic, :83-100) -> float64 tensor [K].  ``n``: only the first ``n`` coordinates count (the model parameters:
    BatchNorm running statistics stored behind ``n_vote`` are not part of the reference's parameter vector)."""
    n = w_global.numel() if n is None else int(n)
    if not w_global.is_cuda:
        return torch.stack([(w[:n].double() - w_global[:n].double()).norm() for w in w_agents])
    # the trust pass with the root parameters at w_global: the root update is 0, so its q_k = ||w_k - w_global||^2 come out of the same
    # fixed-order sums (bitwise reproducible) while w_global is read once per group of participants.  q_k depends on participant k
    # alone, so chunks of the kernel's table size keep any number of participants on the device.
    out = torch.empty(len(w_agents), dtype=torch.float64, device=w_global.device)
    for c in range(0, len(w_agents), MAX_FUSED_AGENTS):
        part = w_agents[c:c + MAX_FUSED_AGENTS]
        torch.sqrt(trust_stats(part, w_global, w_global, n)[len(part):2 * len(part)], out=out[c:c + len(part)])
    return out


def _participant_pass(site, w_agents, others, nv, shape, statement, launch):
    """Dispatch of a per-participant pass over the voted coordinates ``[0, nv)``: the fp64 ``statement()`` on CPU and, recorded as a
    library fall-through at ``site``, for more participants than the kernels' tables hold; else ``launch(table, out)`` on the device
    pointer table of ``w_agents`` and a float64 ``out`` of ``shape``, which it returns.  ``others``: further flat buffers the kernel
    reads."""
    if not w_agents[0].is_cuda:
        return statement()
    if len(w_agents) > MAX_FUSED_AGENTS:
        note_fallback(site, f"K={len(w_agents)} > {MAX_FUSED_AGENTS}")
        return statement()
    assert nv % 4 == 0, "flat buffers are padded to multiples of 4"
    for w in (*w_agents, *others):
        assert w.is_cuda and w.dtype == torch.float32 and w.is_contiguous() and w.numel() >= nv
    dev = w_agents[0].device
    tab = PtrTable([w.data_ptr() for w in w_agents], dev, w_agents)
    out = torch.empty(shape, dtype=torch.float64, device=dev)
    launch(tab.tensor, out)
    return out


# =====================================================================================================================
# participant selection (Krum / Multi-Krum, Blanchard et al. 2017)
# =====================================================================================================================
def sqdist_statement(w_agents, lo, hi, w_global=None, scales=None):
    """fp64 statement of the pairwise squared distances over coordinates ``[lo, hi)``: ``D[i][j] = sum_c (x_i[c] - x_j[c])^2`` with
    ``x_k = w_k`` (no scales: ``w_global`` cancels) or ``x_k = (w_k - w_global) * scales[k]``.  Symmetric, zero diagonal."""
    K = len(w_agents)
    dev = w_agents[0].device
    D = torch.zeros(K, K, dtype=torch.float64, device=dev)
    sc = torch.as_tensor(scales, dtype=torch.float32).to(dev).double()[:, None] if scales is not None else None
    step = max(4, (1 << 24) // max(1, K))                 # coordinates per pass: K * step fp64 values
    for c in range(lo, hi, step):
        e = min(hi, c + step)
        x = torch.stack([w[c:e] for w in w_agents]).double()
        if sc is not None:
            x = (x - w_global[c:e].double()) * sc
        for i in range(K - 1):
            D[i, i + 1:] += ((x[i + 1:] - x[i]) ** 2).sum(1)
    return D + D.T


def pairwise_sqdist(w_agents, n_vote, w_global=None, scales=None):
    """K x K float64 squared distances between the participants' updates over the voted coordinates ``[0, n_vote)`` (the BatchNorm
    running statistics behind ``n_vote`` do not count).  ``scales`` (server clipping) need ``w_global``; without them the updates'
    differences are the parameters' differences.  On CUDA this launches ``pairwise_sqdist_kernel`` (ops/csrc/select.cu); on CPU, and
    for more participants than the kernel's tables hold (recorded as a library fall-through), it evaluates ``sqdist_statement``."""
    nv = w_agents[0].numel() if n_vote is None else int(n_vote)
    if scales is not None and w_global is None:
        raise ValueError("pairwise_sqdist: scales need w_global")

    def launch(tab, out):
        sc = torch.as_tensor(scales, dtype=torch.float32).to(out.device) if scales is not None else None
        ext().pairwise_sqdist(tab, w_global.data_ptr() if sc is not None else 0, sc, 0, nv, out, None, None, 0, 1, 0)
    K = len(w_agents)
    return _participant_pass("pairwise_sqdist", w_agents, (), nv, (K, K), lambda: sqdist_statement(w_agents, 0, nv, w_global, scales),
                             launch)


def krum_select(D, ids, f, m):
    """Krum / Multi-Krum admission on the host, in fp64: ``score_i`` = the sum of the ``K - f - 2`` smallest ``D[i][j]`` (``j != i``),
    added in ascending order; the ``m`` lowest scores are admitted (one-shot Multi-Krum; Krum is ``m = 1``), ties to the lower id in
    ``ids``.  A NaN distance counts as +inf.  Returns the admitted positions (indices into ``ids``) in ascending order, so every rank
    and every placement of the participants admits the same agents."""
    d = np.nan_to_num(torch.as_tensor(D).detach().double().cpu().numpy(), nan=np.inf)
    K = d.shape[0]
    nb = K - int(f) - 2
    if K < 2 * int(f) + 3 or nb < 1:
        raise ValueError(f"Krum needs K >= 2f + 3 participants (K={K}, f={f})")
    if not 1 <= int(m) <= K:
        raise ValueError(f"Multi-Krum keeps m in [1, K] (m={m}, K={K})")
    others = np.sort(d[~np.eye(K, dtype=bool)].reshape(K, K - 1), axis=1)[:, :nb]
    scores = np.cumsum(others, axis=1)[:, -1].tolist()       # cumsum adds sequentially: the ascending order of the statement
    order = sorted(range(K), key=lambda i: (scores[i], ids[i]))
    return sorted(order[: int(m)])


# =====================================================================================================================
# participant selection (DnC, Shejwalkar and Houmansadr, NDSS 2021): spectral scores on coordinate subsamples
# =====================================================================================================================
_DNC_TAG = 0x446E4321                    # "DnC!": keeps the subsample draws apart from every other stream seeded by --seed


def dnc_sample(seed, rnd, t, b, n_vote):
    """DnC's coordinate subsample of iteration ``t`` in round ``rnd``: ``min(b, n_vote)`` distinct coordinates of ``[0, n_vote)`` drawn
    without replacement by a numpy Generator seeded by (seed, round, t) alone, sorted ascending (``b >= n_vote``: every coordinate).
    Every rank, and a resumed run, draws the same sample.  Returns int64 numpy."""
    n_vote, b = int(n_vote), int(b)
    if n_vote >= 1 << 31:
        raise ValueError(f"DnC samples int32 coordinates: n_vote {n_vote} >= 2^31")
    if b >= n_vote:
        return np.arange(n_vote, dtype=np.int64)
    rng = np.random.default_rng([int(seed), int(rnd), int(t), _DNC_TAG])
    return np.sort(rng.choice(n_vote, size=b, replace=False)).astype(np.int64)


def dnc_gather_statement(w_agents, w_global, sample, scales=None):
    """fp64 statement of DnC's gather over the coordinates ``sample``: ``x_k = (w_k - w_global)`` (``* scales[k]``) in fp64,
    ``mu = (sum of the finite x_k, k ascending) / their count`` and ``Y[k] = fp32(x_k - mu)``, every operation rounded on its own -- the
    bits ``dnc_gather_kernel`` writes.  With every update finite ``mu`` is the plain mean over the K participants; a non-finite ``x_k``
    stays out of it and leaves its own entry non-finite.  Returns float32 ``[K][len(sample)]``."""
    dev = w_global.device
    idx = torch.as_tensor(np.asarray(sample, dtype=np.int64), device=dev)
    g = w_global[idx].double()
    x = [w[idx].double() - g for w in w_agents]
    if scales is not None:
        sc = torch.as_tensor(scales, dtype=torch.float32).to(dev).double()
        x = [xk * sc[k] for k, xk in enumerate(x)]
    mu = torch.zeros_like(g)
    n = torch.zeros_like(g)
    for xk in x:
        fin = torch.isfinite(xk)
        mu = torch.where(fin, mu + xk, mu)
        n = n + fin.double()
    mu = torch.where(n > 0, mu / n.clamp_min(1.0), torch.zeros_like(mu))
    return torch.stack([(xk - mu).float() for xk in x])


def dnc_gram_statement(w_agents, w_global, samples, scales=None):
    """fp64 statement of DnC's device pass: for each iteration's sample (row ``t`` of ``samples``), the Gram matrix ``C_t = Y Y^T`` in fp64
    of ``Y = dnc_gather_statement(...)``.  Returns float64 ``[T][K][K]``."""
    out = [(lambda y: y @ y.T)(dnc_gather_statement(w_agents, w_global, s, scales).double()) for s in samples]
    return torch.stack(out)


def _dnc_ranges(samples, lo, hi):
    """Per iteration, the positions ``[a, b)`` of the sorted sample rows that hold coordinates in ``[lo, hi)``, and the padded row
    length: the largest ``b - a`` rounded up to a multiple of 4 (at least 4)."""
    r = [(int(np.searchsorted(s, lo, "left")), int(np.searchsorted(s, hi, "left"))) for s in samples]
    longest = max(b - a for a, b in r)
    return r, max(4, (longest + 3) // 4 * 4)


def dnc_launch(table, K, w_global_ptr, samples, scales, out, dev, lo=0, hi=None, gate=(None, None, 0, 1, 0)):
    """DnC's device pass over the coordinates of ``samples`` (int64 numpy ``[T][S]``, rows sorted) that lie in ``[lo, hi)``: one
    ``dnc_gather_kernel`` launch behind ``gate`` (flag_ptrs, local_sync, rank, world, epoch) into ``Y [T][K][len_pad]``, then one
    ``history_gram`` launch per iteration into ``out[t]`` (float64 ``[T][K][K]``)."""
    samples = np.asarray(samples, dtype=np.int64)
    T = samples.shape[0]
    hi = int(samples.max(initial=-1)) + 1 if hi is None else int(hi)
    ranges, len_pad = _dnc_ranges(samples, lo, hi)
    samp = torch.from_numpy(samples.astype(np.int32)).to(dev)
    rng = torch.tensor(ranges, dtype=torch.int32).to(dev)
    y = torch.empty((T, K, len_pad), dtype=torch.float32, device=dev)
    rows = PtrTable([y[t, k].data_ptr() for t in range(T) for k in range(K)], dev, (y,))
    sc = torch.as_tensor(scales, dtype=torch.float32).to(dev) if scales is not None else None
    ext().dnc_gather(table, w_global_ptr, sc, samp, rng, y, *gate)
    for t in range(T):
        ext().history_gram(rows.tensor[t * K:(t + 1) * K], 0, len_pad, out[t])
    return out


def dnc_grams(w_agents, w_global, samples, n_vote=None, scales=None):
    """DnC's Gram matrices, float64 ``[T][K][K]`` (``dnc_gram_statement``'s values), of the participants' centred updates at the sorted
    coordinate samples ``samples`` (``[T][S]``, every coordinate ``< n_vote``).  ``scales``: the server-clipping scales or None.  On CUDA
    this launches ``dnc_gather_kernel`` and one ``pairwise_sqdist_kernel<true, true>`` per iteration (ops/csrc/select.cu); on CPU, and for
    more participants than the kernels' tables hold (recorded as a library fall-through), it evaluates ``dnc_gram_statement``."""
    nv = w_global.numel() if n_vote is None else int(n_vote)
    samples = np.asarray(samples, dtype=np.int64).reshape(len(samples), -1)
    if samples.size and (samples.min() < 0 or samples.max() >= nv):
        raise ValueError(f"DnC sample coordinates must lie in [0, n_vote={nv})")
    if nv >= 1 << 31:
        raise ValueError(f"DnC samples int32 coordinates: n_vote {nv} >= 2^31")
    for w in (*w_agents, w_global):
        if w.numel() < nv:
            raise ValueError(f"a flat buffer of {w.numel()} values for n_vote {nv}")
    K, T = len(w_agents), samples.shape[0]
    # the gather reads only the sampled coordinates, so n_vote need not be a multiple of 4 (the lengths were checked above)
    return _participant_pass("dnc_grams", w_agents, (w_global,), 0, (T, K, K),
                             lambda: dnc_gram_statement(w_agents, w_global, samples, scales),
                             lambda tab, out: dnc_launch(tab, K, w_global.data_ptr(), samples, scales, out, out.device, 0, nv))


def dnc_scores(C):
    """DnC's outlier scores of one iteration from its Gram matrix ``C = Y Y^T`` (float64 ``[K][K]``), on the host in fp64: with ``(lam, u)``
    the top eigenpair of ``C`` (``numpy.linalg.eigh``), ``s_k = lam * u_k^2`` -- the squared projection ``<Y_k, v>^2`` of the centred update
    onto the top right singular vector ``v`` of ``Y``.  A participant whose ``C_kk`` is not finite scores +inf and the others are scored on
    their own block of ``C``; a NaN score counts as +inf.  Returns float64 numpy ``[K]``."""
    c = np.asarray(torch.as_tensor(C).detach().double().cpu().numpy(), dtype=np.float64)
    K = c.shape[0]
    s = np.full(K, np.inf)
    ok = np.flatnonzero(np.isfinite(np.diag(c)))
    sub = c[np.ix_(ok, ok)]
    if ok.size and np.all(np.isfinite(sub)):
        lam, u = np.linalg.eigh(sub)
        s[ok] = lam[-1] * u[:, -1] ** 2
    s[np.isnan(s)] = np.inf
    return s


def dnc_select(grams, ids, f, c):
    """DnC admission on the host, shared by every path: for each iteration's Gram matrix (``grams[t]``) the ``K - floor(c f)`` positions
    with the lowest ``dnc_scores`` are kept, ties to the lower id in ``ids``; the admitted set is the intersection over the iterations.
    Returns the admitted positions (indices into ``ids``) in ascending order."""
    g = torch.as_tensor(grams).detach().double().cpu()
    K = len(ids)
    if g.dim() != 3 or tuple(g.shape[1:]) != (K, K):
        raise ValueError(f"dnc_select: Gram matrices of shape {tuple(g.shape)} for {K} participants")
    n_keep = K - math.floor(float(c) * int(f))
    if n_keep < 1:
        raise ValueError(f"DnC keeps K - floor(c F) >= 1 participants per iteration (K={K}, c={c}, F={f})")
    keep = set(range(K))
    for t in range(g.shape[0]):
        s = dnc_scores(g[t]).tolist()
        keep &= set(sorted(range(K), key=lambda k: (s[k], ids[k]))[:n_keep])
    return sorted(keep)


# =====================================================================================================================
# FLTrust (Cao, Fang, Liu, Gong, NDSS 2021): trust scores against the server's root update
# =====================================================================================================================
def trust_statement(w_agents, w_ref, w_global, lo, hi):
    """fp64 statement of the FLTrust statistics over coordinates ``[lo, hi)``: a float64 ``[2K + 1]`` tensor holding
    ``d_k = sum_c Δk[c] Δ0[c]`` (K values), ``q_k = sum_c Δk[c]^2`` (K values) and ``q0 = sum_c Δ0[c]^2``, with ``Δk = w_k - w_global``
    and ``Δ0 = w_ref - w_global``."""
    K = len(w_agents)
    dev = w_global.device
    out = torch.zeros(2 * K + 1, dtype=torch.float64, device=dev)
    step = max(4, (1 << 24) // max(1, K))                 # coordinates per pass: K * step fp64 values
    for c in range(lo, hi, step):
        e = min(hi, c + step)
        g = w_global[c:e].double()
        x = torch.stack([w[c:e] for w in w_agents]).double() - g
        d0 = w_ref[c:e].double() - g
        out[:K] += x @ d0
        out[K:2 * K] += (x * x).sum(1)
        out[2 * K] += (d0 * d0).sum()
    return out


def trust_stats(w_agents, w_ref, w_global, n_vote=None):
    """FLTrust statistics (``trust_statement``'s layout) of the participants ``w_agents`` against the root parameters ``w_ref`` over the
    voted coordinates ``[0, n_vote)`` (the BatchNorm running statistics behind ``n_vote`` do not count).  On CUDA this launches
    ``trust_stats_kernel`` (ops/csrc/trust.cu); on CPU, and for more participants than the kernel's tables hold (recorded as a library
    fall-through), it evaluates ``trust_statement``."""
    nv = w_global.numel() if n_vote is None else int(n_vote)
    return _participant_pass("trust_stats", w_agents, (w_ref, w_global), nv, (2 * len(w_agents) + 1,),
                             lambda: trust_statement(w_agents, w_ref, w_global, 0, nv),
                             lambda tab, out: ext().trust_stats(tab, w_ref.data_ptr(), w_global.data_ptr(), 0, nv, out,
                                                                None, None, 0, 1, 0))


def fltrust_weights(d, q, q0):
    """FLTrust trust scores and rescaling on the host, in fp64, shared by every path: ``TS_k = max(0, d_k / sqrt(q_k q0))`` (0 when
    ``q_k`` or ``q0`` is 0, or the cosine is NaN) and ``s_k = fp32(sqrt(q0 / q_k))`` (1 when ``q_k = 0``), which rescales update k to
    the root update's norm.  Returns ``(TS float64 [K], s float32 [K], admitted positions)``: the positions with ``TS > 0``,
    ascending."""
    d = np.asarray(torch.as_tensor(d).detach().double().cpu().numpy(), dtype=np.float64).reshape(-1)
    q = np.asarray(torch.as_tensor(q).detach().double().cpu().numpy(), dtype=np.float64).reshape(-1)
    q0 = float(q0)
    K = d.shape[0]
    ts = np.zeros(K, dtype=np.float64)
    sc = np.ones(K, dtype=np.float32)
    for k in range(K):
        qk = float(q[k])
        if qk > 0 and q0 > 0:
            c = float(d[k]) / math.sqrt(qk * q0)
            ts[k] = c if c > 0 else 0.0             # NaN -> 0
        if qk > 0:
            sc[k] = np.float32(math.sqrt(q0 / qk))
    return torch.from_numpy(ts), torch.from_numpy(sc), [k for k in range(K) if ts[k] > 0]


# =====================================================================================================================
# RFA (Pillutla, Kakade, Harchaoui, IEEE TSP 2022): the smoothed geometric median by Weiszfeld passes
# =====================================================================================================================
def rfa_statement(w_agents, b, lo, hi, w_global=None, scales=None):
    """fp64 statement of the RFA distance pass over coordinates ``[lo, hi)``: a float64 ``[K]`` tensor of
    ``d_k^2 = sum_c (x_k[c] - z[c])^2`` with ``z[c] = sum_j b_j x_j[c]`` (added in position order), ``x_k = w_k`` (no scales: ``w_global``
    cancels because the ``b_j`` sum to 1) or ``x_k = (w_k - w_global) * scales[k]``."""
    K = len(w_agents)
    dev = w_agents[0].device
    bt = torch.as_tensor(b, dtype=torch.float64).to(dev)
    sc = torch.as_tensor(scales, dtype=torch.float32).to(dev).double()[:, None] if scales is not None else None
    out = torch.zeros(K, dtype=torch.float64, device=dev)
    step = max(4, (1 << 24) // max(1, K))                 # coordinates per pass: K * step fp64 values
    for c in range(lo, hi, step):
        e = min(hi, c + step)
        x = torch.stack([w[c:e] for w in w_agents]).double()
        if sc is not None:
            x = (x - w_global[c:e].double()) * sc
        z = bt[0] * x[0]
        for j in range(1, K):
            z = z + bt[j] * x[j]
        out += ((x - z) ** 2).sum(1)
    return out


def rfa_sqdist(w_agents, b, n_vote=None, w_global=None, scales=None):
    """float64 ``[K]`` squared distances of the participants' updates to their ``b``-weighted mean over the voted coordinates
    ``[0, n_vote)`` (``rfa_statement``'s values; ``b`` sums to 1).  ``scales`` (server clipping) need ``w_global``.  On CUDA this launches
    ``rfa_sqdist_kernel`` (ops/csrc/rfa.cu); on CPU, and for more participants than the kernel's tables hold (recorded as a library
    fall-through), it evaluates ``rfa_statement``."""
    nv = w_agents[0].numel() if n_vote is None else int(n_vote)
    if scales is not None and w_global is None:
        raise ValueError("rfa_sqdist: scales need w_global")

    def launch(tab, out):
        sc = torch.as_tensor(scales, dtype=torch.float32).to(out.device) if scales is not None else None
        bt = torch.as_tensor(b, dtype=torch.float64).to(out.device)
        ext().rfa_sqdist(tab, bt, w_global.data_ptr() if sc is not None else 0, sc, 0, nv, out, None, None, 0, 1, 0)
    return _participant_pass("rfa_sqdist", w_agents, (w_global,) if scales is not None else (), nv, (len(w_agents),),
                             lambda: rfa_statement(w_agents, b, 0, nv, w_global, scales), launch)


def rfa_weights(alpha, d2, nu):
    """One smoothed Weiszfeld re-weighting on the host, in fp64: ``beta_k = alpha_k / max(nu, d_k)`` with ``d_k = sqrt(d2_k)``.  Returns
    float64 numpy ``[K]``."""
    a = np.asarray(alpha, dtype=np.float64).reshape(-1)
    d = np.sqrt(np.asarray(torch.as_tensor(d2).detach().double().cpu().numpy(), dtype=np.float64).reshape(-1))
    return a / np.maximum(float(nu), d)


def rfa(alpha, pass_fn, T, nu):
    """RFA's smoothed Weiszfeld loop, shared by every form of the server step.  ``alpha``: the participants' data sizes; ``pass_fn(b)``:
    the squared distances (float64 ``[K]``) of the updates to their ``b``-weighted mean, ``b`` a float64 numpy ``[K]`` summing to 1.
    ``T`` passes of ``b = beta / sum(beta)``, ``beta = rfa_weights(alpha, pass_fn(b), nu)`` from ``beta = alpha``.  Returns
    ``(beta, F)``: the final weights as a list of floats (``T = 0``: exactly ``alpha``) and, per pass, the objective
    ``F(z) = sum_k alpha_k ||z - x_k||`` at that pass's weighted mean ``z``.  While every distance is >= ``nu``, F does not increase
    from one pass to the next (the Weiszfeld property)."""
    a = np.asarray([float(x) for x in alpha], dtype=np.float64)
    beta = a.copy()
    F = []
    for _ in range(int(T)):
        d2 = pass_fn(beta / beta.sum())
        d = np.sqrt(np.asarray(torch.as_tensor(d2).detach().double().cpu().numpy(), dtype=np.float64).reshape(-1))
        F.append(float(np.dot(a, d)))
        beta = rfa_weights(a, d2, nu)
    return [float(x) for x in beta], F


# =====================================================================================================================
# FLAME (Nguyen et al., USENIX Security 2022): cosine clustering, median-norm clipping and adaptive noise
# =====================================================================================================================
def gram_statement(w_agents, w_global, lo, hi):
    """fp64 statement of the FLAME Gram pass over coordinates ``[lo, hi)``: a float64 ``[K][K]`` tensor of ``G[i][j] = sum_c Δi[c] Δj[c]``
    with ``Δk = w_k - w_global``; the diagonal holds the squared update norms."""
    K = len(w_agents)
    dev = w_global.device
    G = torch.zeros(K, K, dtype=torch.float64, device=dev)
    step = max(4, (1 << 24) // max(1, K))                 # coordinates per pass: K * step fp64 values
    for c in range(lo, hi, step):
        e = min(hi, c + step)
        x = torch.stack([w[c:e] for w in w_agents]).double() - w_global[c:e].double()
        G += x @ x.T
    return G


def pairwise_gram(w_agents, w_global, n_vote=None):
    """K x K float64 Gram matrix of the participants' updates ``w_k - w_global`` over the voted coordinates ``[0, n_vote)``
    (``gram_statement``'s values; the BatchNorm running statistics behind ``n_vote`` do not count).  On CUDA this launches
    ``pairwise_sqdist_kernel<true>`` (ops/csrc/select.cu); on CPU, and for more participants than the kernel's tables hold (recorded as a
    library fall-through), it evaluates ``gram_statement``."""
    nv = w_global.numel() if n_vote is None else int(n_vote)
    K = len(w_agents)
    return _participant_pass("pairwise_gram", w_agents, (w_global,), nv, (K, K), lambda: gram_statement(w_agents, w_global, 0, nv),
                             lambda tab, out: ext().pairwise_gram(tab, w_global.data_ptr(), 0, nv, out, None, None, 0, 1, 0))


def _first_cluster(d, m):
    """Single linkage on the symmetric distances ``d`` (float64 ``[n][n]``, +inf allowed): the vertices of the first connected component
    of at least ``m`` vertices in the graph of the edges ``d_ij <= h`` as ``h`` grows, all edges of one ``h`` taken together; [] when
    ``n < m``.  Those components are the ones of the minimum spanning tree's edges ``<= h``, so this is Prim's tree (O(n^2) in numpy)
    and a union-find over its ``n - 1`` edges."""
    n = d.shape[0]
    if n < m:
        return []
    if m <= 1:
        return list(range(n))
    in_tree = np.zeros(n, dtype=bool)
    in_tree[0] = True
    best, parent = d[0].copy(), np.zeros(n, dtype=np.int64)
    edges = []
    for _ in range(n - 1):
        out = np.flatnonzero(~in_tree)
        k = int(out[np.argmin(best[out])])
        edges.append((float(best[k]), int(parent[k]), k))
        in_tree[k] = True
        closer = d[k] < best
        parent[closer] = k
        best[closer] = d[k][closer]
    root, size = list(range(n)), [1] * n

    def find(x):
        while root[x] != x:
            root[x] = root[root[x]]
            x = root[x]
        return x
    edges.sort(key=lambda t: t[0])
    i, hit = 0, None
    while i < len(edges):
        h = edges[i][0]
        while i < len(edges) and edges[i][0] == h:
            a, b = find(edges[i][1]), find(edges[i][2])
            if a != b:
                root[b] = a
                size[a] += size[b]
                if size[a] >= m:
                    hit = a                # m > n / 2: at most one component ever reaches m
            i += 1
        if hit is not None:
            r = find(hit)
            return [k for k in range(n) if find(k) == r]
    return []


def flame_admit(G, ids, lam):
    """FLAME's admission, clip bound and noise on the host, in fp64, shared by every form of the server step.  ``G``: the Gram matrix of
    the candidates' updates (``gram_statement``'s layout); ``ids``: their agent ids; ``lam``: the noise factor lambda.

    ``e_k = sqrt(G_kk)``; ``cos_ij = G_ij / sqrt(G_ii G_jj)`` clamped to [-1, 1] (0 when a norm is 0); ``d_ij = 1 - cos_ij`` (NaN counts
    as +inf).  The admitted set is the first single-linkage cluster of at least ``m = K // 2 + 1`` candidates (``_first_cluster``) among
    those whose ``e_k`` is finite -- HDBSCAN(min_cluster_size=m, min_samples=1, allow_single_cluster=True) on these distances.  The pairs
    are read from the upper triangle in agent-id order, so the admitted ids do not depend on the candidates' positions.  The clip bound
    ``S`` is the median of every candidate's ``e_k`` (numpy's: the mean of the middle two for even K; NaN sorts as +inf) and
    ``s_k = fp32(min(1, S / e_k))`` (1 when ``e_k`` is 0 or NaN).  Returns ``(members, scales, S, noise_std)``: the admitted positions
    (ascending, possibly none), float32 ``[K]`` scales, ``S`` and ``noise_std = lam * S``."""
    g = np.asarray(torch.as_tensor(G).detach().double().cpu().numpy(), dtype=np.float64)
    K = g.shape[0]
    if g.shape != (K, K) or len(ids) != K:
        raise ValueError(f"flame_admit: a {g.shape} Gram matrix for {len(ids)} candidates")
    order = sorted(range(K), key=lambda k: ids[k])
    g = g[np.ix_(order, order)]
    g = np.triu(g) + np.triu(g, 1).T
    q = np.diag(g).copy()
    e = np.sqrt(q)
    with np.errstate(all="ignore"):
        nrm = np.sqrt(np.outer(q, q))
        d = 1.0 - np.clip(np.where(nrm > 0, g / np.where(nrm > 0, nrm, 1.0), 0.0), -1.0, 1.0)
    d[np.isnan(d)] = np.inf
    ok = np.flatnonzero(np.isfinite(e))
    cluster = _first_cluster(d[np.ix_(ok, ok)], K // 2 + 1)
    members = sorted(order[int(ok[j])] for j in cluster)
    e_pos = np.empty(K, dtype=np.float64)
    e_pos[order] = e
    S = float(np.median(np.where(np.isnan(e_pos), np.inf, e_pos)))
    scales = np.ones(K, dtype=np.float32)
    for k in range(K):
        if e_pos[k] > 0:
            scales[k] = np.float32(min(1.0, S / float(e_pos[k])))
    return members, torch.from_numpy(scales), S, float(lam) * S


# =====================================================================================================================
# FoolsGold (Fung, Yoon, Beschastnikh, RAID 2020): per-agent update histories kept across rounds
# =====================================================================================================================
def history_statement(rows, w_agents, w_global, lo, hi):
    """fp32 statement of the history update over coordinates ``[lo, hi)``: ``rows[k][c] + fp32(w_k[c] - w_global[c])``, each operation one
    fp32 rounding.  ``rows[k]`` is candidate k's history row, indexed by absolute coordinate.  Returns the new ``[lo, hi)`` slices."""
    g = w_global[lo:hi].float()
    return [h[lo:hi].float() + (w[lo:hi].float() - g) for h, w in zip(rows, w_agents)]


def history_accumulate(rows, w_agents, w_global, lo=0, hi=None):
    """Fold each candidate's update ``w_k - w_global`` into its history row ``rows[k]`` in place over ``[lo, hi)`` (default
    ``[0, len(rows[0]))``), bit for bit ``history_statement``.  On CUDA this launches ``history_accumulate_kernel``
    (ops/csrc/foolsgold.cu) for any number of candidates; on CPU it evaluates the statement."""
    hi = rows[0].numel() if hi is None else int(hi)
    lo = int(lo)
    if not rows[0].is_cuda:
        for h, new in zip(rows, history_statement(rows, w_agents, w_global, lo, hi)):
            h[lo:hi].copy_(new)
        return
    assert lo % 4 == 0 and hi % 4 == 0, "flat buffers are padded to multiples of 4"
    for t in (*rows, *w_agents, w_global):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() >= hi
    dev = w_global.device
    agents = PtrTable([w.data_ptr() for w in w_agents], dev, w_agents)
    tab = PtrTable([h.data_ptr() for h in rows], dev, rows)
    ext().history_accumulate(agents.tensor, tab.tensor, w_global.data_ptr(), lo, hi, None, None, 0, 1, 0)


def history_gram_statement(rows, lo, hi):
    """fp64 statement of the FoolsGold Gram pass over coordinates ``[lo, hi)``: ``G[i][j] = sum_c rows[i][c] rows[j][c]``."""
    K = len(rows)
    G = torch.zeros(K, K, dtype=torch.float64, device=rows[0].device)
    step = max(4, (1 << 24) // max(1, K))                 # coordinates per pass: K * step fp64 values
    for c in range(lo, hi, step):
        e = min(hi, c + step)
        x = torch.stack([h[c:e] for h in rows]).double()
        G += x @ x.T
    return G


def history_gram(rows, n_vote=None):
    """K x K float64 Gram matrix of the history rows over ``[0, n_vote)`` (``history_gram_statement``'s values).  On CUDA this launches
    ``pairwise_sqdist_kernel<true, true>`` (ops/csrc/select.cu); on CPU, and for more rows than the kernel's tables hold (recorded as a
    library fall-through), it evaluates ``history_gram_statement``."""
    nv = rows[0].numel() if n_vote is None else int(n_vote)
    K = len(rows)
    return _participant_pass("history_gram", rows, (), nv, (K, K), lambda: history_gram_statement(rows, 0, nv),
                             lambda tab, out: ext().history_gram(tab, 0, nv, out))


def foolsgold_weights(G):
    """FoolsGold's weights on the host, in fp64, shared by every form of the server step: the authors' released ``foolsgold()`` on the
    cosines of the candidates' histories, with its divisions by zero defined.  ``G``: the Gram matrix of the history rows
    (``history_gram_statement``'s layout).

    ``cs_ij = G_ij / sqrt(G_ii G_jj)`` clamped to [-1, 1] for ``i != j`` (0 when a norm is 0 or the cosine is NaN; a candidate whose
    ``G_kk`` is not finite has cosine 0 with everyone); ``v_i = max(0, max_{j != i} cs_ij)`` (0 for one candidate: the released code
    subtracts the identity from the cosines, so its row maxima include a diagonal 0); pardoning ``cs_ij *= v_i / v_j`` where
    ``v_i < v_j`` (so ``v_j > 0`` and the factor lies in [0, 1): a candidate anti-correlated with everyone has ``v_i = 0`` and its
    cosines are not turned positive); ``wv_i = clip(1 - max_{j != i} cs_ij, 0, 1)``.  When ``max wv = 0``
    every weight is 0; else ``wv /= max wv``, 1 becomes 0.99 and ``alpha_i = clip(ln(wv_i / (1 - wv_i)) + 0.5, 0, 1)`` (0 where
    ``wv_i = 0``).  A candidate with a non-finite ``G_kk`` gets 0.  Returns float64 numpy ``[K]``."""
    g = np.asarray(torch.as_tensor(G).detach().double().cpu().numpy(), dtype=np.float64)
    K = g.shape[0]
    if g.shape != (K, K):
        raise ValueError(f"foolsgold_weights: a {g.shape} Gram matrix")
    q = np.diag(g).copy()
    ok = np.isfinite(q)
    with np.errstate(all="ignore"):
        nrm = np.sqrt(np.outer(q, q))
        cs = np.where(nrm > 0, g / np.where(nrm > 0, nrm, 1.0), 0.0)
    cs = np.clip(np.nan_to_num(cs, nan=0.0), -1.0, 1.0)              # NaN -> 0; clip sends +-inf to +-1
    cs[~ok, :] = 0.0
    cs[:, ~ok] = 0.0
    off = ~np.eye(K, dtype=bool)
    v = np.maximum(np.where(off, cs, -np.inf).max(axis=1), 0.0) if K > 1 else np.zeros(1)
    vi, vj = v[:, None], v[None, :]
    pardon = off & (vi < vj)                                           # v_i >= 0, so v_j > 0 here
    cs = np.where(pardon, cs * vi / np.where(pardon, vj, 1.0), cs)
    top = np.where(off, cs, -np.inf).max(axis=1) if K > 1 else np.zeros(1)
    wv = np.clip(1.0 - top, 0.0, 1.0)
    alpha = np.zeros(K, dtype=np.float64)
    m = wv.max()
    if m > 0:
        wv = wv / m
        wv[wv == 1.0] = 0.99
        pos = wv > 0
        alpha[pos] = np.clip(np.log(wv[pos] / (1.0 - wv[pos])) + 0.5, 0.0, 1.0)
    alpha[~ok] = 0.0
    return alpha


# =====================================================================================================================
# FLDetector (Zhang, Cao, Jia, Gong, KDD 2022): predicted updates and the detection of agents far from their predictions
# =====================================================================================================================
FLD_REF_SETS = 10                        # B: uniform reference sets of the gap statistic
FLD_MAX_CLUSTERS = 10                    # the gap statistic tries k = 1 .. min(10, n - 1)
_FLD_GAP_TAG = 0x464C4447                # "FLDG": keeps the reference-set draws apart from every other stream seeded by --seed


def fld_ring_statement(w_g, w_prev, lo, hi):
    """fp32 statement of the ring pass over ``[lo, hi)``: the global update ``fp32(w_g[c] - w_prev[c])``."""
    return w_g[lo:hi].float() - w_prev[lo:hi].float()


def fld_ring(w_g, w_prev, s=None, lo=0, hi=None):
    """``s[lo:hi] <- fp32(w_g - w_prev)`` (skipped when ``s`` is None), then ``w_prev[lo:hi] <- w_g[lo:hi]``, in place.  ``w_prev`` and ``s``
    are indexed by absolute coordinate.  On CUDA this launches ``fld_ring_kernel`` (ops/csrc/fldetector.cu); on CPU it evaluates the
    statement."""
    hi = w_prev.numel() if hi is None else int(hi)
    lo = int(lo)
    if not w_g.is_cuda:
        if s is not None:
            s[lo:hi].copy_(fld_ring_statement(w_g, w_prev, lo, hi))
        w_prev[lo:hi].copy_(w_g[lo:hi])
        return
    for t in (w_g, w_prev) + ((s,) if s is not None else ()):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() >= hi
    ext().fld_ring(w_g.data_ptr(), w_prev.data_ptr(), s.data_ptr() if s is not None else 0, lo, hi)


def fld_hvp_statement(ring, coef, lo, hi):
    """Statement of the Hessian-vector product over ``[lo, hi)``: ``fp32(sum_i coef[i] * ring[i][c])`` with the sum in fp64 over the ring
    rows in the order given (chronological), every product and addition rounded on its own, and one rounding to fp32 at the end.  These
    bits are specified exactly.  Returns float32 ``[hi - lo]``."""
    acc = torch.zeros(hi - lo, dtype=torch.float64, device=ring[0].device)
    for c, s in zip(np.asarray(coef, dtype=np.float64).tolist(), ring):
        acc = acc + c * s[lo:hi].double()
    return acc.float()


def fld_hvp(ring, coef, lo=0, hi=None):
    """The Hessian-vector product ``Hv`` over ``[lo, hi)`` of the ring rows ``ring`` (chronological, indexed by absolute coordinate) with
    the coefficients ``coef`` of ``fld_hvp_coefficients``: float32 ``[hi - lo]``, bit for bit ``fld_hvp_statement``.  On CUDA this
    launches ``fld_hvp_kernel``; on CPU it evaluates the statement."""
    hi = ring[0].numel() if hi is None else int(hi)
    lo = int(lo)
    if not ring[0].is_cuda:
        return fld_hvp_statement(ring, coef, lo, hi)
    dev = ring[0].device
    for t in ring:
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() >= hi
    hv = torch.empty(hi - lo, dtype=torch.float32, device=dev)
    tab = PtrTable([t.data_ptr() for t in ring], dev, ring)
    ext().fld_hvp(tab.tensor, torch.as_tensor(np.asarray(coef, dtype=np.float64)).to(dev), hv.data_ptr() - 4 * lo, lo, hi)
    return hv


def fld_predict_statement(rows, w_agents, w_global, hv, lo, hi):
    """Statement of the prediction pass over ``[lo, hi)``: for candidate k the update ``u_k = fp32(w_k - w_global)``, and with ``hv``
    (``[hi - lo]``) the squared distance ``d_k^2 = sum_c fp32(fp32(rows[k][c] + hv[c]) - u_k[c])^2`` in fp64.  ``rows[k]`` is the
    candidate's last-update row, indexed by absolute coordinate.  Returns ``(new row slices u_k, float64 d^2 [K] or None)``."""
    g = w_global[lo:hi].float()
    us = [w[lo:hi].float() - g for w in w_agents]
    if hv is None:
        return us, None
    d2 = torch.stack([(((h[lo:hi].float() + hv) - u).double() ** 2).sum() for h, u in zip(rows, us)])
    return us, d2


def fld_predict(rows, w_agents, w_global, hv=None, lo=0, hi=None):
    """The prediction pass: with ``hv`` (``fld_hvp``'s ``[hi - lo]`` vector) return each candidate's fp64 squared distance to its
    prediction ``rows[k] + hv`` over ``[lo, hi)``; with or without it, then record ``rows[k][lo:hi] <- fp32(w_k - w_global)`` in place.
    Without ``hv`` it returns None.  On CUDA this launches ``fld_predict_kernel`` (``<true>`` with ``hv``, ``<false>`` without); on CPU,
    and for more candidates than the kernels' tables hold (recorded as a library fall-through), it evaluates ``fld_predict_statement``."""
    hi = rows[0].numel() if hi is None else int(hi)
    lo = int(lo)
    K = len(rows)

    def statement():
        us, d2 = fld_predict_statement(rows, w_agents, w_global, hv, lo, hi)
        for h, u in zip(rows, us):
            h[lo:hi].copy_(u)
        return d2 if d2 is not None else torch.zeros(K, dtype=torch.float64, device=rows[0].device)

    def launch(tab, out):
        dev = w_global.device
        rt = PtrTable([h.data_ptr() for h in rows], dev, rows)
        ext().fld_predict(tab, rt.tensor, w_global.data_ptr(), hv.data_ptr() - 4 * lo if hv is not None else 0, lo, hi,
                          out if hv is not None else None, None, None, 0, 1, 0)
        if hv is None:
            out.zero_()

    d2 = _participant_pass("fld_predict", list(w_agents), (w_global, *rows), hi, (K,), statement, launch)
    return d2 if hv is not None else None


def fld_hvp_coefficients(G):
    """L-BFGS Hessian-vector product of FLDetector on the host, in fp64: ``G`` is the ``(N + 1) x (N + 1)`` Gram matrix of the ring
    ``s_{r-N} .. s_r`` (chronological).  With ``S = [s_{r-N} .. s_{r-1}]``, ``Y = [y_i = s_{i+1} - s_i]``, ``v = s_r``,
    ``sigma = y_{r-1}.s_{r-1} / s_{r-1}.s_{r-1}``, ``L`` the strictly lower triangle of ``S^T Y`` and ``D = diag(S^T Y)``, it solves
    ``[[sigma S^T S, L], [L^T, -D]] q = [sigma S^T v; Y^T v]`` and writes ``Bv = sigma v - sigma S q1 - Y q2`` as ``sum_i c_i s_i``.
    Returns ``c`` (float64 numpy ``[N + 1]``).  Fallback -- ``s_{r-1}.s_{r-1} = 0``, a singular system or anything non-finite -- gives
    ``c = 0`` (the prediction is the last update); an all-zero ``c`` marks it."""
    g = np.asarray(torch.as_tensor(G).detach().double().cpu().numpy(), dtype=np.float64)
    n1 = g.shape[0]
    if g.ndim != 2 or g.shape != (n1, n1) or n1 < 2:
        raise ValueError(f"fld_hvp_coefficients: a {g.shape} Gram matrix (need (N + 1) x (N + 1), N >= 1)")
    N = n1 - 1
    zero = np.zeros(n1, dtype=np.float64)
    A_S = np.eye(n1, N)                                       # S = R A_S over the ring basis R
    A_Y = np.eye(n1, N, -1) - np.eye(n1, N)                   # y_i = s_{i+1} - s_i
    e_v = np.eye(n1)[:, N]
    with np.errstate(all="ignore"):
        StS, StY = A_S.T @ g @ A_S, A_S.T @ g @ A_Y
        Stv, Ytv = A_S.T @ g @ e_v, A_Y.T @ g @ e_v
        ss = StS[N - 1, N - 1]
        if not np.all(np.isfinite(g)) or not ss != 0:
            return zero
        sigma = StY[N - 1, N - 1] / ss
        L, D = np.tril(StY, -1), np.diag(np.diag(StY))
        M = np.block([[sigma * StS, L], [L.T, -D]])
        try:
            q = np.linalg.solve(M, np.concatenate([sigma * Stv, Ytv]))
        except np.linalg.LinAlgError:
            return zero
        c = sigma * e_v - sigma * (A_S @ q[:N]) - A_Y @ q[N:]
    return c if np.all(np.isfinite(c)) and np.isfinite(sigma) else zero


def fld_kmeans_sse(x, kmax):
    """Exact 1-D k-means: the least within-cluster sum of squares ``W_k`` of the sorted values ``x`` in ``k = 1 .. kmax`` contiguous
    groups, by dynamic programming over split points (deterministic; no k-means++).  A group whose values are all equal costs exactly 0.
    Returns float64 ``[kmax]`` (``W_1 .. W_kmax``)."""
    x = np.asarray(x, dtype=np.float64)
    n = x.size
    p1 = np.concatenate([[0.0], np.cumsum(x)])
    p2 = np.concatenate([[0.0], np.cumsum(x * x)])

    def cost(a, b):                          # SSE of x[a:b] for arrays of a (b fixed), b > a
        m = b - a
        c = (p2[b] - p2[a]) - (p1[b] - p1[a]) ** 2 / m
        return np.where(x[a] == x[b - 1], 0.0, np.maximum(c, 0.0))

    W = np.empty(kmax, dtype=np.float64)
    prev = np.array([cost(np.array([0]), b)[0] for b in range(1, n + 1)])     # prev[b - 1] = W_1 of x[:b]
    W[0] = prev[n - 1]
    for k in range(2, kmax + 1):
        cur = np.full(n, np.inf)
        for b in range(k, n + 1):
            a = np.arange(k - 1, b)          # the last group is x[a:b], the first a values form k - 1 groups
            cur[b - 1] = np.min(prev[a - 1] + cost(a, b))
        prev = cur
        W[k - 1] = prev[n - 1]
    return W


def fld_two_means(x):
    """The optimal split of the sorted values ``x`` (n >= 2) into two contiguous groups by exact 2-means: the index ``i`` in ``[1, n)``
    that minimises ``SSE(x[:i]) + SSE(x[i:])``, the lowest one on a tie."""
    x = np.asarray(x, dtype=np.float64)
    n = x.size
    sse = [float(np.sum((x[:i] - x[:i].mean()) ** 2) + np.sum((x[i:] - x[i:].mean()) ** 2)) for i in range(1, n)]
    return 1 + int(np.argmin(sse))


def fld_gap_clusters(z, seed, rnd):
    """FLDetector's gap statistic on the values ``z`` in [0, 1]: ``W_k`` the exact 1-D k-means SSE, ``k = 1 .. K_max = min(10, n - 1)``,
    B = 10 uniform reference sets of n points in [0, 1] from a numpy Generator seeded by (seed, round) alone, ``Gap(k) = mean_b log W_kb -
    log W_k`` and ``sd_k = std_b(log W_kb) sqrt(1 + 1/B)`` (a zero W counts as the smallest positive double).  Returns the smallest
    ``k < K_max`` with ``Gap(k) >= Gap(k + 1) - sd_{k + 1}``, else ``K_max``."""
    z = np.sort(np.asarray(z, dtype=np.float64))
    n = z.size
    kmax = min(FLD_MAX_CLUSTERS, n - 1)
    if kmax < 1:
        return 1
    tiny = np.nextafter(0.0, 1.0)
    logw = np.log(np.maximum(fld_kmeans_sse(z, kmax), tiny))
    ref = np.random.default_rng([int(seed), int(rnd), _FLD_GAP_TAG]).random((FLD_REF_SETS, n))
    logr = np.stack([np.log(np.maximum(fld_kmeans_sse(np.sort(r), kmax), tiny)) for r in ref])
    gap = logr.mean(axis=0) - logw
    sd = logr.std(axis=0) * math.sqrt(1.0 + 1.0 / FLD_REF_SETS)
    for k in range(1, kmax):
        if gap[k - 1] >= gap[k] - sd[k]:
            return k
    return kmax


def fld_detect(scores, seed, rnd):
    """FLDetector's decision on the host, shared by every form of the server step: ``scores`` are the candidates' suspicious scores.
    They are min-max normalised to z (all equal: no attack); when the gap statistic (``fld_gap_clusters``) finds more than one cluster,
    sorted z is split by exact 2-means (``fld_two_means``) and the upper group is flagged if it holds fewer than half of the candidates.
    Returns ``(flagged positions in scores, ascending; k_hat)``."""
    s = np.asarray(scores, dtype=np.float64)
    n = s.size
    if n == 0 or not np.all(np.isfinite(s)) or s.max() == s.min():
        return [], 1
    z = (s - s.min()) / (s.max() - s.min())
    khat = fld_gap_clusters(z, seed, rnd)
    if khat <= 1:
        return [], khat
    order = np.argsort(z, kind="stable")
    i = fld_two_means(z[order])
    upper = order[i:]
    if 2 * upper.size >= n:
        return [], khat
    return sorted(int(j) for j in upper), khat


# =====================================================================================================================
# model-poisoning attackers (DESIGN.md section 3)
# =====================================================================================================================
def mask_words(n: int) -> int:
    """Number of 32-bit words of a coordinate mask over ``n`` coordinates."""
    return (int(n) + 31) // 32


def mask_bits(words, n: int):
    """Bool tensor ``[n]`` of a coordinate mask stored as int32 bit words (bit ``c % 32`` of word ``c // 32`` = coordinate ``c``)."""
    shifts = torch.arange(32, dtype=torch.int32, device=words.device)
    return ((words.view(torch.int32)[:, None] >> shifts) & 1).flatten()[:int(n)].bool()


def neurotoxin_statement(w_g, w_prev, n_vote: int, k: int):
    """Neurotoxin's mask, stated in numpy: ``a[c] = bits(|fp32(w_g[c] - w_prev[c])|)`` for ``c < n_vote`` (the fp32 pattern with the
    sign bit cleared, so NaN sorts above +inf), ``tau`` = the k-th largest ``a`` counted with multiplicity, and
    ``M = {c : a[c] >= tau, a[c] > 0}`` (empty for ``k = 0``).  Returns ``(words, |M|)``: ``words`` is a uint32 array of
    ``mask_words(n_vote)`` words, bit ``c % 32`` of word ``c // 32`` set for ``c`` in M."""
    n_vote, k = int(n_vote), int(k)
    if not 0 <= k <= n_vote:
        raise ValueError(f"k = {k} must lie in [0, n_vote = {n_vote}]")
    g = w_g[:n_vote].detach().cpu().numpy().astype(np.float32, copy=False)
    p = w_prev[:n_vote].detach().cpu().numpy().astype(np.float32, copy=False)
    with np.errstate(invalid="ignore", over="ignore"):
        a = (g - p).view(np.uint32) & np.uint32(0x7FFFFFFF)
    m = np.zeros(mask_words(n_vote) * 32, dtype=bool)
    if k > 0:
        tau = np.partition(a, n_vote - k)[n_vote - k]
        m[:n_vote] = a >= max(int(tau), 1)
    return np.packbits(m, bitorder="little").view("<u4").astype(np.uint32), int(m.sum())


def neurotoxin_mask(w_g, w_prev, n_vote: int, k: int, mask, count):
    """Neurotoxin's mask of the last global update ``w_g - w_prev`` over ``[0, n_vote)`` (``neurotoxin_statement``): writes the
    ``mask_words(n_vote)`` int32 words of ``mask`` and ``|M|`` into the int64 ``count``, then refreshes ``w_prev[:n_vote] <- w_g``.
    On the GPU a radix select finds the threshold on the device: no host sync, bitwise reproducible."""
    if w_g.is_cuda:
        ext().neurotoxin_mask(w_g, w_prev, int(n_vote), int(k), mask, count)
        return
    words, c = neurotoxin_statement(w_g, w_prev, n_vote, k)
    mask[:words.size].copy_(torch.from_numpy(words.view(np.int32)))
    count.fill_(c)
    w_prev[:n_vote].copy_(w_g[:n_vote])


def sparsefed_statement(w, w_new, e, n_vote: int, k: int):
    """SparseFed's server step (Panda et al. 2022), stated in numpy, after the plain server step took ``w`` to ``w_new`` (both fp32
    ``[n]``; ``e`` is the fp32 error vector ``[n_vote]``):

    * ``u = fp32(w_new - w)`` and ``e' = fp32(e + u)`` over ``[0, n_vote)``;
    * ``key = bits(|e'|)`` (the fp32 pattern with the sign bit cleared, so NaN sorts above +inf) and ``tau`` = the k-th largest key,
      counted with multiplicity (``neurotoxin_statement``'s convention);
    * ``M = {c : key[c] >= max(tau, 1)}``: every tie at tau is taken, and an error of ±0 is never applied;
    * on M ``w'' = fp32(w + e')`` and ``e'' = 0``, elsewhere ``w'' = w`` and ``e'' = e'``; behind ``n_vote`` ``w'' = w_new``.

    Returns ``(w'' [n] fp32, e'' [n_vote] fp32, |M|, float(tau), ||e''||_2 in fp64)``.  ``1 <= k <= n_vote``."""
    n_vote, k = int(n_vote), int(k)
    if not 1 <= k <= n_vote:
        raise ValueError(f"k = {k} must lie in [1, n_vote = {n_vote}]")
    f32 = lambda t: (t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)).astype(np.float32, copy=False)
    w, wn, e = f32(w), f32(w_new), f32(e)[:n_vote]
    with np.errstate(invalid="ignore", over="ignore"):
        e1 = e + (wn[:n_vote] - w[:n_vote])
        key = e1.view(np.uint32) & np.uint32(0x7FFFFFFF)
        tau = np.partition(key, n_vote - k)[n_vote - k]
        m = key >= max(int(tau), 1)
        out = wn.copy()
        out[:n_vote] = np.where(m, w[:n_vote] + e1, w[:n_vote])
    e2 = np.where(m, np.float32(0.0), e1).astype(np.float32)
    norm = float(np.sqrt(np.sum(e2.astype(np.float64) ** 2)))
    return out, e2, int(m.sum()), float(np.uint32(tau).view(np.float32)), norm


def sparsefed_step(w, w_new, e, n_vote: int, k: int, stats, w_bf16=None):
    """SparseFed's step in place (``sparsefed_statement``): ``w`` (and its bf16 shadow ``w_bf16``, when given) becomes ``w''`` and ``e``
    becomes ``e''``; the float64 ``stats[:3]`` = ``(|M|, float(tau), ||e''||_2)``.  On the GPU the accumulate pass, the radix select and
    the apply pass queue without a host sync and are bitwise reproducible."""
    if w.is_cuda:
        ext().sparsefed(w_new, w, w_bf16, e, int(n_vote), int(k), stats)
        return
    out, e2, applied, tau, norm = sparsefed_statement(w, w_new, e, n_vote, k)
    w.copy_(torch.from_numpy(out))
    e[:int(n_vote)].copy_(torch.from_numpy(e2))
    if w_bf16 is not None:
        w_bf16.copy_(w.to(torch.bfloat16))
    stats[:3].copy_(torch.tensor([applied, tau, norm], dtype=torch.float64))


def sparsefed_k(p: float, n_params: int) -> int:
    """SparseFed's k for ``--server_topk p``: ``floor(p * n_params)``, as Neurotoxin sizes its mask.  Refuses ``p > 0`` with ``k = 0``."""
    k = math.floor(float(p) * int(n_params))
    if p > 0 and k < 1:
        raise ValueError(f"--server_topk {p} applies floor({p} x n_params {n_params}) = 0 coordinates; the smallest usable p is "
                         f"1/{n_params} = {1.0 / n_params:.3g}")
    return k


# =====================================================================================================================
# CRFL (Xie, Chen, Chen, Li, ICML 2021): clip and perturb the global model every round, certify it by parameter smoothing
# =====================================================================================================================
_CRFL_TRAIN_TAG = 0x3C6EF372FE94F82B     # domain tags of the training noise and the certification draws (SHA-512 IV words, like
_CRFL_CERT_TAG = 0xA54FF53A5F1D36F1      # _AUGMENT_TAG): keep both apart from every other Philox stream
CERTIFY_RATIOS = (0.0, 0.5, 1.0, 1.5, 2.0)   # R / sigma at which the certified accuracy is reported


def crfl_stream(index: int, certify: bool = False) -> int:
    """Philox stream word of CRFL's training noise in round ``index`` (``certify=False``) or of certification draw ``index``: a splitmix64
    hash of the domain tag and the index, in the style of ``augment_stream``.  Bit 63 is set, so the word is never an augmentation word
    (kept below 2^63) nor the aggregate noise's bare round number; bit 62 tells training from certification, so those two never meet.
    The key is ``--seed``; the counter is the coordinate / 4."""
    z = ((_CRFL_CERT_TAG if certify else _CRFL_TRAIN_TAG) + (int(index) + 1) * 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    z ^= z >> 31
    return (z & (2 ** 62 - 1)) | (1 << 63) | (int(bool(certify)) << 62)


def _i64(word: int) -> int:
    """An unsigned 64-bit word as the int64 the bindings take."""
    word = int(word) & _M64
    return word - 2 ** 64 if word >= 2 ** 63 else word


def real_mask(layout):
    """CRFL's real-coordinate mask of a ``FlatLayout``: int32 bit words over ``[0, n_vote)`` in Neurotoxin's format (bit ``c % 32`` of word
    ``c // 32``), set for the ``layout.n_params`` coordinates inside parameter tensors and clear on the alignment padding."""
    nv = int(layout.n_vote)
    m = np.zeros(mask_words(nv) * 32, dtype=bool)
    for p in layout.params:
        m[p.offset:p.offset + p.numel] = True
    return torch.from_numpy(np.packbits(m, bitorder="little").view("<u4").astype(np.uint32).view(np.int32).copy())


def philox_normals(seed: int, stream: int, n: int):
    """fp64 Box-Muller of the Philox words behind ``philox_normal4`` (common.cuh) for coordinates ``[0, n)`` (``n % 4 == 0``): counter
    c / 4, lane c % 4 = (r0 cos 2 pi u1, r0 sin 2 pi u1, r1 cos 2 pi u3, r1 sin 2 pi u3), r = sqrt(-2 ln u), u = ((x >> 8) + 1) / 2^24."""
    n4 = int(n) // 4
    u = philox4x32(np.arange(n4, dtype=np.uint64), stream, seed)
    unit = [((x >> np.uint32(8)).astype(np.float64) + 1.0) / 16777216.0 for x in u]
    r0, r1 = np.sqrt(-2.0 * np.log(unit[0])), np.sqrt(-2.0 * np.log(unit[2]))
    z = np.empty((n4, 4), dtype=np.float64)
    c1, s1 = _cos_sin_pi(2.0 * unit[1])
    c3, s3 = _cos_sin_pi(2.0 * unit[3])
    z[:, 0], z[:, 1], z[:, 2], z[:, 3] = r0 * c1, r0 * s1, r1 * c3, r1 * s3
    return z.reshape(-1)


def _cos_sin_pi(t):
    """``(cos(pi t), sin(pi t))`` in fp64 with exact argument reduction, as ``sincospif`` reduces: t = q/2 + f with q = rint(2 t) and
    |f| <= 1/4 exact, so the zeros at quarter turns are exact zeros."""
    q = np.rint(2.0 * t)
    f = t - 0.5 * q
    c, s = np.cos(np.pi * f), np.sin(np.pi * f)
    k = q.astype(np.int64) & 3
    cos = np.select([k == 0, k == 1, k == 2], [c, -s, -c], s)
    sin = np.select([k == 0, k == 1, k == 2], [s, c, -s], -c)
    return cos, sin


def crfl_statement(w_new, mask, n_vote: int, rho: float, sigma: float, seed: int, stream: int, z=None):
    """CRFL's clip-and-perturb pass in numpy, after the complete server step wrote ``w_new`` (fp32 ``[n]``); ``mask``: ``real_mask`` words.

    * ``q = sum w_new[c]^2`` in fp64 over the real coordinates (each square exact, the sum in numpy's fixed order);
    * ``s = 1`` if ``rho`` is 0 (no clip), ``q <= rho^2`` or ``q`` is not finite, else ``fp32(rho / sqrt(q))``;
    * on real coordinates ``w = fp32(fp32(w_new s) + fp32(fp32(sigma) z))`` with ``z = fp32(philox_normals)`` (or the given fp32 ``z``
      ``[n_vote]``), no noise term at ``sigma = 0``; every other coordinate keeps ``w_new``.

    Returns ``(w fp32 [n], sqrt(q), s)``."""
    n_vote = int(n_vote)
    wn = (w_new.detach().cpu().numpy() if torch.is_tensor(w_new) else np.asarray(w_new)).astype(np.float32, copy=True)
    words = mask.detach().cpu() if torch.is_tensor(mask) else torch.from_numpy(np.asarray(mask).view(np.int32))
    real = mask_bits(words, n_vote).numpy()
    v = wn[:n_vote]
    x = v[real].astype(np.float64)
    q = float(np.sum(x * x))
    s = np.float32(1.0)
    rho = float(rho)
    if rho > 0 and math.isfinite(q) and q > rho * rho:
        s = np.float32(rho / math.sqrt(q))
    with np.errstate(invalid="ignore", over="ignore"):
        o = np.where(real, v * s, v).astype(np.float32)
        if sigma > 0:
            zz = philox_normals(seed, stream, n_vote).astype(np.float32) if z is None else np.asarray(z, dtype=np.float32)[:n_vote]
            o = np.where(real, o + np.float32(sigma) * zz, o).astype(np.float32)
    wn[:n_vote] = o
    return wn, math.sqrt(q), float(s)


def crfl_step(w, w_new, mask, n_vote: int, rho: float, sigma: float, seed: int, rnd: int, stats, w_bf16=None):
    """CRFL's clip-and-perturb pass of round ``rnd`` (``crfl_statement`` with the stream ``crfl_stream(rnd)``): ``w`` (and its bf16 shadow,
    when given) becomes the clipped, perturbed ``w_new``; ``w`` may be ``w_new``.  ``rho = 0``: no clip.  The float64 ``stats[:2]`` =
    ``(sqrt(q), s)``.  On the GPU the norm, the ordered sum and the apply pass queue without a host sync."""
    stream = crfl_stream(rnd)
    if w.is_cuda:
        ext().crfl_clip_noise(w_new, w, w_bf16, mask, int(n_vote), float(rho) if rho > 0 else math.inf, float(sigma), _i64(seed),
                              _i64(stream), stats)
        return
    out, norm, s = crfl_statement(w_new, mask, n_vote, rho, sigma, seed, stream)
    w.copy_(torch.from_numpy(out))
    if w_bf16 is not None:
        w_bf16.copy_(w.to(torch.bfloat16))
    stats[:2].copy_(torch.tensor([norm, s], dtype=torch.float64))


def crfl_smooth(w, mask, n_vote: int, sigma: float, seed: int, m: int, out, out_bf16=None):
    """Parameters of certification draw ``m``: ``out = fp32(w + fp32(sigma z_m))`` on the real coordinates, ``w`` elsewhere, with
    ``z_m`` on the stream ``crfl_stream(m, certify=True)``; the bf16 shadow ``out_bf16`` (when given) is written in the same pass."""
    stream = crfl_stream(m, certify=True)
    if w.is_cuda:
        ext().crfl_smooth(w, out, out_bf16, mask, int(n_vote), float(sigma), _i64(seed), _i64(stream))
        return
    o, _, _ = crfl_statement(w, mask, n_vote, 0.0, sigma, seed, stream)
    out.copy_(torch.from_numpy(o))
    if out_bf16 is not None:
        out_bf16.copy_(out.to(torch.bfloat16))


def vote_count(logits, counts, row0: int = 0):
    """``counts[row0 + r][argmax(logits[r])] += 1`` for every row ``r`` of the fp32 ``[rows][classes]`` logits: the lowest class on ties,
    no vote for a row with a non-finite logit.  ``counts``: int32 ``[inputs][classes]``."""
    if logits.is_cuda:
        ext().vote_count(logits if logits.dtype == torch.float32 and logits.is_contiguous() else logits.float().contiguous(), counts,
                         int(row0))
        return
    x = logits.float()
    ok = torch.isfinite(x).all(1)
    rows = torch.arange(x.shape[0])[ok] + int(row0)
    counts.index_put_((rows, x.argmax(1)[ok]), torch.ones(rows.numel(), dtype=counts.dtype), accumulate=True)


def clopper_pearson_lower(k, n: int, alpha: float):
    """One-sided Clopper-Pearson lower bounds of ``k`` successes in ``n`` trials at level ``alpha``: the alpha-quantile of
    Beta(k, n - k + 1), i.e. the p with P(Bin(n, p) >= k) = alpha, and 0 for k = 0.  Bisection in fp64 on the exact binomial tail (log
    terms from ``lgamma``, summed with the largest factored out); the bisection keeps the side whose tail is <= alpha, so the bound is
    never above the exact quantile by more than the last interval.  ``k``: an integer or an array; returns a float64 array."""
    k = np.atleast_1d(np.asarray(k, dtype=np.int64))
    n = int(n)
    if np.any(k < 0) or np.any(k > n):
        raise ValueError(f"success counts must lie in [0, n = {n}]")
    out = np.zeros(k.shape, dtype=np.float64)
    pos = np.flatnonzero(k > 0)
    if pos.size == 0:
        return out
    lf = np.array([math.lgamma(j + 1.0) for j in range(n + 1)])
    j = np.arange(n + 1, dtype=np.float64)
    logc = lf[n] - lf - lf[::-1]
    la = math.log(alpha)
    step = max(1, (1 << 22) // (n + 1))
    for c0 in range(0, pos.size, step):
        kk = k[pos[c0:c0 + step]].astype(np.float64)[:, None]
        lo, hi = np.zeros(kk.shape[0]), np.ones(kk.shape[0])
        for _ in range(64):
            mid = 0.5 * (lo + hi)
            t = logc[None, :] + j[None, :] * np.log(mid)[:, None] + (n - j)[None, :] * np.log1p(-mid)[:, None]
            t = np.where(j[None, :] >= kk, t, -np.inf)
            mx = t.max(1)
            lt = mx + np.log(np.exp(t - mx[:, None]).sum(1))
            up = lt > la
            hi, lo = np.where(up, mid, hi), np.where(up, lo, mid)
        out[pos[c0:c0 + step]] = lo
    return out


def certify_decision(selection, estimation, n: int, alpha: float, sigma: float):
    """Cohen et al.'s CERTIFY on the vote counts of every input (int ``[inputs][classes]``: the selection draws and the ``n`` estimation
    draws): ``c = argmax(selection)`` (lowest class on ties), ``n_A = estimation[c]``, ``p_A = clopper_pearson_lower(n_A, n, alpha)``;
    predict c with radius ``R = sigma Phi^-1(p_A)`` when ``p_A > 1/2``, else abstain.  fp64 on the host, one bound per distinct ``n_A``.
    Returns ``(prediction int64 [inputs] (-1 = abstain), radius float64 [inputs], p_A float64 [inputs])``."""
    from statistics import NormalDist
    sel, est = np.asarray(selection), np.asarray(estimation)
    c = sel.argmax(1) if sel.shape[0] else np.zeros(0, dtype=np.int64)
    n_a = est[np.arange(est.shape[0]), c]
    uniq, inv = np.unique(n_a, return_inverse=True)
    pa_u = clopper_pearson_lower(uniq, n, alpha)
    inv_cdf = NormalDist().inv_cdf
    r_u = np.array([float(sigma) * inv_cdf(p) if p > 0.5 else 0.0 for p in pa_u], dtype=np.float64)
    pa, radius = pa_u[inv].reshape(-1), r_u[inv].reshape(-1)
    pred = np.where(pa > 0.5, c, -1).astype(np.int64)
    return pred, radius, pa


def certified_accuracy(pred, radius, labels, sigma: float, ratios=CERTIFY_RATIOS):
    """Share of inputs predicted correctly with a radius ``R >= r sigma``, for each ``r`` of ``ratios``."""
    pred, radius, labels = np.asarray(pred), np.asarray(radius), np.asarray(labels)
    if pred.size == 0:
        return [0.0 for _ in ratios]
    ok = pred == labels
    return [float(np.mean(ok & (radius >= r * float(sigma)))) for r in ratios]


# =====================================================================================================================
# FLARE (Wang, Xiao, Chen, Hu, Lou, Hou, ASIA CCS 2022): trust from the MMD between the candidates' root-set representations
# =====================================================================================================================
class FlareResult(NamedTuple):
    weights: np.ndarray        # float64 [K]: TS_j for the members of F, 0 for every other candidate
    members: list              # F: the positions of the candidates whose features are all finite (ascending)
    sigma2: float | None       # the pooled bandwidth sigma^2 (None when F pools fewer than two feature rows)
    M: np.ndarray | None       # float64 [|F|][|F|] MMD matrix over F (None when no MMD pass ran)
    counts: np.ndarray | None  # int64 [|F|] neighbour counts c_j (None when no MMD pass ran)


def flare_sigma2(Z, members):
    """FLARE's bandwidth (DESIGN.md section 3, step 4) in fp64 over the pooled feature rows of the candidates ``members``:
    ``sigma^2 = (2N sum ||z||^2 - 2 ||sum z||^2) / (N (N - 1))``, the mean squared distance over distinct pooled pairs, N = |members| n.
    None when N < 2."""
    K, n, d = Z.shape
    N = len(members) * n
    if N < 2:
        return None
    X = Z[torch.as_tensor(members, dtype=torch.int64, device=Z.device)].reshape(N, d).double()
    s1 = float((X * X).sum())
    v = X.sum(0)
    s2 = float((v * v).sum())
    return (2.0 * N * s1 - 2.0 * s2) / (N * (N - 1.0))


def flare_sums_statement(Z, finite, sigma2):
    """fp64 statement of the MMD pass: ``S[i][j] = sum_{a in Z_i, b in Z_j} exp(-||a - b||^2 / sigma^2)`` (float64 numpy ``[K][K]``,
    symmetric) between the finite candidates (``finite[k]``), 0 wherever a non-finite candidate takes part.  Distances are taken from
    direct differences in fp64."""
    K, n, d = Z.shape
    fin = [k for k in range(K) if bool(finite[k])]
    S = np.zeros((K, K), dtype=np.float64)
    if not fin:
        return S
    X = Z.double()
    for a, i in enumerate(fin):
        for j in fin[a:]:
            D = torch.cdist(X[i], X[j], compute_mode="donot_use_mm_for_euclid_dist") ** 2
            S[i, j] = S[j, i] = float(torch.exp(-D / float(sigma2)).sum())
    return S


def flare_sums(Z, finite, sigma2):
    """The MMD pass: ``flare_sums_statement``'s matrix.  On CUDA one launch of ``flare_mmd_kernel`` (ops/csrc/flare.cu) covers every pair
    (i <= j): fp32 distances from direct differences, expf, fp64 sums added in a fixed order (bitwise reproducible); on CPU it evaluates
    the statement."""
    K = Z.shape[0]
    if not Z.is_cuda:
        return flare_sums_statement(Z, finite.cpu().tolist(), sigma2)
    out = torch.empty(K * (K + 1) // 2, dtype=torch.float64, device=Z.device)
    ext().flare_mmd(Z.contiguous(), finite.to(torch.bool).contiguous(), 1.0 / float(sigma2), out)
    p = out.cpu().numpy()
    S = np.zeros((K, K), dtype=np.float64)
    iu = np.triu_indices(K)                                 # row by row: (0, 0), (0, 1), ..., (1, 1), ... as the kernel numbers its pairs
    S[iu] = p
    S.T[iu] = p
    return S


def flare_mmd_matrix(S, members, n: int):
    """FLARE's biased MMD estimates over the candidates ``members`` from the kernel sums ``S`` (``[K][K]``):
    ``M_ij = max(0, S_ii/n^2 + S_jj/n^2 - 2 S_ij/n^2)``, float64 numpy ``[|members|][|members|]``, symmetric with a zero diagonal."""
    idx = np.asarray(members, dtype=np.int64)
    s = np.asarray(S, dtype=np.float64)[np.ix_(idx, idx)]
    nn = float(n) * float(n)
    diag = np.diag(s) / nn
    return np.maximum(0.0, (diag[:, None] + diag[None, :]) - 2.0 * s / nn)


def flare_weights(M, ids, k=None, tau: float = 1.0):
    """FLARE's host half (DESIGN.md section 3, steps 6 and 7) in fp64, over the members of F listed by their positions ``ids``
    (ascending) with their MMD matrix ``M``.  ``k`` (default ``floor(|F|/2)``) is capped at ``|F| - 1``; ``NN(i)`` = the ``k`` other
    members with the smallest ``M_ij``, ties to the lower position; ``c_j`` counts the members whose neighbour lists hold j; ``TS_j =
    exp((c_j - max c)/tau) / sum_l exp((c_l - max c)/tau)``, the denominator added in position order.  Returns ``(TS float64 [|F|],
    c int64 [|F|])``."""
    M = np.asarray(M, dtype=np.float64)
    ids = np.asarray(ids, dtype=np.int64)
    F = len(ids)
    if F == 0:
        return np.zeros(0, dtype=np.float64), np.zeros(0, dtype=np.int64)
    k = F // 2 if k is None else int(k)
    k = max(0, min(k, F - 1))
    counts = np.zeros(F, dtype=np.int64)
    for i in range(F):
        others = np.asarray([j for j in range(F) if j != i], dtype=np.int64)
        if k and others.size:
            order = others[np.lexsort((ids[others], M[i, others]))]     # by M_ij, then by position
            counts[order[:k]] += 1
    e = np.exp((counts - counts.max()).astype(np.float64) / float(tau))
    tot = 0.0
    for v in e:
        tot += float(v)
    return e / tot, counts


def flare(Z, k=None, tau: float = 1.0, sums=None):
    """FLARE's weights (DESIGN.md section 3, steps 3 to 7 and the special cases) from the candidates' features ``Z`` (fp32 ``[K][n][d]``):
    F = the candidates whose features are all finite; ``|F| = 1``: weight 1, no MMD pass; sigma^2 (``flare_sigma2``) not finite or <= 0:
    weight 1/|F| each, no MMD pass; else the MMD pass ``sums(Z, finite, sigma^2)`` (default ``flare_sums``: the device kernel on CUDA),
    ``flare_mmd_matrix`` and ``flare_weights``.  ``|F| = 0`` returns zero weights (the caller runs the nobody-trusted step)."""
    K, n, d = Z.shape
    finite = torch.isfinite(Z.reshape(K, -1)).all(1)
    F = [j for j, f in enumerate(finite.cpu().tolist()) if f]
    w = np.zeros(K, dtype=np.float64)
    if not F:
        return FlareResult(w, F, None, None, None)
    s2 = flare_sigma2(Z, F)
    if len(F) == 1:
        w[F[0]] = 1.0
        return FlareResult(w, F, s2, None, None)
    if not (s2 is not None and math.isfinite(s2) and s2 > 0):
        w[F] = 1.0 / len(F)
        return FlareResult(w, F, s2, None, None)
    S = (sums or flare_sums)(Z, finite, s2)
    M = flare_mmd_matrix(S, F, n)
    ts, counts = flare_weights(M, F, k, tau)
    w[F] = ts
    return FlareResult(w, F, s2, M, counts)


def flare_statement(Z, k=None, tau: float = 1.0):
    """The fp64 statement of FLARE's weights: ``flare`` with the MMD pass evaluated by ``flare_sums_statement`` on any device."""
    return flare(Z, k, tau, sums=lambda z, fin, s2: flare_sums_statement(z, fin.cpu().tolist(), s2))


# =====================================================================================================================
# DeepSight (Rieger, Nguyen, Miettinen, Sadeghi, NDSS 2022): output-layer energy, random-input behaviour and per-cluster acceptance
# =====================================================================================================================
DEEPSIGHT_SEEDS = 3              # S: seeds of random inputs, one DDif clustering each


def deepsight_inputs(meta, seed: int, n: int, device, seeds: int = DEEPSIGHT_SEEDS):
    """DeepSight's random inputs: ``seeds`` blocks of ``n`` images of the dataset's shape, normalised NCHW fp32 ``[seeds n][C][H][W]``.
    Block s holds uniform uint8 pixels (uniform floats in [0, 1) when the dataset stores floats), drawn on the host from a generator
    seeded by ``(seed, s)`` alone -- identical on every rank, in every round and after a resume -- and normalised by the dataset's mean and
    std through ``gather_normalize``, like real images (no augmentation)."""
    raw = []
    for s in range(seeds):
        gen = torch.Generator().manual_seed((int(seed) * 1000003 + 7919 * (s + 1)) & 0x7FFFFFFFFFFFFFFF)
        shape = (int(n), meta.height, meta.width, meta.channels)
        raw.append(torch.rand(shape, generator=gen) if meta.is_float else torch.randint(0, 256, shape, generator=gen, dtype=torch.uint8))
    data = torch.cat(raw).to(device)
    return gather_normalize(data, torch.arange(data.shape[0], dtype=torch.int64, device=data.device), meta.mean, meta.std)


def _deepsight_lse(z):
    """fp64 log-sum-exp of the fp32 logits' last axis: ``max + log(sum_c exp(z_c - max))``, the sum over c ascending; NaN for a row with
    a non-finite logit."""
    z = np.asarray(z, dtype=np.float64)
    with np.errstate(all="ignore"):
        mx = z.max(axis=-1, keepdims=True)
        lse = mx[..., 0] + np.log(np.cumsum(np.exp(z - mx), axis=-1)[..., -1])
    return np.where(np.isfinite(z).all(axis=-1), lse, np.nan)


def deepsight_stats_statement(logits, g_logits, w_agents, w_global, head, seeds: int = DEEPSIGHT_SEEDS):
    """fp64 statement of the DeepSight statistics pass (DESIGN.md section 3).  ``logits``: fp32 ``[K][seeds N][P]`` eval-mode logits of the
    candidates on the random inputs, ``g_logits``: the global model's ``[seeds N][P]``; ``w_agents``: the candidates' flat parameters;
    ``head``: ``(w_off, b_off, P, d)`` of the last linear layer (``models.graph.head_slices``).  Returns float64 ``[K][(seeds + 2) P]``,
    per candidate ``DDif [seeds][P]`` (``(1/N) sum_m exp((z_k - lse z_k) - (z_g - lse z_g))``, m ascending), ``eps [P]`` (``|fp32(db_c)|``
    then ``|fp32(dW_cj)|`` for ascending j, added left to right) and ``db [P]``."""
    w_off, b_off, P, d = (int(v) for v in head)
    z = logits.detach().float().cpu().numpy()
    zg = g_logits.detach().float().cpu().numpy()
    K, SN, _ = z.shape
    N = SN // seeds
    with np.errstate(all="ignore"):
        a = z.astype(np.float64) - _deepsight_lse(z)[..., None]
        b = zg.astype(np.float64) - _deepsight_lse(zg)[..., None]
        terms = np.exp(a - b[None]).reshape(K, seeds, N, P)
        ddif = np.cumsum(terms, axis=2)[:, :, -1, :] / float(N)
    wg = w_global.detach().float().cpu().numpy()
    out = np.empty((K, (seeds + 2) * P), dtype=np.float64)
    for k, w in enumerate(w_agents):
        wk = w.detach().float().cpu().numpy()
        dW = (wk[w_off:w_off + P * d] - wg[w_off:w_off + P * d]).reshape(P, d)          # fp32 differences
        db = wk[b_off:b_off + P] - wg[b_off:b_off + P]
        terms = np.abs(np.concatenate([db[:, None], dW], axis=1).astype(np.float64))
        out[k, :seeds * P] = ddif[k].reshape(-1)
        out[k, seeds * P:(seeds + 1) * P] = np.cumsum(terms, axis=1)[:, -1]
        out[k, (seeds + 1) * P:] = db.astype(np.float64)
    return torch.from_numpy(out)


def deepsight_stats(logits, g_logits, w_agents, w_global, head, seeds: int = DEEPSIGHT_SEEDS):
    """The DeepSight statistics pass: ``deepsight_stats_statement``'s float64 ``[K][(seeds + 2) P]``.  On CUDA one ``deepsight_stats``
    launch pair (ops/csrc/deepsight.cu): one thread per output adding its terms in the stated order, bitwise reproducible; on CPU the
    statement."""
    if not logits.is_cuda:
        return deepsight_stats_statement(logits, g_logits, w_agents, w_global, head, seeds)
    w_off, b_off, P, d = (int(v) for v in head)
    K = logits.shape[0]
    tab = PtrTable([w.data_ptr() for w in w_agents], logits.device, w_agents)
    for w in (*w_agents, w_global):
        assert w.is_cuda and w.dtype == torch.float32 and w.is_contiguous() and w.numel() >= max(w_off + P * d, b_off + P)
    out = torch.empty((K, (seeds + 2) * P), dtype=torch.float64, device=logits.device)
    ext().deepsight_stats(logits.float().contiguous(), g_logits.float().contiguous(), tab.tensor, w_global.data_ptr(), w_off, b_off,
                          int(seeds), d, out)
    return out


def _prim_edges(d):
    """The ``n - 1`` edges ``(weight, u, v)`` of a minimum spanning tree of the symmetric distances ``d`` by Prim's algorithm (as in
    ``_first_cluster``).  Every minimum spanning tree has the same components under ``weight <= h`` for each h: those of ``{d <= h}``."""
    n = d.shape[0]
    in_tree = np.zeros(n, dtype=bool)
    in_tree[0] = True
    best, parent = d[0].copy(), np.zeros(n, dtype=np.int64)
    edges = []
    for _ in range(n - 1):
        out = np.flatnonzero(~in_tree)
        k = int(out[np.argmin(best[out])])
        edges.append((float(best[k]), int(parent[k]), k))
        in_tree[k] = True
        closer = d[k] < best
        parent[closer] = k
        best[closer] = d[k][closer]
    return edges


def _components(points, edges):
    """Connected components of ``points`` under ``edges`` (``(w, u, v)``), each a sorted list, ordered by their smallest point."""
    root = {p: p for p in points}

    def find(x):
        while root[x] != x:
            root[x] = root[root[x]]
            x = root[x]
        return x
    for _, u, v in edges:
        a, b = find(u), find(v)
        if a != b:
            root[max(a, b)] = min(a, b)
    comp = {}
    for p in sorted(points):
        comp.setdefault(find(p), []).append(p)
    return sorted(comp.values(), key=lambda c: c[0])


def hdbscan_labels(D, min_cluster_size: int):
    """HDBSCAN labels of the symmetric distances ``D`` (float64 ``[n][n]``, finite): scikit-learn's ``HDBSCAN(metric="precomputed",
    min_samples=1, min_cluster_size=m, allow_single_cluster=True)`` with equal distances entering together, so the labels do not depend
    on the order of the points.  Level by level from the top: at the largest distance h left inside a cluster, the clusters' points
    split into the connected components of ``{d < h}`` at lambda = 1/h (+inf for h = 0).  Two or more components of at least m points
    are new clusters born at lambda and the cluster ends; with one, the cluster goes on as it; the points of the smaller components leave
    at lambda.  The stability of a cluster is ``sum (lambda_leave - lambda_birth)`` over its points (the root is born at 0); excess of
    mass selects among every cluster, the root included; the points of a selected cluster take its label, and when the root is the one
    selected, only the points that leave it at its last lambda or later.  Every other point is noise (-1), as is a lone point.  Labels
    are numbered by their clusters' smallest point.  Returns int64 ``[n]``."""
    d = np.asarray(D, dtype=np.float64)
    n = d.shape[0]
    m = int(min_cluster_size)
    if m < 2:
        raise ValueError(f"hdbscan_labels: min_cluster_size {m} must be >= 2")
    labels = np.full(n, -1, dtype=np.int64)
    if n < 2:
        return labels
    birth, parent, stab, children, death = [0.0], [-1], [0.0], [[]], [0.0]
    leave = {}                                   # point -> (cluster it leaves, lambda)
    work = [(0, list(range(n)), _prim_edges(d))]
    while work:
        c, pts, edges = work.pop()
        while True:
            h = max(e[0] for e in edges)
            lam = 1.0 / h if h > 0 else math.inf
            kept = [e for e in edges if e[0] < h]
            comps = _components(pts, kept)
            big = [q for q in comps if len(q) >= m]
            for q in comps:
                if len(q) < m:
                    for p in q:
                        leave[p] = (c, lam)
                        stab[c] += lam - birth[c]
            death[c] = lam
            if len(big) >= 2:
                for q in big:
                    stab[c] += (lam - birth[c]) * len(q)
                    qs = set(q)
                    cid = len(birth)
                    birth.append(lam); parent.append(c); stab.append(0.0); children.append([]); death.append(lam)
                    children[c].append(cid)
                    work.append((cid, q, [e for e in kept if e[1] in qs]))
                break
            if not big:
                break
            pts = big[0]
            qs = set(pts)
            edges = [e for e in kept if e[1] in qs]
    n_cl = len(birth)
    selected = [False] * n_cl
    value = list(stab)
    for c in range(n_cl - 1, -1, -1):            # children are numbered after their parents
        sub = sum(value[ch] for ch in children[c])
        if sub > value[c]:
            value[c] = sub
        else:
            selected[c] = True
            todo = list(children[c])
            while todo:
                x = todo.pop()
                selected[x] = False
                todo.extend(children[x])
    for p in range(n):
        c, lam = leave[p]
        while c != -1 and not selected[c]:
            c = parent[c]
        if c > 0 or (c == 0 and lam >= death[0]):
            labels[p] = c
    out = np.full(n, -1, dtype=np.int64)
    names = {}
    for p in range(n):
        if labels[p] >= 0:
            out[p] = names.setdefault(int(labels[p]), len(names))
    return out


def _partition_indicator(labels):
    """``A[i][j] = 0`` when points i and j share a part of the partition of ``labels`` (every noise point, -1, its own part), 1 else."""
    lab = np.asarray(labels, dtype=np.int64)
    same = (lab[:, None] == lab[None, :]) & (lab[:, None] >= 0)
    A = np.where(same, 0, 1).astype(np.int64)
    np.fill_diagonal(A, 0)
    return A


def _pair_sum(f, X):
    """Symmetric float64 ``[n][n]`` of ``sum_c f(x_i, x_j)_c`` for the rows of ``X``, each sum left to right (content-only, so equal rows
    give equal entries wherever they stand)."""
    n = X.shape[0]
    out = np.zeros((n, n), dtype=np.float64)
    for i in range(n):
        if i + 1 < n:
            v = np.cumsum(f(X[i][None, :], X[i + 1:]), axis=1)[:, -1]
            out[i, i + 1:] = v
            out[i + 1:, i] = v
        out[i, i] = np.cumsum(f(X[i], X[i]))[-1] if X.shape[1] else 0.0
    return out


class DeepSightResult(NamedTuple):
    members: list              # A: the accepted positions (ascending)
    scales: torch.Tensor       # float32 [K]: s_k = fp32(min(1, S_clip / e_k)) (1 when e_k = 0 or k is not finite)
    clip_bound: float | None   # S_clip = median over F of e_k (None when F is empty)
    labels: np.ndarray         # int64 [K]: the final part of each candidate (numbered in agent-id order), -1 outside F
    suspicious: np.ndarray     # bool [K]: TE_k <= median_F(TE) / 2 (False outside F)
    te: np.ndarray             # int64 [K]: threshold exceedings (-1 outside F)
    finite: list               # F: the positions of the finite candidates (ascending)


def deepsight_decide(stats, norms, ids, tau: float, seeds: int = DEEPSIGHT_SEEDS):
    """DeepSight's decision on the host, in fp64 (DESIGN.md section 3), from the candidates' statistics ``stats`` (float64
    ``[K][(seeds + 2) P]``, ``deepsight_stats_statement``'s layout), their update norms ``norms`` (``[K]``) and agent ids ``ids``.
    The candidates are taken in agent-id order, so the result does not depend on their positions.  Returns a ``DeepSightResult``."""
    st = np.asarray(torch.as_tensor(stats).detach().double().cpu().numpy(), dtype=np.float64)
    e_all = np.asarray(torch.as_tensor(norms).detach().double().cpu().numpy(), dtype=np.float64).reshape(-1)
    K = st.shape[0]
    if len(ids) != K or e_all.shape[0] != K:
        raise ValueError(f"deepsight_decide: statistics of {K} candidates, {e_all.shape[0]} norms and {len(ids)} ids")
    P = st.shape[1] // (seeds + 2) if K else 0
    ddif = st[:, :seeds * P].reshape(K, seeds, P)
    eps = st[:, seeds * P:(seeds + 1) * P]
    db = st[:, (seeds + 1) * P:]
    with np.errstate(all="ignore"):
        e2 = eps * eps
        tot = np.cumsum(e2, axis=1)[:, -1] if P else np.zeros(K)
        neup = np.where(tot[:, None] > 0, e2 / np.where(tot > 0, tot, 1.0)[:, None], 0.0)
        top = neup.max(axis=1) if P else np.zeros(K)
        te = (neup > max(0.01, 1.0 / max(P, 1)) * top[:, None]).sum(axis=1).astype(np.int64)
    ok = np.isfinite(st).all(axis=1) & np.isfinite(neup).all(axis=1) & np.isfinite(e_all)
    F = sorted((k for k in range(K) if ok[k]), key=lambda k: ids[k])      # agent-id order
    labels = np.full(K, -1, dtype=np.int64)
    sus = np.zeros(K, dtype=bool)
    te_out = np.where(ok, te, -1)
    scales = np.ones(K, dtype=np.float32)
    if not F:
        return DeepSightResult([], torch.from_numpy(scales), None, labels, sus, te_out, [])
    Fi = np.asarray(F, dtype=np.int64)
    B = float(np.median(te[Fi])) / 2.0
    sus[Fi] = te[Fi] <= B
    with np.errstate(all="ignore"):
        x = db[Fi]
        G = _pair_sum(lambda a, b: a * b, x)
        q = np.diag(G).copy()
        nrm = np.sqrt(np.outer(q, q))
        d_cos = 1.0 - np.clip(np.where(nrm > 0, G / np.where(nrm > 0, nrm, 1.0), 0.0), -1.0, 1.0)
    np.fill_diagonal(d_cos, 0.0)
    euclid = lambda X: np.sqrt(_pair_sum(lambda a, b: (a - b) * (a - b), X))
    merged = seeds * _partition_indicator(hdbscan_labels(d_cos, 2)) + seeds * _partition_indicator(hdbscan_labels(euclid(neup[Fi]), 2))
    for s in range(seeds):
        merged = merged + _partition_indicator(hdbscan_labels(euclid(ddif[Fi, s]), 2))
    final = hdbscan_labels(merged.astype(np.float64), 2)
    parts = {}
    for j, lab in enumerate(final.tolist()):
        parts.setdefault(lab if lab >= 0 else -1 - j, []).append(j)     # a noise point is a part of its own
    accepted = []
    for pid, (key, q) in enumerate(sorted(parts.items(), key=lambda kv: kv[1][0])):
        for j in q:
            labels[F[j]] = pid
        if sum(int(sus[F[j]]) for j in q) / len(q) < float(tau):
            accepted.extend(F[j] for j in q)
    S_clip = float(np.median(e_all[Fi]))
    for k in F:
        if e_all[k] > 0:
            scales[k] = np.float32(min(1.0, S_clip / float(e_all[k])))
    return DeepSightResult(sorted(accepted), torch.from_numpy(scales), S_clip, labels, sus, te_out, sorted(F))


def deepsight_statement(logits, g_logits, w_agents, w_global, head, ids, tau: float, n_vote=None, seeds: int = DEEPSIGHT_SEEDS):
    """The fp64 statement of DeepSight's admission: ``deepsight_decide`` on ``deepsight_stats_statement`` and the fp64 update norms
    over the voted coordinates ``[0, n_vote)``."""
    nv = w_global.numel() if n_vote is None else int(n_vote)
    norms = torch.stack([(w[:nv].double() - w_global[:nv].double()).norm() for w in w_agents]).cpu()
    return deepsight_decide(deepsight_stats_statement(logits, g_logits, w_agents, w_global, head, seeds), norms, ids, tau, seeds)


def boost_statement(slot, w_g, gamma: float, n_vote: int):
    """The boosted update in numpy: ``fp32((double)w_g[c] + (double)gamma * (double)fp32(slot[c] - w_g[c]))`` for ``c < n_vote``,
    each fp64 operation rounded on its own.  Returns a float32 array ``[n_vote]``."""
    s = slot[:n_vote].detach().cpu().numpy().astype(np.float32, copy=False)
    g = w_g[:n_vote].detach().cpu().numpy().astype(np.float32, copy=False)
    with np.errstate(invalid="ignore", over="ignore"):
        d = (s - g).astype(np.float64)
        return (g.astype(np.float64) + np.float64(gamma) * d).astype(np.float32)


def boost_update(slot, w_g, gamma: float, n_vote: int):
    """Model replacement: scale the update in ``slot`` by ``gamma`` in place over ``[0, n_vote)`` (``boost_statement``); the
    BatchNorm running statistics behind ``n_vote`` are left alone."""
    if slot.is_cuda:
        ext().boost_update(slot, w_g, float(gamma), int(n_vote))
        return
    slot[:n_vote].copy_(torch.from_numpy(boost_statement(slot, w_g, gamma, n_vote)))


# ---- colluding attackers: ALIE (Baruch et al. 2019), Min-Max / Min-Sum (Shejwalkar and Houmansadr 2021) --------------------------------
COLLUDE_DIR_IDS = {"backdoor": 0, "std": 1, "sign": 2, "unit": 3}     # ColludeParams::dir of ops/csrc/collude.cu


def collude_z(H: int, C: int) -> float:
    """ALIE's default z for ``H`` honest and ``C`` corrupt participants: ``Phi^-1((K - s) / K)`` with ``K = H + C`` and
    ``s = max(1, floor(K / 2) + 1 - C)``, floored at 0."""
    from statistics import NormalDist
    K = int(H) + int(C)
    s = max(1, K // 2 + 1 - int(C))
    p = (K - s) / K if K > 0 else 0.0
    return max(0.0, NormalDist().inv_cdf(p)) if 0.0 < p < 1.0 else 0.0


def collude_gamma(mode: str, a, e, q, D) -> float:
    """The largest ``gamma >= 0`` for which ``m = mu - gamma u`` meets the Min-Max (``max_k ||m - x_k||^2 <= max_ij D_ij``) or Min-Sum
    (``sum_k ||m - x_k||^2 <= max_i sum_j D_ij``) constraint, in closed form in fp64 on the host.  ``a_k = ||mu - x_k||^2``,
    ``e_k = <mu - x_k, u>`` and ``q = ||u||^2`` over the H honest participants, ``D`` their squared-distance matrix.  Since
    ``||m - x_k||^2 = a_k - 2 gamma e_k + gamma^2 q``: Min-Max takes ``min_k (e_k + sqrt(e_k^2 + q (Dmax - a_k))) / q`` and Min-Sum
    ``(E + sqrt(E^2 + H q (S - A))) / (H q)`` with ``E = sum e_k``, ``A = sum a_k``.  A discriminant below 0 (rounding) counts as 0;
    ``q = 0``, a non-finite input or result, or a result below 0 gives 0."""
    if mode not in ("minmax", "minsum"):
        raise ValueError(f"collude_gamma: unknown mode {mode!r}")
    a = np.asarray(torch.as_tensor(a).double().cpu(), dtype=np.float64).reshape(-1)
    e = np.asarray(torch.as_tensor(e).double().cpu(), dtype=np.float64).reshape(-1)
    D = np.asarray(torch.as_tensor(D).double().cpu(), dtype=np.float64).reshape(a.size, a.size)
    q = float(q)
    if not (math.isfinite(q) and q > 0 and np.isfinite(a).all() and np.isfinite(e).all() and np.isfinite(D).all()):
        return 0.0
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if mode == "minmax":
            disc = np.maximum(e * e + q * (D.max() - a), 0.0)
            g = float(((e + np.sqrt(disc)) / q).min())
        else:
            E, A, Hq = float(e.sum()), float(a.sum()), a.size * q
            disc = E * E + Hq * (float(D.sum(1).max()) - A)
            g = (E + math.sqrt(max(disc, 0.0))) / Hq if math.isfinite(disc) else math.nan
    return g if (math.isfinite(g) and g > 0) else 0.0


def _collude_coords(honest, corrupt, w_g, lo, hi, direction, need_sig):
    """fp64 ``(g, x, fin, mu, sig, xc, u)`` over coordinates ``[lo, hi)``, every operation a separate torch op rounded on its own."""
    H = len(honest)
    g = w_g[lo:hi].double()
    x = torch.stack([w[lo:hi] for w in (*honest, *corrupt)]).double() - g
    fin = torch.isfinite(x)
    z = torch.zeros_like(g)
    s, n = z.clone(), fin[:H].sum(0)
    for j in range(H):
        s = torch.where(fin[j], s + x[j], s)
    mu = torch.where(n > 0, s / n.clamp(min=1).double(), z)
    sig = z
    if need_sig:
        v = z.clone()
        for j in range(H):
            d = x[j] - mu
            v = torch.where(fin[j], v + d * d, v)
        sig = torch.where(n >= 2, torch.sqrt(v / (n - 1).clamp(min=1).double()), z)
    xc = mu
    if direction == "backdoor":
        sc, nc = z.clone(), fin[H:].sum(0)
        for j in range(H, x.shape[0]):
            sc = torch.where(fin[j], sc + x[j], sc)
        xc = torch.where(nc > 0, sc / nc.clamp(min=1).double(), mu)
    u = {"std": lambda: sig, "sign": lambda: (mu > 0).double() - (mu < 0).double(), "unit": lambda: mu,
         "backdoor": lambda: mu - xc}[direction]()
    return g, x, fin, mu, sig, xc, u


def collude_statement(honest, corrupt, w_g, n_vote, mode, direction, z=None, gamma=None, D=None, lo=0, hi=None):
    """The colluding attackers' crafted update over coordinates ``[lo, hi)`` (default ``[lo, n_vote)``) in fp64, every operation rounded
    on its own (ops/csrc/collude.cu states the rule).  ``honest`` / ``corrupt``: the flat parameter vectors of the round's honest and
    corrupt participants, each in position order.  ``z`` (alie) defaults to ``collude_z``; ``gamma`` (minmax / minsum) defaults to
    ``collude_gamma`` on this statement's ``a``, ``e``, ``q`` and ``D`` (the honest squared distances, ``sqdist_statement``'s by default).
    Returns a dict: ``slot`` (fp32 ``[hi - lo]``, what every corrupt participant submits there), ``a`` / ``e`` (float64 ``[H]``), ``q``,
    ``dev2 = sum (m - mu)^2``, ``gamma`` and ``z``."""
    H, C = len(honest), len(corrupt)
    hi = int(n_vote) if hi is None else int(hi)
    dev = w_g.device
    alie = mode == "alie"
    if alie and z is None:
        z = collude_z(H, C)
    need_sig = alie or direction == "std"
    step = max(4, (1 << 24) // max(1, H + C))
    a = torch.zeros(H, dtype=torch.float64, device=dev)
    e = torch.zeros(H, dtype=torch.float64, device=dev)
    q = torch.zeros((), dtype=torch.float64, device=dev)
    if not alie:
        for c in range(lo, hi, step):
            _, x, fin, mu, _, _, u = _collude_coords(honest, corrupt, w_g, c, min(hi, c + step), direction, need_sig)
            d = torch.where(fin[:H], mu - x[:H], torch.zeros_like(x[:H]))
            a += (d * d).sum(1)
            e += (d * u).sum(1)
            q += (u * u).sum()
        if gamma is None:
            D = sqdist_statement(list(honest), lo, hi) if D is None else D
            gamma = collude_gamma(mode, a, e, q, D)
    slot = torch.empty(hi - lo, dtype=torch.float32, device=dev)
    dev2 = torch.zeros((), dtype=torch.float64, device=dev)
    for c in range(lo, hi, step):
        g, _, _, mu, sig, xc, u = _collude_coords(honest, corrupt, w_g, c, min(hi, c + step), direction, need_sig)
        if alie:
            t = float(z) * sig
            m = mu - t if direction == "std" else torch.minimum(torch.maximum(xc, mu - t), mu + t)
        else:
            m = mu - float(gamma) * u
        slot[c - lo:min(hi, c + step) - lo] = (g + m).float()
        dev2 += ((m - mu) ** 2).sum()
    return {"slot": slot, "a": a, "e": e, "q": float(q), "dev2": float(dev2), "gamma": None if alie else float(gamma),
            "z": float(z) if alie else None}


def collude_stats(honest, corrupt, w_g, n_vote, direction):
    """Min-Max / Min-Sum statistics pass: float64 ``[2H + 1]`` = ``(a_k, e_k, q)`` over ``[0, n_vote)`` (``collude_statement``'s values).
    On CUDA this launches ``collude_kernel<STATS>`` (ops/csrc/collude.cu); on CPU, and for more participants than the kernel's tables hold
    (recorded as a library fall-through), it evaluates the statement."""
    H = len(honest)
    nv = int(n_vote)

    def statement():
        st = collude_statement(honest, corrupt, w_g, nv, "minmax", direction, gamma=0.0)
        return torch.cat([st["a"], st["e"], torch.tensor([st["q"]], dtype=torch.float64, device=st["a"].device)])

    def launch(tab, out):
        ext().collude_stats(tab, H, w_g.data_ptr(), COLLUDE_DIR_IDS[direction], 0, nv, out, None, None, 0, 1, 0)
    return _participant_pass("collude_stats", [*honest, *corrupt], (w_g,), nv, (2 * H + 1,), statement, launch)


def collude_write(honest, corrupt, outs, w_g, n_vote, mode, direction, z=0.0, gamma=0.0):
    """Write pass: every buffer of ``outs`` (the corrupt participants' slots; they may be the ``corrupt`` inputs themselves) gets the
    crafted update over ``[0, n_vote)`` (``collude_statement``'s ``slot``, with ``z`` for alie and ``gamma`` for minmax / minsum); the
    BatchNorm statistics behind ``n_vote`` are left alone.  Returns float64 ``[1]`` = ``sum (m - mu)^2``.  On CUDA this launches
    ``collude_kernel<WRITE>`` (ops/csrc/collude.cu); on CPU, and for more participants than the kernel's tables hold (recorded as a
    library fall-through), it evaluates the statement."""
    H = len(honest)
    nv = int(n_vote)

    def statement():
        st = collude_statement(honest, corrupt, w_g, nv, mode, direction, z=z, gamma=gamma)
        for o in outs:
            o[:nv].copy_(st["slot"])
        return torch.tensor([st["dev2"]], dtype=torch.float64, device=w_g.device)

    def launch(tab, out):
        ot = PtrTable([o.data_ptr() for o in outs], out.device, list(outs)) if outs else None
        ext().collude_write(tab, H, ot.tensor if ot is not None else None, w_g.data_ptr(), 0 if mode == "alie" else 1,
                            COLLUDE_DIR_IDS[direction], float(z or 0.0), float(gamma or 0.0), 0, nv, out, None, None, 0, 1, 0)
    return _participant_pass("collude_write", [*honest, *corrupt], (w_g, *outs), nv, (1,), statement, launch)


def swap_samples(data, targets, idx, side_data, side_targets):
    """Attack schedules: exchange the dataset rows and labels at ``idx`` with the side copy in place, ``data[idx[i]] <-> side_data[i]``
    and ``targets[idx[i]] <-> side_targets[i]``.  The ``idx`` must be distinct (checked once, where the side copy is built), so the
    swap is its own inverse and every tensor keeps its address.  One launch on the GPU, none for an empty ``idx``."""
    if data.is_cuda:
        ext().swap_samples(data, targets, idx, side_data, side_targets)
        return
    x, y = data[idx], targets[idx]
    data[idx] = side_data
    targets[idx] = side_targets
    side_data.copy_(x)
    side_targets.copy_(y)


# =====================================================================================================================
# optimiser over flat buffers
# =====================================================================================================================
def round_init(w_global, w_local=None, w_bf16=None, mom=None):
    """Start of an agent's round: ``w_local <- w_global``, refresh the bf16 operand shadow, zero the momentum."""
    if w_global.is_cuda:
        ext().round_init(w_global, w_local, w_bf16, mom)
        return
    if w_local is not None:
        w_local.copy_(w_global)
    if w_bf16 is not None:
        w_bf16.copy_(w_global.to(torch.bfloat16))
    if mom is not None:
        mom.zero_()


def objective_gradient(g, w, w0, objective, n_pgd: int, masked=None):
    """The gradient ``G`` of the local objective ``a CE + b ||d|| + (mu/2) ||d||^2`` that ``FlatSGD`` applies, with ``g`` the
    cross-entropy gradient (Neurotoxin-masked already), ``objective = (a, b, mu)`` and ``d = w - w0`` over the model parameters
    ``[0, n_pgd)`` (the BatchNorm tail behind them never counts).  ``w`` is the parameters the step reads (``w_in`` on a first step).

    The statement, in fp64 unless a rounding ``r()`` to the buffers' dtype (fp32 in training) is written:

    * ``a, b, mu`` are taken at the buffers' precision: ``a = r(a)``, ``b = r(b)``, ``mu = r(mu)``;
    * ``d = r(w - w0)`` over ``[0, n_pgd)``, and ``d[c] = 0`` where the mask zeroes ``g[c]`` (a masked step never moves ``w`` off
      ``w0`` there, so this changes nothing in a run; it keeps ``G[c] = 0`` on the mask);
    * ``S_gg = sum g^2`` over every coordinate, ``S_gd = sum g d`` and ``S_dd = sum d^2`` over ``[0, n_pgd)``;
    * ``beta = b / sqrt(S_dd) + mu``, with ``b / sqrt(S_dd) := 0`` when ``S_dd = 0`` (the subgradient torch's norm backward takes at
      0; it covers the first step of every round, where ``d = 0``);
    * ``||G||^2 = max(0, a^2 S_gg + 2 a beta S_gd + beta^2 S_dd)``;
    * ``G = r(r(a g) + r(r(beta) d))`` over ``[0, n_pgd)`` and ``G = r(a g)`` behind it.

    Returns ``(G, ||G||, (S_gg, S_gd, S_dd))``.  The sm_90a kernels compute the three sums with fp32-squared ``g^2`` pairs and exact
    fp64 products for ``g d`` and ``d^2``, added in a fixed order, and every other step exactly as written here."""
    k = int(n_pgd)
    rnd = lambda x: float(torch.tensor(float(x), dtype=g.dtype))  # noqa: E731
    a, b, mu = (rnd(x) for x in objective)
    d = w[:k] - w0[:k]
    if masked is not None:
        d = d.masked_fill(masked, 0.0)
    s_gg = float((g.double() * g.double()).sum())
    s_gd = float((g[:k].double() * d.double()).sum())
    s_dd = float((d.double() * d.double()).sum())
    dn = math.sqrt(s_dd)
    beta = (b / dn if dn > 0 else 0.0) + mu
    G = g * a
    G[:k] += d * rnd(beta)
    return G, math.sqrt(max(0.0, a * a * s_gg + 2 * a * beta * s_gd + beta * beta * s_dd)), (s_gg, s_gd, s_dd)


class FlatSGD:
    """Fused ``clip_grad_norm_(., max_grad_norm)`` + momentum SGD + optional PGD projection over flat buffers.

    Reference: src/agent.py:37-38 (SGD, fresh momentum each round), :50 (clip 10), :54-60 (PGD onto the L2 ball of
    radius ``clip`` around the round's global params).  All norms stay on the device (the reference syncs to the host
    for ``max(1, norm/clip)``); the whole step is 2 kernels (+2 with PGD) regardless of the number of tensors.

    A local objective ``(a, b, mu)`` other than plain cross-entropy (FedProx, constrain-and-scale) replaces ``g`` by its gradient
    ``G`` (``objective_gradient``) ahead of the same chain: mask, ``clip_grad_norm_`` on ``||G||``, momentum SGD, PGD.  It takes
    the same launches: the norm pass also reads ``w`` and ``w0``, and the step ``w0``.
    """

    def __init__(self, n, device, lr, momentum, max_grad_norm=10.0, pgd_clip=0.0, n_pgd=None):
        self.lr, self.momentum, self.max_grad_norm, self.pgd_clip = float(lr), float(momentum), float(max_grad_norm), float(pgd_clip)
        # the PGD ball is measured and projected over the model parameters [0, n_pgd) only (layout.n_vote): BatchNorm running
        # statistics behind them are not in the reference's parameters_to_vector() (src/agent.py:54-60)
        self.n_pgd = int(n if n_pgd is None else n_pgd)
        # [||g||^2, ||w-w0||^2, S_gg, S_gd, S_dd]: the last three are the objective's norm pass (only a step with an objective writes
        # them, and its ||g||^2 is S_gg)
        self.norms = torch.zeros(5, dtype=torch.float64, device=device)

    def step(self, w, g, m, w0=None, w_bf16=None, w_in=None, grad_mask=None, objective=None):
        """``w_in``: first local step of a round fused with the hand-off -- parameters are read from ``w_in`` (the round's global
        parameters, i.e. the broadcast buffer) instead of ``w`` and the momentum counts as zero, so no separate
        ``w <- w_global, m <- 0`` pass is needed; coordinates ``>= n_pgd`` (BatchNorm running statistics already updated in ``w``
        by this step's forward pass) keep their value.

        ``grad_mask``: int32 bit words over ``[0, n_pgd)`` (Neurotoxin): ``g[c]`` counts as zero for every set bit, before the
        gradient norm is taken, and the PGD projection leaves those coordinates alone.  Same launches as without it.

        ``objective``: ``(a, b, mu)`` of the local objective ``a CE + b ||w - w0|| + (mu/2) ||w - w0||^2`` (``objective_gradient``),
        needs ``w0``; None or ``(1, 0, 0)`` is plain cross-entropy, the step as it is without the argument."""
        if objective is not None and tuple(float(x) for x in objective) == (1.0, 0.0, 0.0):
            objective = None
        if objective is not None and w0 is None:
            raise ValueError("FlatSGD.step: a local objective pulls toward w0, which is missing")
        if w.is_cuda:
            e = ext()
            e.memset_zero(self.norms)
            pgd = self.pgd_clip > 0
            if objective is not None:
                sums = self.norms[2:5]
                e.sqnorm(g, sums, grad_mask, self.n_pgd, w_in if w_in is not None else w, w0, self.n_pgd)
                e.sgd_step(w, g, m, w0, w_bf16, self.lr, self.momentum, self.max_grad_norm, sums, self.norms[1:2] if pgd else None,
                           self.n_pgd, w_in, grad_mask, [float(x) for x in objective])
                if pgd:
                    e.pgd_project(w, w0, w_bf16, self.pgd_clip, self.norms[1:2], self.n_pgd, grad_mask)
                return
            if grad_mask is None:
                e.sqnorm(g, self.norms[0:1])
                e.sgd_step(w, g, m, w0 if pgd else None, w_bf16, self.lr, self.momentum, self.max_grad_norm,
                           self.norms[0:1], self.norms[1:2] if pgd else None, self.n_pgd, w_in)
                if pgd:
                    e.pgd_project(w, w0, w_bf16, self.pgd_clip, self.norms[1:2], self.n_pgd)
                return
            e.sqnorm(g, self.norms[0:1], grad_mask, self.n_pgd)
            e.sgd_step(w, g, m, w0 if pgd else None, w_bf16, self.lr, self.momentum, self.max_grad_norm,
                       self.norms[0:1], self.norms[1:2] if pgd else None, self.n_pgd, w_in, grad_mask)
            if pgd:
                e.pgd_project(w, w0, w_bf16, self.pgd_clip, self.norms[1:2], self.n_pgd, grad_mask)
            return
        masked = None
        if grad_mask is not None:
            masked = mask_bits(grad_mask, self.n_pgd)
            g = g.clone()
            g[:self.n_pgd].masked_fill_(masked, 0.0)
        if objective is None:
            gn = float(g.double().norm())
        else:
            g, gn, _ = objective_gradient(g, w_in if w_in is not None else w, w0, objective, self.n_pgd, masked)
        coef = min(1.0, self.max_grad_norm / (gn + 1e-6)) if self.max_grad_norm > 0 else 1.0
        if w_in is not None:
            k = self.n_pgd
            m.zero_()
            m[:k].add_(g[:k], alpha=coef)
            w[:k].copy_(w_in[:k] - self.lr * m[:k])
        else:
            m.mul_(self.momentum).add_(g, alpha=coef)
            w.add_(m, alpha=-self.lr)
        if self.pgd_clip > 0:
            k = self.n_pgd
            d = w[:k] - w0[:k]
            denom = max(1.0, float(d.double().norm()) / self.pgd_clip)
            if denom > 1.0:
                proj = w0[:k] + d / denom
                w[:k].copy_(proj if masked is None else torch.where(masked, w[:k], proj))
        if w_bf16 is not None:
            w_bf16.copy_(w.to(torch.bfloat16))


# =====================================================================================================================
# loss / evaluation
# =====================================================================================================================
def softmax_xent(logits, labels, want_grad=True, loss_sum=None, correct=None, dlogits=None):
    """Fused softmax cross-entropy (mean reduction) forward + backward: returns ``(loss_sum_tensor, dlogits)`` where
    ``dlogits = (softmax - onehot) / B`` (SURVEY.md K7).  ``dlogits``: optional pre-allocated output of the logits' dtype and
    shape (the native executor passes its gradient buffer, so the loss kernel writes the head's gradient in place)."""
    B = logits.shape[0]
    if logits.is_cuda:
        dl = (dlogits if dlogits is not None else torch.empty_like(logits)) if want_grad else None
        if loss_sum is None:
            loss_sum = torch.zeros(1, dtype=torch.float32, device=logits.device)
        ext().softmax_xent(logits.contiguous(), labels, dl, loss_sum, correct, 1.0 / B)
        return loss_sum, dl
    lf = logits.float()
    lsm = torch.log_softmax(lf, dim=1)
    loss = -lsm.gather(1, labels[:, None]).sum()
    dl = None
    if want_grad:
        dl = (lsm.exp() - torch.nn.functional.one_hot(labels, lf.shape[1]).float()) / B
        dl = dl.to(logits.dtype)
        if dlogits is not None:
            dlogits.copy_(dl)
            dl = dlogits
    if loss_sum is None:
        loss_sum = torch.zeros(1)
    loss_sum += loss
    if correct is not None:
        correct += (lf.argmax(1) == labels).sum().to(correct.dtype)
    return loss_sum, dl


def eval_metrics(logits, labels, loss_sum, confusion):
    """Accumulate the summed per-sample loss and the confusion matrix ``confusion[true, pred]`` on the device
    (replaces the per-sample host loop of src/utils.py:144-152)."""
    if logits.is_cuda:
        ext().eval_metrics(logits.contiguous(), labels, loss_sum, confusion)
        return
    lf = logits.float()
    loss_sum += torch.nn.functional.cross_entropy(lf, labels, reduction="sum").double()
    C = lf.shape[1]
    pred = lf.argmax(1)
    confusion.view(-1).index_add_(0, labels * C + pred, torch.ones_like(labels))


from .nn import (avgpool_bwd, avgpool_fwd, bn_bwd, bn_fwd, conv2d_dgrad_sm100, conv2d_fwd_sm100, conv2d_wgrad_sm100, conv_supported,  # noqa: E402,F401
                 dropout_bwd, dropout_fwd, gn_bwd, gn_fwd, linear_bwd, linear_fused_dropout_ok, linear_fwd, maxpool2_bwd, maxpool2_fwd, relu_bwd_, scratch, stem_geometry, STAT_SLOTS)
