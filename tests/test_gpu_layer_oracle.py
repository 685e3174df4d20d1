"""Every memory-bound layer-kernel call against the fp64 statements of tests/layer_oracle.py, element by element: BatchNorm (statistics,
apply, two-pass backward, mask recompute), GroupNorm, ReLU backward, max / average pooling, stand-alone dropout and the dropout fused
into the pooling kernel, the wgmma GEMM epilogue and the split-K finishing pass.

* Harvested calls: one NativeNet training step of each of the ten zoo models at batch 256 and at the ragged last batches of an epoch
  (96 for FMNIST, 80 for CIFAR-10), with dropout left on, records each call and its flags (residual, ReLU, mask recompute, fused
  ReLU mask of the pooling backward, fused dropout); each distinct call is replayed alone on fresh data into NaN-prefilled,
  guard-banded outputs.
* Edges: the ends of the channel range (C = 8 ... 2048), 1 / 2 / 3 rows and one row-slot iteration +- 1, ragged reversed-walk tiles,
  multi-slot statistics and backward sums, evaluation mode, staged and unstaged GroupNorm tiles, odd-sized pooling over ties, dropout
  rates whose scale is not a power of two and step counters near 2^62.
* Whole step: the reference CNNs' gradients with dropout on against fp64 autograd with the same keep-masks, fused and stand-alone.

The last test asserts that every layer-kernel instantiation ran in a call the tests before it judged (run the whole file) and prints the
largest error each family needed against its bound."""
import math
from collections import defaultdict

import pytest
import torch

import layer_oracle as lo
import rlr_b200  # noqa: F401
from rlr_b200 import ops
from rlr_b200.models import get_layout
from rlr_b200.models import graph as graph_mod
from rlr_b200.models import native
from rlr_b200.models.native import NativeNet, dropout_stream_base
from rlr_b200.ops import nn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16
EPS, MOM, SEED = 1e-5, 0.1, 0

MODELS = ["resnet18", "resnet34", "vgg11", "vgg16", "cnn_cifar", "cnn_mnist", "resnet18_gn", "resnet34_gn", "vgg11_gn", "vgg16_gn"]
BATCHES = [256, 96, 80]
STEP_HI = dropout_stream_base(SEED, 3, 7)      # a step base as the trainer sets it (< 2^62)

SUMMARY = defaultdict(lambda: [0.0, 0.0, 0])   # family -> (largest kappa needed, largest mismatch fraction, checks)
KERNELS = set()                                # kernel names run by judged calls
DROP_GEMM = set()                              # kernel names run by judged linear calls with fused dropout
RATIO_REPORT = {}


def _profiled(fn, into=KERNELS):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        into.add(e.key)


def _judge(fails, family, r):
    s = SUMMARY[family]
    if r.kappa != math.inf:
        s[0] = max(s[0], r.kappa)
    s[1], s[2] = max(s[1], r.mismatch), s[2] + 1
    if not r.ok:
        fails.append((family, r))


def _exact(fails, family, got, want):
    SUMMARY[family][2] += 1
    if not torch.equal(got, want):
        bad = (got.float() != want.float()) & ~(got.float().isnan() & want.float().isnan())
        fails.append((family, f"{int(bad.sum())} of {bad.numel()} elements differ from the exact statement"))


def _guard(fails, family, buf):
    if not lo.guard_intact(buf):
        fails.append((family, "guard band written"))


def _guarded_u8(shape):
    n = math.prod(shape)
    buf = torch.full((n + lo.GUARD,), 0xAB, dtype=torch.uint8, device=DEV)
    return buf[:n].view(shape), buf


def _guard_u8(fails, family, buf):
    if not bool((buf[-lo.GUARD:] == 0xAB).all()):
        fails.append((family, "guard band written"))


def _step(v):
    return torch.tensor([int(v)], dtype=torch.int64, device=DEV)


def _assert_clean(fails):
    torch.cuda.synchronize()
    assert not fails, fails[:10]


def _act(shape, ratio=None, seed_off=0.0):
    """bf16 activations: per-channel offsets of up to 1 std (or exactly ``ratio`` std), per-channel scales."""
    C = shape[-1]
    off = torch.linspace(-1, 1, C, device=DEV) if ratio is None else torch.full((C,), float(ratio), device=DEV)
    sc = torch.rand(C, device=DEV) + 0.5
    return ((torch.randn(shape, device=DEV) + off + seed_off) * sc).to(BF)


# =====================================================================================================================
# BatchNorm
# =====================================================================================================================
def _bn_params(C):
    gamma, beta = torch.rand(C, device=DEV) + 0.5, torch.randn(C, device=DEV) * 0.2
    rm, rv = torch.randn(C, device=DEV) * 0.1, torch.rand(C, device=DEV) * 0.1      # small old running variance: see the unbiased factor
    return gamma, beta, rm, rv


def run_bn_fwd(fails, fam, M, C, relu, resid, slots=1, chunks=1, train=True, x=None):
    """channel_stats into ``slots`` slots (``chunks`` > 1: each slot the sums of one row chunk, as conv epilogues leave them) +
    bn_apply with the training finalize (fin.mode 1) or the running statistics (fin.mode 2).  Returns (x, y, mean_rstd, gamma, beta)."""
    e = ops.ext()
    x = _act((M, C)) if x is None else x
    gamma, beta, rm, rv = _bn_params(C)
    res = _act((M, C)) if resid else None
    y, yb = lo.guarded((M, C), BF, DEV)
    mr, mrb = lo.guarded((2, C), torch.float32, DEV)
    rm_k, rmb = lo.guarded((C,), torch.float32, DEV)
    rv_k, rvb = lo.guarded((C,), torch.float32, DEV)
    rm_k.copy_(rm); rv_k.copy_(rv)
    stats = torch.zeros(max(slots, chunks), 2, C, device=DEV)
    f = ("bn_fwd " if train else "bn_eval ") + fam
    if train:
        if chunks > 1:
            bounds = torch.linspace(0, M, chunks + 1).long().tolist()
            for k in range(chunks):
                if bounds[k + 1] > bounds[k]:
                    e.channel_stats(x[bounds[k]:bounds[k + 1]], stats[k:k + 1])
        else:
            e.channel_stats(x, stats)
        e.bn_apply(x, res, y, gamma, beta, mr, bool(relu), 1, stats, float(M), EPS, MOM, rm_k, rv_k)
        torch.cuda.synchronize()
        _judge(fails, "bn_stats " + fam, lo.check_stats(fam, stats, x, lo.KAPPA_CSTATS))
        d1, d2 = lo.stat_slots_bound(stats)
        s = stats.double().sum(0)
        for r in lo.check_fin(fam + " own", lo.bn_finalize(s[0], s[1], M, EPS, MOM, rm, rv, d1, d2), mr, rm_k, rv_k):
            _judge(fails, "bn_fin " + fam, r)
        xd = x.double()
        tb = lo.KAPPA_STATS * lo.U * (math.sqrt(M) + 1)
        truth = lo.bn_finalize(xd.sum(0), (xd * xd).sum(0), M, EPS, MOM, rm, rv, tb * xd.abs().sum(0) + d1, tb * (xd * xd).sum(0) + d2)
        for r in lo.check_fin(fam + " truth", truth, mr, rm_k, rv_k):
            _judge(fails, "bn_fin_truth " + fam, r)
        v, unit = lo.affine_statement(x, mr[0], mr[1], gamma, beta, res)
        _guard(fails, f, mrb)
    else:
        e.bn_apply(x, res, y, gamma, beta, mr, bool(relu), 2, None, float(M), EPS, MOM, rm_k, rv_k)
        torch.cuda.synchronize()
        _exact(fails, f + " running stats untouched", torch.stack([rm_k, rv_k]), torch.stack([rm, rv]))
        fin = lo.bn_eval(rm, rv, EPS)
        v, unit = lo.affine_statement(x, fin.mean, fin.rstd, gamma, beta, res, u_rstd=fin.u_rstd)
    _judge(fails, f, lo.check_value(fam, y, v, unit, lo.epi_relu(relu)))
    for b in (yb, rmb, rvb):
        _guard(fails, f, b)
    return x, y, mr, gamma, beta, res


def run_bn_bwd(fails, fam, M, C, relu, resid, recompute, slots=1):
    """bn_bwd (y-read ReLU mask) or bn_bwd_recompute on the output of the forward kernels: dsum against fp64 truth, dgamma / dbeta from
    the kernel's own dsum, dx given its own dsum, dres exact."""
    e = ops.ext()
    x, y, mr, gamma, beta, res = run_bn_fwd(fails, fam, M, C, relu, resid)
    mean_rstd = mr.clone()
    dy = _act((M, C))
    dsum = torch.full((slots, 2, C), float("nan"), device=DEV)           # zero_dsum: the binding clears it
    dx, dxb = lo.guarded((M, C), BF, DEV)
    dres, drb = lo.guarded((M, C), BF, DEV) if resid else (None, None)
    dg, dgb = lo.guarded((C,), torch.float32, DEV)
    db, dbb = lo.guarded((C,), torch.float32, DEV)
    if recompute:
        e.bn_bwd_recompute(dy, x, gamma, beta, mean_rstd, dsum, dx, dg, db, True)
    else:
        e.bn_bwd(dy, y, x, gamma, mean_rstd, dsum, dx, dres, dg, db, bool(relu), True)
    torch.cuda.synchronize()
    f = ("bn_bwd_recompute " if recompute else "bn_bwd ") + fam
    mask = (y.double() > 0) if relu else torch.ones(M, C, dtype=torch.float64, device=DEV)
    terms, xhat = lo.bn_bwd_terms(dy, x, mask, mean_rstd)
    _judge(fails, "bn_dsum " + fam, lo.check_sums(fam, dsum, terms, rounding=3))
    wg, wb, ug, ub = lo.bn_param_grads(dsum)
    _judge(fails, "bn_dparam " + fam, lo.check_value(fam + " dgamma", dg, wg, ug))
    _judge(fails, "bn_dparam " + fam, lo.check_value(fam + " dbeta", db, wb, ub))
    v, unit = lo.bn_dx_statement(terms[0], xhat, gamma, mean_rstd, dsum)
    _judge(fails, f, lo.check_value(fam, dx, v, unit, lo.rn_bf16))
    if resid:
        _exact(fails, "bn_dres " + fam, dres, terms[0].to(BF))
    for b in (dxb, drb, dgb, dbb):
        if b is not None:
            _guard(fails, f, b)


# =====================================================================================================================
# GroupNorm
# =====================================================================================================================
def run_gn(fails, fam, B, H, W, C, G, relu, resid):
    """gn_fwd then gn_bwd (dgamma / dbeta prefilled: the kernel adds into them)."""
    e = ops.ext()
    x = _act((B, H, W, C))
    gamma, beta, _, _ = _bn_params(C)
    res = _act((B, H, W, C)) if resid else None
    y, yb = lo.guarded((B, H, W, C), BF, DEV)
    mr, mrb = lo.guarded((B, 2, G), torch.float32, DEV)
    e.gn_fwd(x, res, y, gamma, beta, mr, G, EPS, bool(relu))
    torch.cuda.synchronize()
    mean, u_mean, rstd, u_rstd = lo.gn_stats(x, G, mr[:, 0], EPS)
    _judge(fails, "gn_stats " + fam, lo.check_value(fam + " mean", mr[:, 0], mean, u_mean, kappa=lo.KAPPA_FIN))
    _judge(fails, "gn_stats " + fam, lo.check_value(fam + " rstd", mr[:, 1], rstd, u_rstd, kappa=lo.KAPPA_FIN))
    v, unit = lo.affine_statement(x, lo.per_channel(mr[:, 0], C), lo.per_channel(mr[:, 1], C), gamma, beta, res)
    _judge(fails, "gn_fwd " + fam, lo.check_value(fam, y, v, unit, lo.epi_relu(relu)))
    _guard(fails, "gn_fwd " + fam, yb)
    _guard(fails, "gn_fwd " + fam, mrb)
    dy = _act((B, H, W, C))
    dx, dxb = lo.guarded((B, H, W, C), BF, DEV)
    dres, drb = lo.guarded((B, H, W, C), BF, DEV) if resid else (None, None)
    dg, dgb = lo.guarded((C,), torch.float32, DEV)
    db, dbb = lo.guarded((C,), torch.float32, DEV)
    old = torch.randn(2, C, device=DEV)
    dg.copy_(old[0]); db.copy_(old[1])
    e.gn_bwd(dy, y if relu else None, x, gamma, mr, dx, dres, dg, db, G, bool(relu))
    torch.cuda.synchronize()
    dz = torch.where(y.double() > 0, dy.double(), torch.zeros_like(dy, dtype=torch.float64)) if relu else dy.double()
    v, unit, xhat = lo.gn_dx_statement(dz, x, gamma, mr, G)
    _judge(fails, "gn_bwd " + fam, lo.check_value(fam, dx, v, unit, lo.rn_bf16))
    terms = torch.stack([(dz * xhat).reshape(-1, C), dz.reshape(-1, C)])
    _judge(fails, "gn_dparam " + fam, lo.check_sums(fam, torch.stack([dg, db]), terms, old, rounding=3))
    if resid:
        _exact(fails, "gn_dres " + fam, dres, dz.to(BF))
    for b in (dxb, drb, dgb, dbb):
        if b is not None:
            _guard(fails, "gn_bwd " + fam, b)


# =====================================================================================================================
# pooling, ReLU backward, dropout
# =====================================================================================================================
def _pool_input(shape, ties):
    if ties:   # post-ReLU values on a coarse grid: zeros and repeated values in most windows
        return (torch.randint(-3, 4, shape, device=DEV).float() * 0.5).clamp_min(0).to(BF)
    return torch.randn(shape, device=DEV).to(BF)


def run_maxpool(fails, fam, B, H, W, C, p=0.0, zmask=False, ties=True, step=STEP_HI, node=6):
    e = ops.ext()
    x = _pool_input((B, H, W, C), ties)
    Ho, Wo = H // 2, W // 2
    d = lo.Drop(p, SEED, step, node) if p else None
    st = _step(step)
    y, yb = lo.guarded((B, Ho, Wo, C), BF, DEV)
    idx, ib = _guarded_u8((B, Ho, Wo, C))
    dk = (p, SEED, st, node) if p else ()
    e.maxpool2_fwd(x, y, idx, *dk)
    torch.cuda.synchronize()
    wy, wi = lo.maxpool_statement(x, d)
    f = f"maxpool p{p} " + fam
    _exact(fails, f, y, wy)
    _exact(fails, f + " idx", idx, wi)
    _guard(fails, f, yb)
    _guard_u8(fails, f, ib)
    dy = _act((B, Ho, Wo, C))
    dx, dxb = lo.guarded((B, H, W, C), BF, DEV)
    z = wy if zmask else None
    if zmask:
        e.maxpool2_bwd(dy, wi, dx, *(dk or (0.0, 0, None, 0)), relu_out=z)
    else:
        e.maxpool2_bwd(dy, wi, dx, *dk)
    torch.cuda.synchronize()
    _exact(fails, f"maxpool_bwd p{p} z{int(zmask)} " + fam, dx, lo.maxpool_bwd_statement(dy, wi, x.shape, d, z))
    _guard(fails, "maxpool_bwd " + fam, dxb)


def run_avgpool(fails, fam, B, H, W, C):
    e = ops.ext()
    x = _act((B, H, W, C))
    y, yb = lo.guarded((B, 1, 1, C), BF, DEV)
    e.avgpool_fwd(x, y)
    dy = _act((B, 1, 1, C))
    dx, dxb = lo.guarded((B, H, W, C), BF, DEV)
    e.avgpool_bwd(dy, dx)
    torch.cuda.synchronize()
    st, phi = lo.avgpool_statement(x)
    _judge(fails, "avgpool " + fam, lo.check(fam, y.reshape(B, C), st, phi))
    _exact(fails, "avgpool_bwd " + fam, dx, lo.avgpool_bwd_statement(dy.reshape(B, C), x.shape))
    _guard(fails, "avgpool " + fam, yb)
    _guard(fails, "avgpool_bwd " + fam, dxb)


def run_dropout(fails, fam, shape, p, step=STEP_HI, node=9):
    e = ops.ext()
    x = _act(shape)
    d = lo.Drop(p, SEED, step, node)
    y, yb = lo.guarded(shape, BF, DEV)
    m, mb = _guarded_u8(shape)
    e.dropout_fwd(x, y, m, p, SEED, _step(step), node)
    dy = _act(shape)
    dx, dxb = lo.guarded(shape, BF, DEV)
    e.dropout_bwd(dy, m, dx, p)
    torch.cuda.synchronize()
    wy, wm = lo.dropout_statement(x, d)
    f = f"dropout p{p} " + fam
    _exact(fails, f, y, wy)
    _exact(fails, f + " mask", m, wm)
    _exact(fails, f"dropout_bwd p{p} " + fam, dx, lo.dropout_bwd_statement(dy, wm, p))
    for b in (yb, dxb):
        _guard(fails, f, b)
    _guard_u8(fails, f, mb)


def run_relu_bwd(fails, fam, shape, scale):
    dy, db = lo.guarded(shape, BF, DEV)
    dy.copy_(_act(shape))
    y = _pool_input(shape, True)
    want = lo.relu_bwd_statement(dy, y, scale)
    ops.ext().relu_bwd(dy, y, float(scale))
    torch.cuda.synchronize()
    _exact(fails, f"relu_bwd s{scale:.4f} " + fam, dy, want)
    _guard(fails, "relu_bwd " + fam, db)


def run_linear_drop(fails, fam, M, K, N, p, step=STEP_HI, node=10, relu=True, bias=True):
    """Linear layer with dropout fused into the wgmma GEMM epilogue or the split-K finishing pass: rn_bf16(relu(acc + b) * keep * scale),
    the keep-mask of element row * N + col."""
    x, w = _act((M, K)), (torch.randn(N, K, device=DEV) / math.sqrt(K)).to(BF)
    b = torch.randn(N, device=DEV) * 0.1 if bias else None
    y, yb = lo.guarded((M, N), BF, DEV)
    d = lo.Drop(p, SEED, step, node)
    ops.linear_fwd(x, w, b, y, relu, "sm100", drop=(p, SEED, _step(step), node))
    torch.cuda.synchronize()
    keep = lo.dropout_keep((M, N), d, DEV)
    f = f"linear_drop p{p} " + fam
    _judge(fails, f, lo.check(fam, y, lo.gemm_statement(x, w), lo.epi_linear_drop(b, relu, keep, d.scale("f64"))))
    _guard(fails, f, yb)


# =====================================================================================================================
# harvested calls
# =====================================================================================================================
HARVEST_OPS = ("bn_fwd", "bn_bwd", "gn_fwd", "gn_bwd", "maxpool2_fwd", "maxpool2_bwd", "avgpool_fwd", "avgpool_bwd", "dropout_fwd",
               "dropout_bwd", "relu_bwd_", "linear_fwd")


def _harvest():
    """{signature: None} of every layer-kernel call one NativeNet training step of each zoo model makes, dropout on."""
    calls = {}
    real = {n: getattr(ops, n) for n in HARVEST_OPS}

    def rec(name, key):
        def f(*a, **k):
            calls[key(*a, **k)] = None
            return real[name](*a, **k)
        return f

    def bn_fwd_key(x, y, res, gamma, beta, rm, rv, stats, mean_rstd, count, eps, momentum, train, relu, impl, stats_buf=None):
        return ("bn_fwd", x.numel() // x.shape[-1], x.shape[-1], res is not None, bool(relu), bool(train), stats_buf.shape[0] if stats_buf is not None else 1)

    def bn_bwd_key(dy, y, x, gamma, mean_rstd, dsum, dx, dres, dgamma, dbeta, relu, impl, zero_dsum=True, beta=None):
        rec_ = nn.USE_BN_RECOMPUTE and bool(relu) and dres is None and beta is not None
        return ("bn_bwd", x.numel() // x.shape[-1], x.shape[-1], bool(relu), dres is not None, rec_, dsum.shape[0])

    def gn_key(kind):
        def k(*a, **kw):
            x = a[0]
            relu = a[8] if kind == "gn_fwd" else a[10]
            res = a[2] is not None if kind == "gn_fwd" else a[6] is not None
            groups = a[6] if kind == "gn_fwd" else a[9]
            return ("gn",) + tuple(x.shape) + (int(groups), bool(relu), res)
        return k

    def mp_fwd_key(x, y, idx, impl, drop=None, mask=None):
        return ("maxpool",) + tuple(x.shape) + (float(drop[0]) if drop else 0.0, False)

    def mp_bwd_key(dy, idx, dx, impl, drop=None, mask=None, relu_out=None):
        return ("maxpool",) + tuple(dx.shape) + (float(drop[0]) if drop else 0.0, relu_out is not None)

    def avg_key(a, b, impl):
        return ("avgpool",) + tuple((a if a.shape[1] > 1 else b).shape)

    def drop_fwd_key(x, y, mask, p, seed, step, stream, impl):
        return ("dropout", tuple(x.shape), float(p))

    def drop_bwd_key(dy, mask, dx, p, impl):
        return ("dropout", tuple(dx.shape), float(p))

    def relu_key(dy, y, impl, scale=1.0):
        return ("relu_bwd", tuple(dy.shape), float(scale))

    def lin_key(x, w, bias, y, relu, impl, drop=None):
        return ("linear_drop", x.shape[0], w.shape[1], w.shape[0], float(drop[0]) if drop else 0.0, bool(relu), bias is not None)

    keys = dict(bn_fwd=bn_fwd_key, bn_bwd=bn_bwd_key, gn_fwd=gn_key("gn_fwd"), gn_bwd=gn_key("gn_bwd"), maxpool2_fwd=mp_fwd_key,
                maxpool2_bwd=mp_bwd_key, avgpool_fwd=avg_key, avgpool_bwd=avg_key, dropout_fwd=drop_fwd_key, dropout_bwd=drop_bwd_key,
                relu_bwd_=relu_key, linear_fwd=lin_key)
    try:
        for n in HARVEST_OPS:
            setattr(ops, n, rec(n, keys[n]))
        for model in MODELS:
            for B in BATCHES:
                torch.manual_seed(0)
                lay = get_layout(model)
                w = lay.init_(torch.zeros(lay.n_total, device=DEV), 1)
                C, H, W = lay.in_shape
                net = NativeNet(lay, DEV, B, impl="sm100")
                net.step_counter.fill_(STEP_HI)
                g = torch.zeros_like(w)
                net.bind(w, w.to(BF), g)
                logits = net.forward(torch.randn(B, H, W, C, device=DEV).to(BF), True).clone()
                _, dl = ops.softmax_xent(logits, torch.randint(0, 10, (B,), device=DEV))
                net.backward(dl)
                torch.cuda.synchronize()
                del net
    finally:
        for n, f in real.items():
            setattr(ops, n, f)
    return list(calls)


@pytest.fixture(scope="module")
def harvested():
    calls = _harvest()
    print(f"\nharvested {len(calls)} distinct layer-kernel calls from {len(MODELS)} models x batches {BATCHES}")
    return calls


def _replay(fails, key):
    kind = key[0]
    if kind == "bn_fwd":
        _, M, C, res, relu, train, slots = key
        run_bn_fwd(fails, f"{M}x{C}", M, C, relu, res, slots=slots, train=train)
    elif kind == "bn_bwd":
        _, M, C, relu, res, recompute, slots = key
        run_bn_bwd(fails, f"{M}x{C}", M, C, relu, res, recompute, slots)
    elif kind == "gn":
        _, B, H, W, C, G, relu, res = key
        run_gn(fails, f"{B}x{H}x{W}x{C}/{G}", B, H, W, C, G, relu, res)
    elif kind == "maxpool":
        _, B, H, W, C, p, z = key
        run_maxpool(fails, f"{B}x{H}x{W}x{C}", B, H, W, C, p, z)
    elif kind == "avgpool":
        _, B, H, W, C = key
        run_avgpool(fails, f"{B}x{H}x{W}x{C}", B, H, W, C)
    elif kind == "dropout":
        _, shape, p = key
        run_dropout(fails, f"{shape}", shape, p)
    elif kind == "relu_bwd":
        _, shape, scale = key
        run_relu_bwd(fails, f"{shape}", shape, scale)
    elif kind == "linear_drop":
        _, M, K, N, p, relu, bias = key
        if p:
            run_linear_drop(fails, f"{M}x{K}->{N}", M, K, N, p, relu=relu, bias=bias)


@pytest.mark.parametrize("kind", ["bn_fwd", "bn_bwd", "gn", "maxpool", "avgpool", "relu_bwd", "linear_drop"])
def test_harvested_calls_against_fp64(harvested, kind):
    """Each distinct layer-kernel call of the zoo models' training steps, alone on fresh data."""
    torch.manual_seed(1)
    fails = []
    todo = [k for k in harvested if k[0] == kind]
    print(f"{kind}: {len(todo)} harvested calls replayed")
    assert todo
    if kind == "maxpool":
        assert any(k[5] for k in todo), "no max-pool with fused dropout was harvested"
    if kind == "linear_drop":
        assert any(k[4] for k in todo), "no linear layer with fused dropout was harvested"
    _profiled(lambda: [_replay(fails, k) for k in todo], DROP_GEMM if kind == "linear_drop" else KERNELS)
    _assert_clean(fails)


# =====================================================================================================================
# edges
# =====================================================================================================================
def _rows(C):
    rpi = 256 // (C // 8)
    return sorted({m for m in (1, 2, 3, rpi - 1, rpi, rpi + 1, 37 * rpi + 5, 1000 * rpi - 1) if m >= 1})


def test_batchnorm_edges_against_fp64():
    """Channel counts at the ends of chan_ok, 1 / 2 / 3 rows, one row-slot iteration +- 1, ragged reversed-walk tiles; residual and
    mask-recompute variants of the backward pass."""
    torch.manual_seed(2)
    fails = []

    def body():
        for C in (8, 16, 32, 2048):
            for M in _rows(C):
                fam = f"edge M{M} C{C}"
                run_bn_fwd(fails, fam, M, C, True, M % 2 == 1)
                run_bn_bwd(fails, fam, M, C, True, False, True)
                run_bn_bwd(fails, fam, M, C, True, True, False)
                if M < 5000:
                    run_bn_bwd(fails, fam + " norelu", M, C, False, False, False)
    _profiled(body)
    _assert_clean(fails)


def test_batchnorm_slots_and_eval_against_fp64():
    """Multi-slot buffers: [2..16, 2, C] statistics into bn_apply (each slot one row chunk), [4, 2, C] into channel_stats (the four-CTA
    grid), [3, 2, C] backward sums (the three-CTA grid, y-read and recomputed masks); evaluation mode (running statistics)."""
    torch.manual_seed(3)
    fails = []

    def body():
        for slots in (2, 3, 16):
            run_bn_fwd(fails, f"chunks{slots}", 16384 + 77, 64, True, False, chunks=slots)
        for M, C in ((65536, 64), (4100, 512), (3, 8)):
            run_bn_fwd(fails, f"slots4 {M}x{C}", M, C, True, True, slots=4)
            run_bn_bwd(fails, f"slots3 {M}x{C}", M, C, True, False, True, slots=3)
            run_bn_bwd(fails, f"slots3 {M}x{C}", M, C, True, False, False, slots=3)
            run_bn_bwd(fails, f"slots3-res {M}x{C}", M, C, True, True, False, slots=3)
            run_bn_fwd(fails, f"eval {M}x{C}", M, C, True, M > 10, train=False)
            run_bn_fwd(fails, f"eval-norelu {M}x{C}", M, C, False, False, train=False)
    _profiled(body)
    _assert_clean(fails)


def test_groupnorm_edges_against_fp64():
    """Staged and unstaged tiles (forward and backward), group widths of 2 / 16 / 64 channels, one pixel, dgamma / dbeta added into
    nonzero values."""
    torch.manual_seed(4)
    fails = []

    def body():
        for B, H, W, C, G, relu, res in ((2, 64, 64, 64, 32, True, True), (3, 1, 1, 512, 32, False, True), (2, 96, 96, 64, 32, True, False),
                                         (4, 3, 5, 128, 2, True, False), (5, 4, 4, 2048, 32, True, True), (1, 7, 9, 16, 8, False, False),
                                         (1, 128, 128, 64, 32, False, True)):
            run_gn(fails, f"edge {B}x{H}x{W}x{C}/{G}", B, H, W, C, G, relu, res)
    _profiled(body)
    _assert_clean(fails)


def test_pooling_relu_dropout_edges_exact():
    """Odd-sized max-pools over ties (fused ReLU mask and dropout), average pools, ReLU backward scales, stand-alone dropout; dropout
    rates 0.5 / 0.1 / 0.3, step counters 0, 1 and near 2^62, two node ids, and a rate whose threshold ties an element's random bits."""
    torch.manual_seed(5)
    fails = []
    tie_bits = int(lo.dropout_bits(64, lo.Drop(0.5, SEED, 1, 4))[17])
    p_tie = tie_bits / 65536.0

    def body():
        for B, H, W, C in ((2, 7, 9, 16), (3, 30, 30, 64), (4, 13, 13, 128), (1, 3, 2, 8), (2, 24, 24, 64)):
            for p, z in ((0.0, False), (0.0, True), (0.5, True), (0.1, False), (0.3, True)):
                run_maxpool(fails, f"edge {B}x{H}x{W}x{C}", B, H, W, C, p, z)
            run_maxpool(fails, f"edge-randn {B}x{H}x{W}x{C}", B, H, W, C, 0.3, False, ties=False, step=1, node=3)
        for B, H, W, C in ((1, 1, 1, 8), (3, 4, 4, 512), (80, 4, 4, 512), (5, 8, 8, 2048)):
            run_avgpool(fails, f"edge {B}x{H}x{W}x{C}", B, H, W, C)
        for shape in ((8,), (3, 1024), (256, 9216), (7, 72)):
            for scale in (1.0, 2.0, 1 / 0.9, 1 / 0.7):
                run_relu_bwd(fails, f"edge {shape}", shape, scale)
            for p in (0.5, 0.1, 0.3):
                for step, node in ((0, 6), (1, 9), (STEP_HI, 6), ((1 << 62) - 3, 11)):
                    run_dropout(fails, f"edge {shape} step{step} node{node}", shape, p, step, node)
        run_dropout(fails, "tie", (1, 64), p_tie, 1, 4)
        run_maxpool(fails, "tie", 1, 4, 4, 16, p_tie, False, step=1, node=4)
    _profiled(body)
    _assert_clean(fails)


def test_linear_dropout_epilogues_against_fp64():
    """Dropout fused into the wgmma GEMM epilogue and the split-K finishing pass (fc1 of cnn_mnist, K = 9216), rates whose scale is not a
    power of two, several steps."""
    torch.manual_seed(6)
    fails = []

    def body():
        for M, K, N in ((256, 9216, 128), (96, 9216, 128), (256, 1024, 128), (80, 128, 256), (256, 128, 256), (7, 64, 64)):
            for p, step in ((0.5, STEP_HI), (0.1, 1), (0.3, (1 << 62) - 3)):
                run_linear_drop(fails, f"{M}x{K}->{N}", M, K, N, p, step)
    _profiled(body, DROP_GEMM)
    _assert_clean(fails)


# =====================================================================================================================
# BatchNorm's one-pass variance far from zero mean
# =====================================================================================================================
def test_batchnorm_output_at_large_mean_to_std_ratio():
    """BatchNorm statistics use the one-pass E[x^2] - mean^2 in fp32.  For channels with |mean| / std of 0 ... 32 (65,536 rows), the
    output is compared with the fp64 truth of the same bf16 input (exact mean, biased variance): an element is within bf16 rounding if
    it is within one bf16 ulp of the truth (ulp taken at max(|truth|, 2^-6)).  Realistic ratios (<= 4) must stay within it."""
    torch.manual_seed(7)
    e = ops.ext()
    M, C = 65536, 8
    worst = {}
    for ratio in (0, 1, 2, 4, 8, 16, 32):
        x = ((torch.randn(M, C, device=DEV) + ratio) * (torch.rand(C, device=DEV) + 0.5)).to(BF)
        gamma, beta = torch.ones(C, device=DEV), torch.zeros(C, device=DEV)
        y = torch.empty_like(x)
        mr = torch.empty(2, C, device=DEV)
        stats = torch.zeros(1, 2, C, device=DEV)
        e.channel_stats(x, stats)
        e.bn_apply(x, None, y, gamma, beta, mr, False, 1, stats, float(M), EPS, MOM, torch.zeros(C, device=DEV), torch.ones(C, device=DEV))
        xd = x.double()
        mu, var = xd.mean(0), xd.var(0, unbiased=False)
        truth = (xd - mu) * (var + lo.f32(EPS)).rsqrt()
        ulp = torch.exp2(torch.floor(torch.log2(truth.abs().clamp_min(2.0 ** -6))) - 7)
        worst[ratio] = float(((y.double() - truth).abs() / ulp).max())
    RATIO_REPORT.update(worst)
    ok = [r for r, v in worst.items() if v <= 1.0]
    print("\nBatchNorm y vs fp64 truth, largest error in bf16 ulps by |mean|/std:", {r: round(v, 3) for r, v in worst.items()},
          "| within bf16 rounding up to ratio", max(r for r in worst if all(worst[q] <= 1.0 for q in worst if q <= r)) if ok else None)
    assert all(worst[r] <= 1.0 for r in (0, 1, 2, 4)), worst


# =====================================================================================================================
# whole step of the reference CNNs with dropout on
# =====================================================================================================================
class _MaskedF:
    """torch.nn.functional with ``dropout`` replaced by the given keep-masks, in node order."""

    def __init__(self, masks):
        self.masks = list(masks)

    def __getattr__(self, name):
        return getattr(torch.nn.functional, name)

    def dropout(self, t, p, training):
        m = self.masks.pop(0)
        return t * m.to(t.dtype) / (1 - p)


def _reference(lay, w, x, y, masks):
    """Flat gradient of GraphNet in fp64 autograd with the dropout layers replaced by ``masks``."""
    wi, g = w.double(), torch.zeros(lay.n_total, dtype=torch.float64, device=DEV)
    net = graph_mod.GraphNet(lay, wi, g, torch.float64)
    net.train()
    old = graph_mod.F
    graph_mod.F = _MaskedF(masks)
    try:
        logits = net(x.double().permute(0, 3, 1, 2).contiguous())
        torch.nn.functional.cross_entropy(logits, y).backward()
    finally:
        graph_mod.F = old
    return g


def _masks(lay, B, p, step):
    """Keep-mask of every dropout node at ``step``: node i's [B, F] tensor, flat element b * F + j (NHWC flatten order)."""
    out, shape = [], lay.in_shape
    C, H, W = shape
    feat = None
    for i, nd in enumerate(lay.nodes):
        a = nd.attrs
        if nd.op == "conv":
            H, W, C = (H + 2 * a.get("pad", 0) - a["k"]) // a.get("stride", 1) + 1, (W + 2 * a.get("pad", 0) - a["k"]) // a.get("stride", 1) + 1, a["cout"]
        elif nd.op == "maxpool":
            H, W = H // 2, W // 2
        elif nd.op == "flatten":
            feat = H * W * C
        elif nd.op == "linear":
            feat = a["cout"]
        elif nd.op == "dropout":
            out.append(lo.dropout_keep((B, feat), lo.Drop(p, SEED, step, i), DEV))
    return out


def _native_steps(lay, w, x, y, fuse):
    """Two training steps of NativeNet (the second after advance_cursor bumps the step counter): flat gradients and step values."""
    old = native.FUSE_DROPOUT
    native.FUSE_DROPOUT = fuse
    try:
        ops.reset_fallbacks()
        B = x.shape[0]
        net = NativeNet(lay, DEV, B, impl="sm100", seed=SEED)
        net.step_counter.fill_(STEP_HI)
        wi, g = w.clone(), torch.zeros_like(w)
        net.bind(wi, wi.to(BF), g)
        cursor = torch.zeros(1, dtype=torch.int32, device=DEV)
        out = []
        for _ in range(2):
            step = int(net.step_counter.item())
            logits = net.forward(x, True).clone()
            _dropped_outputs_are_zero(net, B, step)
            _, dl = ops.softmax_xent(logits, y)
            net.backward(dl)
            torch.cuda.synchronize()
            out.append((g.clone(), step))
            ops.ext().advance_cursor(cursor, B, net.step_counter)
        assert ops.fallback_calls() == {}, ops.fallback_calls()
        if any(nd.op == "dropout" and nd.attrs["p"] > 0 for nd in lay.nodes):      # p = 0 is never fused
            assert ("dropout" in {op.kind for op in net.plan}) == (not fuse)
        return out
    finally:
        native.FUSE_DROPOUT = old


def _dropped_outputs_are_zero(net, B, step):
    """Every element the statement drops is exactly zero in the dropped tensor the forward pass left (fused: the max-pool / linear
    output; stand-alone: the dropout output), and the statement keeps about 1 - p of them."""
    for op in net.plan:
        d = op.saved.get("drop") if op.saved.get("drop_on") else ((op.attrs["p"], op.node) if op.kind == "dropout" else None)
        if d is None or d[0] == 0:
            continue
        t = net.T(op.y, B).reshape(B, -1)
        keep = lo.dropout_keep(tuple(t.shape), lo.Drop(d[0], SEED, step, d[1]), DEV)
        assert bool((t[~keep] == 0).all()), (op.kind, d, int((t[~keep] != 0).sum()))
        assert abs(float(keep.float().mean()) - (1 - d[0])) < 0.1


def _errs(lay, g, ref):
    out = {}
    for p in lay.params:
        a, b = lay.view(g, p).double(), lay.view(ref, p)
        out[p.name] = (float((a - b).abs().max() / b.abs().max().clamp_min(1e-30)), float((a - b).norm() / b.norm().clamp_min(1e-30)))
    return out


@pytest.mark.parametrize("fuse", [True, False])
@pytest.mark.parametrize("model", ["cnn_mnist", "cnn_cifar"])
def test_reference_cnn_gradients_with_dropout(model, fuse):
    """cnn_mnist / cnn_cifar forward + backward on the sm100 back-end with dropout p = 0.5 against fp64 autograd of GraphNet fed the
    statement's keep-masks, for two consecutive steps (the second with the masks of step + 1).  Every element the statement drops is
    zero in the forward pass's dropped tensors.  Per parameter tensor, the RMS error relative to the reference must stay within 4x that
    of the same comparison with dropout off, + 0.05: ReLU decisions within rounding of zero differ between bf16 and fp64 and move single
    gradient elements by O(1) in both runs (the max-abs error is printed, not judged), while masks keyed by a wrong step, node or
    index change half the kept elements and move the RMS error to O(1)."""
    torch.manual_seed(8)
    B = 8
    lay = get_layout(model)
    w = lay.init_(torch.zeros(lay.n_total, device=DEV), 1)
    w[: lay.n_vote] = w[: lay.n_vote].to(BF).float()
    C, H, W = lay.in_shape
    x = torch.randn(B, H, W, C, device=DEV).to(BF)
    y = torch.randint(0, 10, (B,), device=DEV)
    errs = {}
    for p in (0.0, 0.5):
        for nd in lay.nodes:
            if nd.op == "dropout":
                nd.attrs["p"] = p
        for k, (g, step) in enumerate(_native_steps(lay, w, x, y, fuse)):
            assert step == STEP_HI + k
            ref = _reference(lay, w, x, y, _masks(lay, B, p, step))
            errs[(p, k)] = _errs(lay, g, ref)
    bad = []
    for k in (0, 1):
        for name, (mx, rms) in errs[(0.5, k)].items():
            mx0, rms0 = errs[(0.0, k)][name]
            if not rms <= 4 * rms0 + 0.05:
                bad.append((k, name, round(mx, 5), round(mx0, 5), round(rms, 5), round(rms0, 5)))
    print(model, "fused" if fuse else "stand-alone", "largest (max-rel, rms-rel) with dropout:",
          max(v[0] for v in errs[(0.5, 0)].values()), max(v[1] for v in errs[(0.5, 0)].values()),
          "without:", max(v[0] for v in errs[(0.0, 0)].values()), max(v[1] for v in errs[(0.0, 0)].values()))
    assert not bad, bad


# =====================================================================================================================
# coverage (run the whole file: it judges what the tests above called)
# =====================================================================================================================
REQUIRED = ["channel_reduce_kernel<0, false, 8, 2>", "channel_reduce_kernel<0, false, 4, 4>", "channel_reduce_kernel<1, false, 4, 2>",
            "channel_reduce_kernel<1, true, 4, 2>", "channel_reduce_kernel<1, false, 2, 3>", "channel_reduce_kernel<1, true, 2, 3>",
            "bn_bwd_apply_kernel<true, 4>", "bn_bwd_apply_kernel<false, 4>", "bn_apply_kernel<4>",
            "gn_fwd_kernel<true>", "gn_fwd_kernel<false>", "gn_bwd_kernel<true>", "gn_bwd_kernel<false>",
            "maxpool2_fwd_kernel", "maxpool2_bwd_kernel", "avgpool_fwd_kernel", "avgpool_bwd_kernel", "dropout_fwd_kernel",
            "dropout_bwd_kernel", "relu_bwd_kernel"]


def test_coverage_and_summary():
    print(f"\nlayer oracle summary: family -> (largest kappa needed, largest mismatch fraction, checks); KAPPA_EW={lo.KAPPA_EW} "
          f"KAPPA_FIN={lo.KAPPA_FIN} KAPPA_STATS={lo.KAPPA_STATS} RHO={lo.RHO}")
    groups = defaultdict(lambda: [0.0, 0.0, 0])
    for fam, (k, m, n) in sorted(SUMMARY.items()):
        g = groups[fam.split(" ")[0]]
        g[0], g[1], g[2] = max(g[0], k), max(g[1], m), g[2] + n
    for g, (k, m, n) in sorted(groups.items()):
        print(f"  {g:20s} kappa {k:.4f}  mismatch {m:.5f}  checks {n}")
    worst = sorted(SUMMARY.items(), key=lambda kv: -kv[1][0])[:8]
    print("  worst:", [(f, round(v[0], 4)) for f, v in worst])
    if RATIO_REPORT:
        print("  BatchNorm y error (bf16 ulps) by |mean|/std:", RATIO_REPORT)
    if not SUMMARY:
        pytest.skip("run the whole file: nothing was checked before this test")
    print("  layer kernels met:", sorted({n[n.index("rlr::") + 5:].split("(")[0] for n in KERNELS if "rlr::" in n}))
    missing = [k for k in REQUIRED if not any(k in name for name in KERNELS)]
    assert not missing, missing
    assert any("splitk_finish_kernel" in n for n in DROP_GEMM), sorted(DROP_GEMM)
    assert any("umma_conv_gemm_kernel" in n for n in DROP_GEMM), sorted(DROP_GEMM)
