"""Every conv, GEMM and weight-gradient kernel path against the fp64 statements of tests/gemm_oracle.py, element by element.

* Harvested shapes: one training step of every zoo model at batch 256 and at the ragged last batches of an epoch (96 = 60,000 mod 256
  for FMNIST, 80 = 50,000 mod 256 for CIFAR-10) records each problem the native executor hands to the conv / linear primitives; each
  distinct problem is replayed alone on fresh random operands.
* Edge shapes the dispatch predicates accept but no model uses: odd filter counts, channel padding, 1 / 127 / 128 / 129 output rows,
  halo tiles exactly at the half-area boundary, one-k-block and uneven-split weight gradients.
* Knob matrix: a representative subset under every non-default kernel switch.

Overwritten outputs are prefilled with NaN and followed by a guard band that must come back untouched; elements no tap reaches must
be exact zeros.  The last test asserts that every dispatch path of the primitives (the set of extension entry points one call runs),
every weight-gradient kernel and every instantiation of the implicit-GEMM conv kernel the dispatch can pick on this device were
taken by a call the tests before it judged against fp64 (run the whole file)."""
import contextlib
import math
from collections import defaultdict

import pytest
import torch

import gemm_oracle as go
import rlr_b200  # noqa: F401
from rlr_b200 import ops
from rlr_b200.models import get_layout
from rlr_b200.models.native import NativeNet
from rlr_b200.ops import nn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16

MODELS = ["resnet18", "resnet34", "vgg11", "vgg16", "cnn_cifar", "cnn_mnist"]
BATCHES = [256, 96, 80]

# per family: (largest kappa needed, largest mismatch fraction, checks)
SUMMARY = defaultdict(lambda: [0.0, 0.0, 0])
PATHS = set()           # (primitive, frozenset of the extension entry points one oracle-judged call of it ran)
WGRAD_LAUNCHES = [0, 0, 0]   # launches of (umma_wgrad_kernel, umma_wgrad_halo_kernel, umma_wgrad_rows_kernel) by judged calls
INSTS = set()           # umma_conv_gemm_kernel instantiations met (profiled tests, every call judged)
_CUR = None             # entry points of the judged call in progress
# every dispatch branch of ops/nn.py's conv / linear primitives, as the entry points it runs (conv_bf16 split by how it reads the
# filter: [mn-major] = the forward filter with a tap list, [k-major] = a plain or transposed copy)
PATHS_REQUIRED = [
    ("fwd", {"conv_bf16[k-major]"}), ("fwd", {"pad_rows", "conv_bf16[k-major]"}), ("fwd", {"space_to_depth", "conv_bf16[k-major]"}),
    ("fwd", {"conv_bf16_strided"}), ("fwd", {"im2col_small", "stem_gemm_bf16"}), ("fwd", {"conv3x3_halo_bf16"}),
    ("fwd", {"conv3x3_halo3_bf16"}),
    ("dgrad", {"conv_bf16[mn-major]"}),                                               # stride 1, forward filter read MN-major
    ("dgrad", {"filter_transpose", "conv_bf16[k-major]"}),                            # stride 1, Cin % 64 != 0: transposed filter
    ("dgrad", {"filter_transpose", "conv3x3_halo_bf16"}), ("dgrad", {"filter_transpose", "conv3x3_halo3_bf16"}),
    ("dgrad", {"conv_bf16_strided"}),                                                 # stride 2, planes stored into dX
    ("dgrad", {"conv_bf16[mn-major]", "depth_to_space"}),                             # stride 2, parity buffer
    ("dgrad", {"filter_gather_transpose", "conv_bf16[k-major]", "depth_to_space"}),   # stride 2, Cin % 64 != 0
    ("wgrad", {"conv_wgrad_bf16"}), ("wgrad", {"conv_wgrad_halo_bf16"}), ("wgrad", {"conv_wgrad_bf16_strided"}),
    ("wgrad", {"linear_wgrad_bf16", "unpad_add"}), ("wgrad", {"bias_grad"}),
    ("linear", {"gemm_bf16"}), ("linear", {"gemm_splitk_bf16"}), ("linear", {"linear_small_fwd2"}), ("linear", {"linear_small_fwd"}),
    ("linear_bwd", {"linear_wgrad_bf16", "bias_grad", "filter_transpose", "gemm_bf16"}), ("linear_bwd", {"linear_small_bwd2"}),
    ("linear_bwd", {"linear_small_bwd"}),
]


class _RecordingExt:
    """Wraps the extension object of ``ops``; inside a judged call it records the entry points that call runs."""

    def __init__(self, inner):
        self._inner = inner

    def __getattr__(self, name):
        attr = getattr(self._inner, name)
        if _CUR is None or not callable(attr):
            return attr

        def call(*a, **k):
            _CUR.add(name + ("[mn-major]" if a[12] else "[k-major]") if name == "conv_bf16" else name)   # a[12]: filter tap list
            return attr(*a, **k)
        return call


@contextlib.contextmanager
def _judged(prim):
    """Records the dispatch path (and weight-gradient kernel launches) of one primitive call whose result is then judged."""
    global _CUR
    before = ops.ext().wgrad_launch_counts()
    _CUR = set()
    try:
        yield
    finally:
        PATHS.add((prim, frozenset(_CUR)))
        _CUR = None
        for i, (a, b) in enumerate(zip(ops.ext().wgrad_launch_counts(), before)):
            WGRAD_LAUNCHES[i] += a - b


@pytest.fixture(scope="module", autouse=True)
def _record_entries():
    ops.ext()
    inner = ops._ext
    ops._ext = _RecordingExt(inner)
    try:
        yield
    finally:
        ops._ext = inner


@pytest.fixture(autouse=True)
def _fresh_scratch():
    """Scratch copies keyed by data pointers of this test's tensors are dropped afterwards (they would only pile up)."""
    keys, done = set(nn._scratch), set(nn._s2d_done)
    yield
    torch.cuda.synchronize()
    for k in set(nn._scratch) - keys:
        del nn._scratch[k]
    for k in set(nn._s2d_done) - done:
        del nn._s2d_done[k]


def _judge(fails, family, r):
    s = SUMMARY[family]
    s[0], s[1], s[2] = max(s[0], r.kappa), max(s[1], r.mismatch), s[2] + 1
    if not r.ok:
        fails.append((family, r))


def _guard(fails, family, buf):
    if not go.guard_intact(buf):
        fails.append((family, "guard band written"))


def _rand(shape, scale=1.0):
    return (torch.randn(shape, device=DEV) * scale).to(BF)


# =====================================================================================================================
# replay of one problem per primitive
# =====================================================================================================================
def run_fwd(fails, fam, B, H, W, Cin, Cout, k, s, p, bias=True, relu=True, stats=False):
    x, w = _rand((B, H, W, Cin)), _rand((Cout, k, k, Cin), 1 / math.sqrt(k * k * Cin))
    b = torch.randn(Cout, device=DEV) * 0.1 if bias else None
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    y, buf = go.guarded((B, Ho, Wo, Cout), BF, DEV)
    st_buf = torch.zeros(ops.STAT_SLOTS, 2, Cout, device=DEV) if stats else None
    with _judged("fwd"):
        ops.conv2d_fwd_sm100(x, w, b, y, s, p, relu, st_buf, tag=("oracle-fwd", B, H, W, Cin, Cout, k, s, p))
    _judge(fails, "fwd " + fam, go.check(fam, y, go.conv_statement(x, w, s, p), go.epi_store(b, relu)))
    _guard(fails, "fwd " + fam, buf)
    if stats:
        _judge(fails, "stats " + fam, go.check_stats(fam, st_buf, y))


def run_dgrad(fails, fam, B, H, W, Cin, Cout, k, s, p, modes=(False, True)):
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy, w = _rand((B, Ho, Wo, Cout)), _rand((Cout, k, k, Cin), 1 / math.sqrt(k * k * Cout))
    st = go.dgrad_statement(dy, w, (B, H, W, Cin), s, p)
    for acc in modes:
        dx, buf = go.guarded((B, H, W, Cin), BF, DEV)
        old = _rand((B, H, W, Cin)) if acc else None
        if acc:
            dx.copy_(old)
        with _judged("dgrad"):
            ops.conv2d_dgrad_sm100(dy, w, dx, s, p, acc)
        f = ("dgrad+acc " if acc else "dgrad ") + fam
        _judge(fails, f, go.check(fam, dx, st, go.epi_acc_twice(old) if acc else go.epi_store()))
        _guard(fails, f, buf)


def run_wgrad(fails, fam, B, H, W, Cin, Cout, k, s, p, bias=True):
    x, w = _rand((B, H, W, Cin)), _rand((Cout, k, k, Cin), 1 / math.sqrt(k * k * Cin))
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy = _rand((B, Ho, Wo, Cout))
    tag = ("oracle-wgrad", B, H, W, Cin, Cout, k, s, p)
    ops.conv2d_fwd_sm100(x, w, None, torch.empty(B, Ho, Wo, Cout, device=DEV, dtype=BF), s, p, False, None, tag=tag)  # fills the copies of x
    st, stb = go.wgrad_statement(x, dy, k, s, p), go.colsum_statement(dy)
    for zero in (True, False):
        gw, bw = go.guarded((Cout, k, k, Cin), torch.float32, DEV)
        gb, bb = go.guarded((Cout,), torch.float32, DEV)
        if not zero:
            gw.copy_(torch.randn_like(gw)); gb.copy_(torch.randn_like(gb))
        ow, ob = gw.clone(), gb.clone()
        with _judged("wgrad"):
            ops.conv2d_wgrad_sm100(x, dy, gw, gb if bias else None, s, p, tag=tag, zero=zero)
        f = ("wgrad " if zero else "wgrad+add ") + fam
        _judge(fails, f, go.check(fam, gw, st if zero else go.plus_old(st, ow), go.epi_f32))
        _guard(fails, f, bw)
        if bias:
            _judge(fails, "bias_grad " + fam, go.check(fam, gb, stb if zero else go.plus_old(stb, ob), go.epi_f32))
            _guard(fails, "bias_grad " + fam, bb)


def run_linear(fails, fam, M, K, N, bias=True, relu=True):
    run_linear_fwd(fails, fam, M, K, N, bias, relu)
    run_linear_bwd(fails, fam, M, K, N, bias)


def run_linear_fwd(fails, fam, M, K, N, bias=True, relu=True):
    x, w = _rand((M, K)), _rand((N, K), 1 / math.sqrt(K))
    b = torch.randn(N, device=DEV) * 0.1 if bias else None
    y, buf = go.guarded((M, N), BF, DEV)
    with _judged("linear"):
        ops.linear_fwd(x, w, b, y, relu, "sm100")
    _judge(fails, "linear " + fam, go.check(fam, y, go.gemm_statement(x, w), go.epi_store(b, relu)))
    _guard(fails, "linear " + fam, buf)


def run_linear_bwd(fails, fam, M, K, N, bias=True, need_dx=True):
    x, w, dy = _rand((M, K)), _rand((N, K), 1 / math.sqrt(K)), _rand((M, N))
    st_w, st_b, st_x = go.gemm_statement(dy.t(), x.t()), go.colsum_statement(dy), go.gemm_statement(dy, w.t())
    head = N <= 32
    # the first head kernels (USE_HEAD_V2 off) store dW / db rather than add into them: their accumulating call zeroes first
    adds = not (head and not nn.USE_HEAD_V2)
    for acc in ((False, True) if need_dx else (False,)):
        dx, bx = go.guarded((M, K), BF, DEV)
        dw, bw = go.guarded((N, K), torch.float32, DEV)
        db, bb = go.guarded((N,), torch.float32, DEV)
        old = _rand((M, K)) if acc else None
        add = acc and adds
        if acc:      # the accumulating call also adds dW / db into existing gradients (zero=False)
            dx.copy_(old)
        if add:
            dw.copy_(torch.randn_like(dw)); db.copy_(torch.randn_like(db))
        ow, ob = dw.clone(), db.clone()
        with _judged("linear_bwd"):
            ops.linear_bwd(x, dy, w, dx if need_dx else None, dw, db if bias else None, acc, "sm100", zero=not add)
        sfx = "+acc " if acc else " "
        epi = (go.epi_acc_once(old) if head else go.epi_acc_twice(old)) if acc else go.epi_store()
        if need_dx:
            _judge(fails, "linear dgrad" + sfx + fam, go.check(fam, dx, st_x, epi))
        _judge(fails, "linear wgrad" + sfx + fam, go.check(fam, dw, go.plus_old(st_w, ow) if add else st_w, go.epi_f32))
        for f, bf in (("linear dgrad", bx), ("linear wgrad", bw), ("linear bgrad", bb)):
            _guard(fails, f + sfx + fam, bf)
        if bias:
            _judge(fails, "linear bgrad" + sfx + fam, go.check(fam, db, go.plus_old(st_b, ob) if add else st_b, go.epi_f32))


def _assert_clean(fails):
    torch.cuda.synchronize()
    assert not fails, fails[:10]


# =====================================================================================================================
# harvested shapes
# =====================================================================================================================
def _harvest():
    """{signature: None} of every conv / linear problem one NativeNet training step of each zoo model hands to the primitives."""
    probs = {}
    real = {n: getattr(ops, n) for n in ("conv2d_fwd_sm100", "conv2d_dgrad_sm100", "conv2d_wgrad_sm100", "linear_fwd", "linear_bwd")}

    def fwd(x, w, bias, y, stride, pad, relu, stats, **kw):
        Cout, k = w.shape[0], w.shape[1]
        B, Ho, Wo = y.shape[:3]
        xs = tuple(x.shape) if x.dim() == 4 else (B, (Ho - 1) * stride + k - 2 * pad, (Wo - 1) * stride + k - 2 * pad, w.shape[3])
        probs[("fwd",) + xs + (Cout, k, stride, pad, bias is not None, bool(relu), stats is not None)] = None
        return real["conv2d_fwd_sm100"](x, w, bias, y, stride, pad, relu, stats, **kw)

    def dgrad(dy, w, dx, stride, pad, accumulate):
        probs[("dgrad",) + tuple(dx.shape) + (w.shape[0], w.shape[1], stride, pad)] = None
        return real["conv2d_dgrad_sm100"](dy, w, dx, stride, pad, accumulate)

    def wgrad(x, dy, gw, gb, stride, pad, **kw):
        Cout, k, _, Cin = gw.shape
        B, Ho, Wo = dy.shape[:3]
        xs = tuple(x.shape) if x.dim() == 4 else (B, (Ho - 1) * stride + k - 2 * pad, (Wo - 1) * stride + k - 2 * pad, Cin)
        probs[("wgrad",) + xs + (Cout, k, stride, pad, gb is not None)] = None
        return real["conv2d_wgrad_sm100"](x, dy, gw, gb, stride, pad, **kw)

    def lfwd(x, w, bias, y, relu, impl, drop=None):
        probs[("linear", x.shape[0], w.shape[1], w.shape[0], bias is not None, bool(relu))] = None
        return real["linear_fwd"](x, w, bias, y, relu, impl, drop)

    def lbwd(x, dy, w, dx, dw, db, acc_dx, impl, zero=True):
        probs[("linear_bwd", x.shape[0], w.shape[1], w.shape[0], db is not None, dx is not None)] = None
        return real["linear_bwd"](x, dy, w, dx, dw, db, acc_dx, impl, zero)

    patched = dict(conv2d_fwd_sm100=fwd, conv2d_dgrad_sm100=dgrad, conv2d_wgrad_sm100=wgrad, linear_fwd=lfwd, linear_bwd=lbwd)
    try:
        for n, f in patched.items():
            setattr(ops, n, f)
        for model in MODELS:
            for B in BATCHES:
                torch.manual_seed(0)
                lay = get_layout(model)
                for nd in lay.nodes:
                    if nd.op == "dropout":
                        nd.attrs["p"] = 0.0
                w = lay.init_(torch.zeros(lay.n_total, device=DEV), 1)
                C, H, W = lay.in_shape
                net = NativeNet(lay, DEV, B, impl="sm100")
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
    return list(probs)


@pytest.fixture(scope="module")
def harvested():
    probs = _harvest()
    print(f"\nharvested {len(probs)} distinct problems from {len(MODELS)} models x batches {BATCHES}")
    return probs


@pytest.mark.parametrize("kind", ["fwd", "dgrad", "wgrad", "linear", "linear_bwd"])
def test_harvested_shapes_against_fp64(harvested, kind):
    """Each distinct problem of the zoo models' training steps, alone on fresh operands: forward with its epilogue (and its BatchNorm
    statistics where the step asked for them), the data gradient overwriting and accumulating, the weight and bias gradient zeroing and
    adding, the linear layers' forward and backward."""
    torch.manual_seed(1)
    fails, n = [], 0
    for key in harvested:
        if key[0] != kind:
            continue
        n += 1
        if kind == "fwd":
            _, B, H, W, Cin, Cout, k, s, p, bias, relu, stats = key
            run_fwd(fails, f"{B}x{H}x{W}x{Cin}->{Cout} k{k}s{s}p{p}", B, H, W, Cin, Cout, k, s, p, bias, relu, stats)
        elif kind == "dgrad":
            _, B, H, W, Cin, Cout, k, s, p = key
            run_dgrad(fails, f"{B}x{H}x{W}x{Cin}<-{Cout} k{k}s{s}p{p}", B, H, W, Cin, Cout, k, s, p)
        elif kind == "wgrad":
            _, B, H, W, Cin, Cout, k, s, p, bias = key
            run_wgrad(fails, f"{B}x{H}x{W}x{Cin}->{Cout} k{k}s{s}p{p}", B, H, W, Cin, Cout, k, s, p, bias)
        elif kind == "linear":
            _, M, K, N, bias, relu = key
            run_linear_fwd(fails, f"{M}x{K}->{N}", M, K, N, bias, relu)
        else:
            _, M, K, N, bias, need_dx = key
            run_linear_bwd(fails, f"{M}x{K}->{N}", M, K, N, bias, need_dx)
    print(f"{kind}: {n} harvested problems replayed")
    assert n > 0
    _assert_clean(fails)


# =====================================================================================================================
# edge shapes
# =====================================================================================================================
def _profiled(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if "umma_conv_gemm_kernel<" in e.key:
            INSTS.add(e.key[e.key.index("umma_conv_gemm_kernel<"):].split(">")[0] + ">")


def test_edge_shapes_against_fp64():
    torch.manual_seed(2)
    fails = []

    def body():
        for cout in (8, 24, 72, 200):                                  # filter counts off the 64 / 128 tiles
            run_fwd(fails, f"cout{cout}-halo", 16, 8, 8, 64, cout, 3, 1, 1)
            run_fwd(fails, f"cout{cout}", 16, 8, 8, 128, cout, 3, 1, 1, stats=True)
        for cin, s in ((1, 2), (3, 2), (8, 1), (32, 1), (48, 1)):      # channel padding (pad_rows), stride 2 keeps 1 / 3 off the stem
            run_fwd(fails, f"cin{cin}s{s}", 8, 16, 16, cin, 64, 3, s, 1, stats=s == 1)
            run_wgrad(fails, f"cin{cin}s{s}", 8, 16, 16, cin, 64, 3, s, 1)
        run_fwd(fails, "cin96-1x1", 8, 16, 16, 96, 64, 1, 1, 0)        # channel padding on the generic implicit GEMM
        run_fwd(fails, "cin32-4x4", 16, 4, 4, 32, 64, 3, 1, 1)
        for cin in (8, 32, 48):                                        # data gradients into Cin % 64 != 0: transposed filter copies
            for k, s, p in ((3, 1, 1), (3, 2, 1), (1, 2, 0)):
                run_dgrad(fails, f"cin{cin}k{k}s{s}", 16, 16, 16, cin, 128, k, s, p)
        for B in (1, 127, 128, 129):                                   # B * Ho * Wo output rows around one 128-row tile
            run_fwd(fails, f"rows{B}", B, 1, 1, 64, 64, 1, 1, 0, stats=True)
            run_fwd(fails, f"rows{B}-3x3", B, 1, 1, 128, 128, 3, 1, 1)
            run_dgrad(fails, f"rows{B}", B, 1, 1, 64, 64, 1, 1, 0)
            run_linear(fails, f"rows{B}", B, 128, 64)
        for H, W in ((8, 8), (16, 4), (8, 7), (9, 8), (15, 15)):      # halo tiles at / below half the 16 x 8 tile area
            run_fwd(fails, f"halo{H}x{W}", 4, H, W, 64, 64, 3, 1, 1)
            run_dgrad(fails, f"halo{H}x{W}", 4, H, W, 64, 64, 3, 1, 1)
        for cout in (8, 64, 128, 256):                                 # weight-gradient filter tiles
            run_wgrad(fails, f"cout{cout}", 8, 16, 16, 64, cout, 3, 1, 1)
        for B, H in ((1, 8), (3, 8), (5, 8), (7, 32), (1, 2)):          # one k-block, uneven last split
            run_wgrad(fails, f"B{B}H{H}", B, H, H, 64, 128, 3, 1, 1)
            run_wgrad(fails, f"B{B}H{H}-c128", B, H, H, 128, 128, 3, 1, 1)
        for M, K, N in ((256, 9216, 128), (100, 1024, 128), (256, 512, 10), (7, 64, 32), (256, 128, 256), (33, 640, 24)):
            run_linear(fails, f"{M}x{K}->{N}", M, K, N)

    _profiled(body)
    _assert_clean(fails)


def test_gemm_rejects_a_strided_output():
    """The GEMM writes rows of exactly N elements (ldc = N): an output view with a wider row pitch is refused, not written wrongly."""
    A, Bm = _rand((128, 64)), _rand((64, 64))
    wide = torch.zeros(128, 72, device=DEV, dtype=BF)
    with pytest.raises(RuntimeError):
        ops.ext().gemm_bf16(A, Bm, wide[:, :64], None, False, False, None)
    torch.cuda.synchronize()
    assert float(wide.abs().max()) == 0


# =====================================================================================================================
# knob matrix
# =====================================================================================================================
def _subset(fails, tag):
    run_fwd(fails, tag + " l1", 80, 32, 32, 64, 64, 3, 1, 1, stats=True)
    run_fwd(fails, tag + " l1-plain", 80, 32, 32, 64, 64, 3, 1, 1)
    run_fwd(fails, tag + " l3", 96, 8, 8, 256, 256, 3, 1, 1, stats=True)
    run_fwd(fails, tag + " l3-256", 256, 8, 8, 256, 256, 3, 1, 1, stats=True)
    run_fwd(fails, tag + " l4", 256, 4, 4, 512, 512, 3, 1, 1)
    run_fwd(fails, tag + " l4-stats", 256, 4, 4, 512, 512, 3, 1, 1, stats=True)
    run_fwd(fails, tag + " s2", 80, 32, 32, 64, 128, 3, 2, 1)
    run_fwd(fails, tag + " s2-1x1", 80, 16, 16, 128, 256, 1, 2, 0, bias=False, relu=False)
    run_fwd(fails, tag + " stem", 80, 32, 32, 3, 64, 3, 1, 1, stats=True)
    run_fwd(fails, tag + " valid", 96, 26, 26, 32, 64, 3, 1, 0)
    run_dgrad(fails, tag + " l1", 80, 32, 32, 64, 64, 3, 1, 1)
    run_dgrad(fails, tag + " l2", 96, 16, 16, 128, 128, 3, 1, 1)
    run_dgrad(fails, tag + " l4", 256, 4, 4, 512, 512, 3, 1, 1)
    run_dgrad(fails, tag + " s2", 80, 32, 32, 64, 128, 3, 2, 1)
    run_dgrad(fails, tag + " s2-1x1", 80, 16, 16, 128, 256, 1, 2, 0)
    run_dgrad(fails, tag + " cin32", 96, 26, 26, 32, 64, 3, 1, 0)
    run_dgrad(fails, tag + " cin32-s1", 16, 16, 16, 32, 128, 3, 1, 1)
    run_dgrad(fails, tag + " cin32-s2", 16, 16, 16, 32, 128, 3, 2, 1)
    run_dgrad(fails, tag + " cin32-s2-1x1", 16, 16, 16, 32, 128, 1, 2, 0)
    run_dgrad(fails, tag + " full", 96, 13, 13, 64, 64, 3, 1, 0)
    run_wgrad(fails, tag + " l1", 80, 32, 32, 64, 64, 3, 1, 1)
    run_wgrad(fails, tag + " l2", 96, 16, 16, 128, 128, 3, 1, 1)
    run_wgrad(fails, tag + " s2", 80, 32, 32, 64, 128, 3, 2, 1)
    run_wgrad(fails, tag + " stem", 80, 32, 32, 3, 64, 3, 1, 1)
    run_linear(fails, tag + " fc1", 256, 9216, 128)
    run_linear(fails, tag + " head", 96, 512, 10)


def _ext_knob(setter, value, default):
    def apply(on):
        getattr(ops.ext(), setter)(value if on else default)
    return apply


def _py_knob(name, value):
    old = getattr(nn, name)

    def apply(on):
        setattr(nn, name, value if on else old)
    return apply


KNOBS = {
    "persistent_conv": lambda: _ext_knob("set_persistent_conv", True, False),
    "conv_occ3=0": lambda: _ext_knob("set_conv_occ3", 0, 1),      # levels above 1 are level 1, the default
    "one_wave=off": lambda: _ext_knob("set_conv_one_wave", False, True),
    "tma_store=off": lambda: _ext_knob("set_conv_tma_store", False, True),
    "split_producer=off": lambda: _ext_knob("set_conv_split_producer", False, True),
    "wgrad_rows=off": lambda: _ext_knob("set_wgrad_rows", False, True),
    "strided_tma=off": lambda: _py_knob("USE_STRIDED_TMA", False),
    "halo3=on": lambda: _py_knob("USE_HALO3", True),
    "splitk=off": lambda: _py_knob("USE_SPLITK", False),
    "head_v2=off": lambda: _py_knob("USE_HEAD_V2", False),
    "im2col_stem=off": lambda: _py_knob("USE_IM2COL_STEM", False),
}


@pytest.mark.parametrize("knob", list(KNOBS) + ["default"])
def test_knob_matrix_against_fp64(knob):
    torch.manual_seed(3)
    fails = []
    apply = KNOBS[knob]() if knob != "default" else (lambda on: None)
    try:
        apply(True)
        _profiled(lambda: _subset(fails, knob))
    finally:
        apply(False)
    _assert_clean(fails)


# =====================================================================================================================
# layout kernels, bit-exact
# =====================================================================================================================
def test_layout_kernels_bit_exact():
    torch.manual_seed(4)
    e = ops.ext()
    x = _rand((300, 48))
    xp, buf = go.guarded((300, 64), BF, DEV)
    e.pad_rows(x, xp)
    assert torch.equal(xp[:, :48], x) and float(xp[:, 48:].float().abs().max()) == 0 and go.guard_intact(buf)
    dW = torch.randn(24, 64, device=DEV)
    gw = torch.randn(24, 27, device=DEV)
    want = gw + dW[:, :27]
    e.unpad_add(dW, gw)
    assert torch.equal(gw, want)
    s = _rand((3, 8, 6, 64))
    s4, buf = go.guarded((12, 4, 3, 64), BF, DEV)
    e.space_to_depth(s, s4)
    assert go.guard_intact(buf)
    for ph in range(2):
        for pw in range(2):
            assert torch.equal(s4[(ph * 2 + pw) * 3:(ph * 2 + pw + 1) * 3], s[:, ph::2, pw::2])
    for mask in (0b1111, 0b0001, 0b1010):
        for acc in (False, True):
            old = _rand((3, 8, 6, 64))
            y, buf = go.guarded((3, 8, 6, 64), BF, DEV)
            if acc:
                y.copy_(old)
            e.depth_to_space(s4, y, acc, mask)
            want = torch.zeros(3, 8, 6, 64, device=DEV)
            for ph in range(2):
                for pw in range(2):
                    if mask >> (ph * 2 + pw) & 1:
                        want[:, ph::2, pw::2] = s4[(ph * 2 + pw) * 3:(ph * 2 + pw + 1) * 3].float()
            want = go.rn_bf16(want + old.float()) if acc else want
            assert torch.equal(y.float(), want) and go.guard_intact(buf), (mask, acc)
    w = _rand((72, 3, 3, 40))
    wt, buf = go.guarded((40, 9 * 72), BF, DEV)
    e.filter_transpose(w, wt, 72, 9, 40)
    assert torch.equal(wt.view(40, 3, 3, 72), w.flip(1, 2).permute(3, 1, 2, 0)) and go.guard_intact(buf)
    taps = [1, 4, 7]
    wt, buf = go.guarded((40, 3 * 72), BF, DEV)
    e.filter_gather_transpose(w, wt, 72, 9, 40, taps)
    assert torch.equal(wt.view(40, 3, 72), w.reshape(72, 9, 40)[:, taps].permute(2, 1, 0)) and go.guard_intact(buf)
    for C, k, pad in ((3, 3, 1), (1, 3, 0), (7, 3, 1), (64, 1, 0)):
        xi = _rand((5, 9, 11, C))
        Ho, Wo = 9 + 2 * pad - k + 1, 11 + 2 * pad - k + 1
        A, buf = go.guarded((5 * Ho * Wo, 64), BF, DEV)
        e.im2col_small(xi, A, k, pad)
        cols = torch.nn.functional.unfold(xi.float().permute(0, 3, 1, 2), k, padding=pad)            # [B, C*k*k, L], C-major
        cols = cols.view(5, C, k * k, Ho * Wo).permute(0, 3, 2, 1).reshape(5 * Ho * Wo, k * k * C)    # tap-major, channel-minor
        want = torch.zeros(5 * Ho * Wo, 64, device=DEV)
        want[:, :k * k * C] = cols
        assert torch.equal(A.float(), want) and go.guard_intact(buf), (C, k, pad)


# =====================================================================================================================
# coverage (run the whole file: it judges what the tests above called)
# =====================================================================================================================
def test_coverage_and_summary():
    print("\nfp64 oracle summary: family -> (largest kappa needed, largest mismatch fraction, checks); "
          f"KAPPA={go.KAPPA} KAPPA_STATS={go.KAPPA_STATS} RHO={go.RHO}")
    groups = defaultdict(lambda: [0.0, 0.0, 0])
    for fam, (k, m, n) in sorted(SUMMARY.items()):
        g = groups[fam.split(" ")[0]]
        g[0], g[1], g[2] = max(g[0], k), max(g[1], m), g[2] + n
    for g, (k, m, n) in sorted(groups.items()):
        print(f"  {g:16s} kappa {k:.4f}  mismatch {m:.5f}  checks {n}")
    worst = sorted(SUMMARY.items(), key=lambda kv: -kv[1][0])[:8]
    print("  worst shapes:", [(f, round(v[0], 4)) for f, v in worst])
    for prim, path in sorted(PATHS, key=lambda t: (t[0], sorted(t[1]))):
        print(f"  path {prim:10s} {sorted(path - {'memset_zero'})}")
    print("  conv GEMM instantiations met:", sorted(INSTS))
    print("  wgrad launches by judged calls (generic, halo, rows):", WGRAD_LAUNCHES)
    if not SUMMARY:
        pytest.skip("run the whole file: nothing was checked before this test")
    missing = [(prim, sorted(need)) for prim, need in PATHS_REQUIRED if not any(p == prim and need <= path for p, path in PATHS)]
    assert not missing, missing
    assert all(c > 0 for c in WGRAD_LAUNCHES), WGRAD_LAUNCHES
    want = {f"umma_conv_gemm_kernel<{bn}, {st}, {mn}, {occ}>" for bn in (64, 128) for st, mn in (("false", "false"), ("false", "true"))
            for occ in (2, 3 if bn == 64 else 1)} | {f"umma_conv_gemm_kernel<{bn}, true, false, 2>" for bn in (64, 128)}
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if not (128 <= sms and 9 * sms <= 10 * 128):    # the one-wave configuration exists only where 128 CTAs fill one wave
        want = {w for w in want if not w.endswith(", 1>")}
    assert not want - INSTS, (sorted(want - INSTS), sorted(INSTS))
