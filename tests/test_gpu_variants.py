"""GPU tests of the kernel VARIANTS behind the run-time knobs of ops/nn.py / ops.ext(): strided-TMA stride-2 convs, im2col stem, BN mask
recompute, head kernels v2, split-K GEMM (all default on), and the ones that are not the default (three-tap N = 192 halo conv, PDL
launches, 3-CTA occupancy levels, agents in flight)."""
import os

import pytest
import torch

import rlr_b200  # noqa: F401
from rlr_b200 import ops
from rlr_b200.ops import nn

pytestmark = [pytest.mark.gpu]
DEV = "cuda:0"
BF = torch.bfloat16

S2_CASES = [  # B, H, W, Cin, Cout, k, pad
    (32, 32, 32, 64, 128, 3, 1), (32, 32, 32, 64, 128, 1, 0), (40, 16, 16, 128, 256, 3, 1), (40, 16, 16, 128, 256, 1, 0),
    (24, 8, 8, 256, 512, 3, 1), (24, 8, 8, 256, 512, 1, 0), (256, 32, 32, 64, 128, 3, 1),
]


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,p", S2_CASES)
def test_strided_tma_stride2_convs_match_parity_copy_path(B, H, W, Cin, Cout, k, p):
    """RLR_STRIDED_TMA: forward / weight gradient through a TMA box with element strides 2 and data-gradient parity planes stored
    straight into dX must be bit-identical to the space_to_depth / depth_to_space path (same MMAs, same order)."""
    torch.manual_seed(B + H + Cin + k)
    x = torch.randn(B, H, W, Cin, device=DEV).to(BF)
    w = (torch.randn(Cout, k, k, Cin, device=DEV) / (k * k * Cin) ** 0.5).to(BF)
    bias = torch.randn(Cout, device=DEV) * 0.1
    Ho, Wo = (H + 2 * p - k) // 2 + 1, (W + 2 * p - k) // 2 + 1
    dy = torch.randn(B, Ho, Wo, Cout, device=DEV).to(BF)
    base = torch.randn(B, H, W, Cin, device=DEV).to(BF)
    outs = {}
    old = nn.USE_STRIDED_TMA
    try:
        for mode in (False, True):
            nn.USE_STRIDED_TMA = mode
            tag = ("strided-test", mode, B, H, Cin, k)
            y = torch.full((B, Ho, Wo, Cout), 7.0, device=DEV, dtype=BF)
            ops.conv2d_fwd_sm100(x, w, bias, y, 2, p, True, None, tag=tag)
            dx0 = torch.full_like(base, 3.0)
            dx1 = base.clone()
            ops.conv2d_dgrad_sm100(dy, w, dx0, 2, p, False)
            ops.conv2d_dgrad_sm100(dy, w, dx1, 2, p, True)
            gw = torch.zeros(Cout, k, k, Cin, device=DEV)
            ops.conv2d_wgrad_sm100(x, dy, gw, None, 2, p, tag=tag)
            torch.cuda.synchronize()
            outs[mode] = (y, dx0, dx1, gw)
    finally:
        nn.USE_STRIDED_TMA = old
    ref = torch.relu(torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), bias, 2, p)).permute(0, 2, 3, 1)
    assert float((outs[True][0].float() - ref).abs().max() / ref.abs().max()) < 1e-2
    for name, a, b in zip(("fwd", "dgrad", "dgrad+acc"), outs[False][:3], outs[True][:3]):
        assert torch.equal(a, b), name
    # weight gradient: the two paths split the pixel range differently -> compare to tolerance
    torch.testing.assert_close(outs[True][3], outs[False][3], rtol=2e-3, atol=2e-2)


def test_native_net_with_strided_tma_matches_default():
    """Whole ResNet-18 forward/backward with and without the parity-split copies: matching logits and gradients."""
    from rlr_b200.models import get_layout
    from rlr_b200.models.native import NativeNet
    torch.manual_seed(0)
    lay = get_layout("resnet18")
    B = 64
    w = lay.init_(torch.zeros(lay.n_total, device=DEV), 1)
    x = torch.randn(B, 32, 32, 3, device=DEV).to(BF)
    t = torch.randint(0, 10, (B,), device=DEV)
    res = {}
    old = nn.USE_STRIDED_TMA
    try:
        for mode in (False, "again", True):
            nn.USE_STRIDED_TMA = mode is True
            net = NativeNet(lay, DEV, B, impl="sm100")
            wi, g = w.clone(), torch.zeros_like(w)
            net.bind(wi, wi.to(BF), g)
            logits = net.forward(x, True).clone()
            _, dl = ops.softmax_xent(logits, t)
            net.backward(dl)
            torch.cuda.synchronize()
            res[mode] = (logits.float(), g[: lay.n_vote].clone())
    finally:
        nn.USE_STRIDED_TMA = old
    # BatchNorm statistics / split-K weight gradients are reduced with float atomics (order varies run to run, amplified by BatchNorm
    # at random init): the parity-copy path run twice is the yardstick for the strided path
    rel = lambda a, b: float((a.double() - b.double()).norm() / (b.double().norm() + 1e-12))
    assert float((res[False][0] - res[True][0]).abs().max() / res[False][0].abs().max()) < 2e-2
    noise, diff = rel(res["again"][1], res[False][1]), rel(res[True][1], res[False][1])
    print(f"strided TMA whole-net gradient: copy-vs-copy {noise:.2e}  strided-vs-copy {diff:.2e}")
    assert diff <= 3 * noise + 1e-3, (diff, noise)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,p", [(64, 32, 32, 3, 64, 3, 1), (32, 28, 28, 1, 32, 3, 0), (32, 32, 32, 3, 64, 3, 0), (256, 32, 32, 3, 64, 3, 1)])
def test_im2col_stem_conv_and_wgrad(B, H, W, Cin, Cout, k, p):
    """RLR_IM2COL_STEM: stem conv as one 64-deep GEMM k-block over gathered patches, weight gradient as a [Cout x 64] GEMM."""
    import torch.nn.functional as F
    torch.manual_seed(B + H + Cin)
    x = torch.randn(B, H, W, Cin, device=DEV).to(BF)
    w = (torch.randn(Cout, k, k, Cin, device=DEV) / (k * k * Cin) ** 0.5).to(BF)
    bias = torch.randn(Cout, device=DEV) * 0.1
    Ho, Wo = H + 2 * p - k + 1, W + 2 * p - k + 1
    dy = torch.randn(B, Ho, Wo, Cout, device=DEV).to(BF)
    old = nn.USE_IM2COL_STEM
    nn.USE_IM2COL_STEM = True
    try:
        tag = ("stem-test", B, H, Cin, k, p)
        y = torch.full((B, Ho, Wo, Cout), 7.0, device=DEV, dtype=BF)
        ops.conv2d_fwd_sm100(x, w, bias, y, 1, p, True, None, tag=tag)
        gw = torch.zeros(Cout, k, k, Cin, device=DEV)
        gb = torch.zeros(Cout, device=DEV)
        ops.conv2d_wgrad_sm100(x, dy, gw, gb, 1, p, tag=tag)
        torch.cuda.synchronize()
    finally:
        nn.USE_IM2COL_STEM = old
    xf, wf = x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2)
    ref = F.relu(F.conv2d(xf, wf, bias, 1, p)).permute(0, 2, 3, 1)
    assert float((y.float() - ref).abs().max() / ref.abs().max()) < 1e-2
    _, gw_ref, gb_ref = torch.ops.aten.convolution_backward(dy.float().permute(0, 3, 1, 2), xf, wf, [Cout], [1, 1], [p, p], [1, 1], False, [0, 0], 1,
                                                            [False, True, True])
    gw_ref = gw_ref.permute(0, 2, 3, 1)
    assert float((gw - gw_ref).abs().max() / gw_ref.abs().max()) < 1e-2
    torch.testing.assert_close(gb, gb_ref, rtol=1e-3, atol=1e-2 * (B * Ho * Wo) ** 0.5)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,s,p", [(128, 16, 16, 128, 128, 3, 1, 1), (256, 8, 8, 256, 256, 3, 1, 1), (128, 16, 16, 128, 256, 1, 2, 0)])
def test_conv_occ3_level2_matches_two_cta_kernel(B, H, W, Cin, Cout, k, s, p):
    """RLR_CONV_OCC3=2 (selects level 1: three CTAs per SM only for the 64-wide tile) -- bit-identical to level 0."""
    torch.manual_seed(B + H + Cin)
    x = torch.randn(B, H, W, Cin, device=DEV).to(BF)
    w = (torch.randn(Cout, k, k, Cin, device=DEV) / (k * k * Cin) ** 0.5).to(BF)
    bias = torch.randn(Cout, device=DEV) * 0.1
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy = torch.randn(B, Ho, Wo, Cout, device=DEV).to(BF)
    base = torch.randn(B, H, W, Cin, device=DEV).to(BF)
    outs = {}
    try:
        for level in (0, 2):
            ops.ext().set_conv_occ3(level)
            y = torch.full((B, Ho, Wo, Cout), 7.0, device=DEV, dtype=BF)
            ops.conv2d_fwd_sm100(x, w, bias, y, s, p, True, None, tag=("occ3x", level, B, H, Cin, k, s))
            dx = base.clone()
            ops.conv2d_dgrad_sm100(dy, w, dx, s, p, True)
            torch.cuda.synchronize()
            outs[level] = (y, dx)
    finally:
        ops.ext().set_conv_occ3(1)
    for a, b in zip(outs[0], outs[2]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("C,M", [(64, 65536), (128, 16384), (512, 4100), (256, 999)])
def test_bn_backward_with_recomputed_relu_mask(C, M):
    """RLR_BN_RECOMPUTE: BN+ReLU (no residual) backward derives the ReLU mask from x instead of reading y; must equal the
    y-based kernels up to the reduction order."""
    torch.manual_seed(C + M)
    x = (torch.randn(M, C, device=DEV) * 1.5 + 0.3).to(BF)
    gamma = torch.rand(C, device=DEV) + 0.5
    beta = torch.randn(C, device=DEV) * 0.2
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    mean_rstd = torch.zeros(2, C, device=DEV)
    y = torch.empty_like(x)
    nn.bn_fwd(x, y, None, gamma, beta, rm, rv, None, mean_rstd, M, 1e-5, 0.1, True, True, "sm100")
    dy = torch.randn(M, C, device=DEV).to(BF)
    res = {}
    old = nn.USE_BN_RECOMPUTE
    try:
        for mode in (False, True):
            nn.USE_BN_RECOMPUTE = mode
            dsum = torch.zeros(2, C, device=DEV)
            dx = torch.empty_like(x)
            dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
            nn.bn_bwd(dy, y, x, gamma, mean_rstd, dsum, dx, None, dg, db, True, "sm100", zero_dsum=True, beta=beta)
            torch.cuda.synchronize()
            res[mode] = (dx.float(), dg, db)
    finally:
        nn.USE_BN_RECOMPUTE = old
    # masks agree except where the pre-activation is within rounding of 0; the channel sums differ by reduction order only
    mism = (~torch.isclose(res[False][0], res[True][0], rtol=2e-2, atol=2e-2)).float().mean()
    assert float(mism) < 1e-3, float(mism)
    torch.testing.assert_close(res[True][1], res[False][1], rtol=2e-3, atol=2e-2 * M ** 0.5)
    torch.testing.assert_close(res[True][2], res[False][2], rtol=2e-3, atol=2e-2 * M ** 0.5)


def test_programmatic_dependent_launch_matches_plain_launches():
    """RLR_PDL: hot kernels launched with programmatic stream serialization (prologue overlaps the predecessor's tail, then
    griddepcontrol.wait).  Eager and CUDA-graph-captured ResNet-18 steps must reproduce the plain-launch results."""
    from rlr_b200.models import get_layout
    from rlr_b200.models.native import NativeNet
    torch.manual_seed(0)
    lay = get_layout("resnet18")
    B = 64
    w = lay.init_(torch.zeros(lay.n_total, device=DEV), 1)
    x = torch.randn(B, 32, 32, 3, device=DEV).to(BF)
    t = torch.randint(0, 10, (B,), device=DEV)
    res = {}
    try:
        for mode in ("plain", "plain2", "pdl", "pdl-graph"):
            ops.ext().set_pdl(mode.startswith("pdl"))
            net = NativeNet(lay, DEV, B, impl="sm100")
            wi, g = w.clone(), torch.zeros_like(w)
            net.bind(wi, wi.to(BF), g)

            def step():
                logits = net.forward(x, True)
                _, dl = ops.softmax_xent(logits, t)
                net.backward(dl)
                return logits

            logits = step()                       # eager (also allocates every scratch buffer before a capture)
            if mode == "pdl-graph":
                torch.cuda.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    logits = step()
                wi.copy_(w)                      # the eager step advanced the BatchNorm running statistics: restore, then replay
                gr.replay()
            torch.cuda.synchronize()
            res[mode] = (logits.float().clone(), g[: lay.n_vote].clone())
    finally:
        ops.ext().set_pdl(False)
    # the same step run twice with plain launches differs by the summation order of the split-K atomics, amplified by BatchNorm at
    # random init: that run-to-run difference is the yardstick (a whole-gradient cosine of ~0.98 is NORMAL here)
    rel = lambda a, b: float((a.double() - b.double()).norm() / (b.double().norm() + 1e-12))
    noise = rel(res["plain2"][1], res["plain"][1])
    for mode in ("pdl", "pdl-graph"):
        assert float((res["plain"][0] - res[mode][0]).abs().max() / res["plain"][0].abs().max()) < 2e-2, mode
        assert rel(res[mode][1], res["plain"][1]) <= 3 * noise + 1e-3, (mode, rel(res[mode][1], res["plain"][1]), noise)


@pytest.mark.parametrize("B,K,N,relu", [(256, 512, 10, False), (100, 256, 10, False), (37, 128, 10, True), (256, 1024, 16, False)])
def test_head_kernels_v2(B, K, N, relu):
    """RLR_HEAD_V2 classifier-head kernels against fp32 references (forward, dX with/without accumulation, dW, db)."""
    torch.manual_seed(B + K)
    x = torch.randn(B, K, device=DEV).to(BF)
    w = (torch.randn(N, K, device=DEV) / K ** 0.5).to(BF)
    bias = torch.randn(N, device=DEV) * 0.1
    dy = (torch.randn(B, N, device=DEV) / B).to(BF)
    base = torch.randn(B, K, device=DEV).to(BF)
    old = nn.USE_HEAD_V2
    nn.USE_HEAD_V2 = True
    try:
        y = torch.empty(B, N, device=DEV, dtype=BF)
        nn.linear_fwd(x, w, bias, y, relu, "sm100")
        dx0, dx1 = torch.empty_like(x), base.clone()
        dw, db = torch.full((N, K), 3.0, device=DEV), torch.full((N,), 3.0, device=DEV)
        nn.linear_bwd(x, dy, w, dx0, dw, db, False, "sm100", zero=True)
        dw2, db2 = torch.zeros(N, K, device=DEV), torch.zeros(N, device=DEV)
        nn.linear_bwd(x, dy, w, dx1, dw2, db2, True, "sm100", zero=False)
        torch.cuda.synchronize()
    finally:
        nn.USE_HEAD_V2 = old
    ref = x.float() @ w.float().t() + bias
    if relu:
        ref = ref.clamp_min(0)
    assert float((y.float() - ref).abs().max() / ref.abs().max()) < 1e-2
    dxr = dy.float() @ w.float()
    assert float((dx0.float() - dxr).abs().max() / dxr.abs().max()) < 1e-2
    assert float((dx1.float() - (dxr + base.float())).abs().max() / (dxr + base.float()).abs().max()) < 1e-2
    dwr, dbr = dy.float().t() @ x.float(), dy.float().sum(0)
    for got_w, got_b in ((dw, db), (dw2, db2)):
        torch.testing.assert_close(got_w, dwr, rtol=1e-3, atol=1e-4)
        torch.testing.assert_close(got_b, dbr, rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("B,H,W,Cout,acc", [(64, 32, 32, 64, False), (37, 16, 16, 64, True), (8, 32, 32, 128, False), (5, 16, 8, 32, False),
                                            (256, 32, 32, 64, True), (3, 16, 24, 64, False)])
def test_conv3x3_halo3_kernel(B, H, W, Cout, acc):
    """RLR_HALO3: three filter taps per N = 192 MMA over one A view, column shift-add with warp shuffles in the epilogue, tiles
    advancing by six columns -- against the fp32 reference (and the nine-MMA halo kernel for the error scale)."""
    import torch.nn.functional as F
    torch.manual_seed(B + H)
    x = torch.randn(B, H, W, 64, device=DEV).to(BF)
    w = (torch.randn(Cout, 3, 3, 64, device=DEV) / 24).to(BF)
    bias = torch.randn(Cout, device=DEV) * 0.1
    base = torch.randn(B, H, W, Cout, device=DEV).to(BF)
    ref = F.relu(F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), bias, 1, 1)).permute(0, 2, 3, 1)
    if acc:
        ref = ref + base.float()
    y3 = base.clone() if acc else torch.full_like(base, 5.0)
    ops.ext().conv3x3_halo3_bf16(x, w.reshape(Cout, 576), y3, bias, True, acc)
    y1 = base.clone() if acc else torch.full_like(base, 5.0)
    if W % 8 == 0:
        ops.ext().conv3x3_halo_bf16(x, w.reshape(Cout, 576), y1, bias, True, acc, None, 0, None)
    torch.cuda.synchronize()
    e3 = float((y3.float() - ref).abs().max() / ref.abs().max())
    e1 = float((y1.float() - ref).abs().max() / ref.abs().max()) if W % 8 == 0 else float("nan")
    print(f"halo3 rel err {e3:.2e} (nine-MMA halo kernel {e1:.2e})")
    assert e3 < 1e-2


def test_agents_in_flight_matches_sequential_training():
    """--agents_in_flight 2: two agents of a round train concurrently on one GPU (own trainer and CUDA stream each); the aggregated
    parameters must match the sequential schedule up to float-atomic ordering (yardstick: two sequential runs against each other;
    FedAvg without the discontinuous sign vote)."""
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args

    def run(n_flight):
        args = make_args(data="cifar10", model="resnet18", num_agents=4, local_ep=1, bs=64, synthetic=256, synthetic_val=128, log_dir="",
                         device=DEV, seed=2, agents_in_flight=n_flight)
        eng = FLEngine(args, verbose=False)
        assert len(eng.trainers) == n_flight
        eng.run_round(1)
        loss, _ = eng.round_result()
        w = eng.global_params()[: eng.layout.n_vote].clone()
        torch.cuda.synchronize()
        eng.close()
        return w, loss
    rel = lambda a, b: float((a.double() - b.double()).norm() / (b.double().norm() + 1e-12))
    (wa, la), (wb, lb), (wc, lc) = run(1), run(1), run(2)
    noise, diff = rel(wb, wa), rel(wc, wa)
    print(f"agents_in_flight: sequential-vs-sequential {noise:.2e}, concurrent-vs-sequential {diff:.2e}; losses {la:.3f} {lb:.3f} {lc:.3f}")
    assert diff <= 3 * noise + 1e-5, (diff, noise)
    assert abs(lc - la) <= 3 * abs(lb - la) + 1e-3 * abs(la)


def test_small_batch_gemm_shapes():
    """Linear layers of the small CNNs as the wgmma GEMM sees them (M = 256): correctness at these shapes with whatever tile
    heuristic is active (run with RLR_GEMM_SMALL_BN64=1 to cover the 64-wide choice); prints the device time of each."""
    for M, N, K in [(256, 128, 9216), (256, 128, 1024), (256, 256, 128), (64, 128, 9216)]:
        torch.manual_seed(K)
        A = torch.randn(M, K, device=DEV).to(BF)
        Bm = (torch.randn(N, K, device=DEV) / K ** 0.5).to(BF)
        bias = torch.randn(N, device=DEV) * 0.1
        out = torch.empty(M, N, device=DEV, dtype=BF)
        ops.ext().gemm_bf16(A, Bm, out, bias, True, False, None)
        ref = torch.relu(A.float() @ Bm.float().t() + bias)
        assert float((out.float() - ref).abs().max() / ref.abs().max()) < 1e-2
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            ops.ext().gemm_bf16(A, Bm, out, bias, True, False, None)
        e1.record(); torch.cuda.synchronize()
        print(f"gemm {M}x{N}x{K}: {e0.elapsed_time(e1) / 20 * 1000:.1f} us")


@pytest.mark.parametrize("M,N,K,relu", [(256, 128, 9216, True), (64, 128, 9216, False), (256, 256, 1024, True), (100, 192, 2048, False)])
def test_splitk_gemm(M, N, K, relu):
    """RLR_SPLITK: grid.z CTAs share a tile's k range and add fp32 partials into a workspace; finish pass applies bias / ReLU, packs
    bf16 and re-zeroes the workspace (second call must give the same result)."""
    torch.manual_seed(M + K)
    A = torch.randn(M, K, device=DEV).to(BF)
    Bm = (torch.randn(N, K, device=DEV) / K ** 0.5).to(BF)
    bias = torch.randn(N, device=DEV) * 0.1
    ws = torch.zeros(M, N, device=DEV)
    ref = A.float() @ Bm.float().t() + bias
    if relu:
        ref = ref.clamp_min(0)
    for _ in range(2):
        out = torch.full((M, N), 9.0, device=DEV, dtype=BF)
        ops.ext().gemm_splitk_bf16(A, Bm, out, ws, bias, relu)
        torch.cuda.synchronize()
        assert float((out.float() - ref).abs().max() / ref.abs().max()) < 1e-2
        assert float(ws.abs().max()) == 0.0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        ops.ext().gemm_splitk_bf16(A, Bm, out, ws, bias, relu)
    e1.record(); torch.cuda.synchronize()
    print(f"split-K gemm {M}x{N}x{K}: {e0.elapsed_time(e1) / 20 * 1000:.1f} us (two kernels)")
