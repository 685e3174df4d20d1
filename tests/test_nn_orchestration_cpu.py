"""CPU check of the HOST-SIDE orchestration in ops/nn.py (tap tables, parity planes, padding, scratch reuse, opt-in code paths)
against PyTorch convolutions, with the CUDA extension replaced by a small fp32 emulator of each kernel's documented contract
(ops/csrc/gemm_binding.cpp).  The kernels themselves are tested on the GPU (tests/test_gpu_native.py, test_gpu_variants.py);
this suite makes sure that what Python hands them is right -- in particular for paths that could not be run on hardware yet."""
import pytest
import torch
import torch.nn.functional as F

import rlr_b200  # noqa: F401
from rlr_b200.ops import nn


def _gather(x, n_idx, hh, ww):
    """x[n_idx, hh, ww, :] with zeros outside the image; hh / ww are [Ho, Wo] index grids."""
    NB_tot, H, W, C = x.shape
    ok = (hh >= 0) & (hh < H) & (ww >= 0) & (ww < W)
    v = x[n_idx][:, hh.clamp(0, H - 1), ww.clamp(0, W - 1), :]          # [N, Ho, Wo, C]
    return v * ok[None, :, :, None]


class FakeExt:
    """fp32 emulation of the extension entry points used by the convolution wrappers."""

    def __init__(self):
        self.calls = []

    # ---- layout helpers ------------------------------------------------------------------------------------------------
    def space_to_depth(self, x, x4):
        self.calls.append("space_to_depth")
        NB = x.shape[0]
        for ph in range(2):
            for pw in range(2):
                pl = ph * 2 + pw
                x4[pl * NB:(pl + 1) * NB] = x[:, ph::2, pw::2]

    def depth_to_space(self, x4, y, accumulate, mask):
        self.calls.append("depth_to_space")
        NB = y.shape[0]
        if not accumulate:
            y.zero_()
        for ph in range(2):
            for pw in range(2):
                pl = ph * 2 + pw
                if mask >> pl & 1:
                    y[:, ph::2, pw::2] += x4[pl * NB:(pl + 1) * NB]

    def filter_transpose(self, w, wt, Cout, T, Cin):
        self.calls.append("filter_transpose")
        w3 = w.reshape(Cout, T, Cin)
        wt.copy_(w3.flip(1).permute(2, 1, 0).reshape(wt.shape))          # wt[ci][T-1-t][co] = w[co][t][ci]

    def filter_gather_transpose(self, w, wt, Cout, T, Cin, taps):
        self.calls.append("filter_gather_transpose")
        w3 = w.reshape(Cout, T, Cin)
        wt.copy_(w3[:, list(taps), :].permute(2, 1, 0).reshape(wt.shape))  # wt[ci][i][co] = w[co][taps[i]][ci]

    # ---- implicit-GEMM convolution -------------------------------------------------------------------------------------
    def _conv(self, x, w, out, NB, dh, dw, dplane, bias, relu, accumulate, wtap, w_taps_total, in_stride, out_stride, ph, pw):
        Cin = x.shape[3]
        Cout = out.shape[3]
        Ho, Wo = out.shape[1] // out_stride, out.shape[2] // out_stride
        hh, ww = torch.meshgrid(torch.arange(Ho), torch.arange(Wo), indexing="ij")
        acc = torch.zeros(NB, Ho, Wo, Cout)
        n_idx = torch.arange(NB)
        for t in range(len(dh)):
            v = _gather(x, n_idx + dplane[t] * NB, in_stride * hh + dh[t], in_stride * ww + dw[t])
            if wtap:       # MN-major B: w is [K = Cin_here][w_taps_total * Cout_here]
                Wt = w[:, wtap[t] * Cout:(wtap[t] + 1) * Cout]           # [Cin][Cout]
                acc += v @ Wt
            else:          # K-major B: w is [Cout][T * Cin]
                Wt = w[:, t * Cin:(t + 1) * Cin]                          # [Cout][Cin]
                acc += v @ Wt.t()
        if bias is not None:
            acc += bias
        if relu:
            acc = acc.clamp_min(0)
        view = out[:, ph::out_stride, pw::out_stride]
        if accumulate:
            view += acc
        else:
            view.copy_(acc)

    def conv_bf16(self, x, w, out, NB, planes, dh, dw, dplane, bias, relu, accumulate, stats, wtap, w_taps_total):
        self.calls.append("conv_bf16")
        assert x.shape[0] == planes * NB and out.shape[0] == NB
        self._conv(x, w, out, NB, dh, dw, dplane, bias, relu, accumulate, list(wtap), w_taps_total, 1, 1, 0, 0)
        if stats is not None:                       # epilogue statistics: [slots][sum, sum^2][Cout] partials ADDED to (kernel contract)
            assert not accumulate and not wtap and stats.shape[-2:] == (2, out.shape[3])
            self.calls.append("conv_bf16+stats")
            o = out.reshape(-1, out.shape[3]).float()
            stats.reshape(-1, 2, out.shape[3])[0, 0] += o.sum(0)
            stats.reshape(-1, 2, out.shape[3])[0, 1] += (o * o).sum(0)

    def conv_bf16_strided(self, x, w, out, dh, dw, bias, relu, accumulate, wtap, w_taps_total, in_stride, out_stride, ph, pw):
        self.calls.append("conv_bf16_strided")
        assert x.shape[0] == out.shape[0]
        self._conv(x, w, out, x.shape[0], dh, dw, [0] * len(dh), bias, relu, accumulate, list(wtap), w_taps_total, in_stride, out_stride, ph, pw)

    def conv3x3_halo_bf16(self, x, w, out, bias, relu, accumulate, stats, bo_mode, dbg):
        self.calls.append("conv3x3_halo_bf16")
        pad = (out.shape[1] - x.shape[1] + 2) // 2                       # valid / same / full (conv_halo.cu launcher contract)
        assert pad in (0, 1, 2) and out.shape[1] == x.shape[1] + 2 * pad - 2 and out.shape[2] == x.shape[2] + 2 * pad - 2
        assert x.shape[3] == 64 and (stats is None or (out.shape[1] % 16 == 0 and out.shape[2] % 8 == 0))
        dh = [d - pad for d in range(3) for _ in range(3)]
        dw = [d - pad for _ in range(3) for d in range(3)]
        self._conv(x, w, out, x.shape[0], dh, dw, [0] * 9, bias, relu, accumulate, [], 0, 1, 1, 0, 0)

    def conv3x3_halo3_bf16(self, x, w, out, bias, relu, accumulate):
        self.calls.append("conv3x3_halo3_bf16")
        self.conv3x3_halo_bf16(x, w, out, bias, relu, accumulate, None, 0, None)
        self.calls.pop()

    # ---- weight gradients ---------------------------------------------------------------------------------------------
    def _wgrad(self, dy, x, dW, NB, cin_valid, dh, dw, dplane, in_stride):
        Cout = dy.shape[3]
        Ho, Wo = dy.shape[1], dy.shape[2]
        hh, ww = torch.meshgrid(torch.arange(Ho), torch.arange(Wo), indexing="ij")
        g = dW.view(Cout, len(dh), cin_valid)
        n_idx = torch.arange(NB)
        for t in range(len(dh)):
            v = _gather(x, n_idx + dplane[t] * NB, in_stride * hh + dh[t], in_stride * ww + dw[t])[..., :cin_valid]
            g[:, t, :] += torch.einsum("nhwo,nhwi->oi", dy, v)

    def conv_wgrad_bf16(self, dy, x, dW, NB, planes, cin_valid, dh, dw, dplane):
        self.calls.append("conv_wgrad_bf16")
        assert x.shape[0] == planes * NB
        self._wgrad(dy, x, dW, NB, cin_valid, dh, dw, dplane, 1)

    def conv_wgrad_bf16_strided(self, dy, x, dW, cin_valid, dh, dw, in_stride):
        self.calls.append("conv_wgrad_bf16_strided")
        self._wgrad(dy, x, dW, x.shape[0], cin_valid, dh, dw, [0] * len(dh), in_stride)

    def conv_wgrad_halo_bf16(self, dy, x, dW, cin_valid):
        self.calls.append("conv_wgrad_halo_bf16")
        dh = [d - 1 for d in range(3) for _ in range(3)]
        dw = [d - 1 for _ in range(3) for d in range(3)]
        self._wgrad(dy, x, dW, x.shape[0], cin_valid, dh, dw, [0] * 9, 1)

    # ---- GEMM-shaped helpers (stem path) -------------------------------------------------------------------------------
    def im2col_small(self, x, A, k, pad):
        self.calls.append("im2col_small")
        NB, H, W, C = x.shape
        Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
        hh, ww = torch.meshgrid(torch.arange(Ho), torch.arange(Wo), indexing="ij")
        A.zero_()
        A3 = A.view(NB, Ho, Wo, 64)
        for t in range(k * k):
            A3[..., t * C:(t + 1) * C] = _gather(x, torch.arange(NB), hh + t // k - pad, ww + t % k - pad)

    def gemm_bf16(self, A, B, out, bias, relu, accumulate, stats):
        self.calls.append("gemm_bf16")
        r = A @ B.t()
        if bias is not None:
            r = r + bias
        if relu:
            r = r.clamp_min(0)
        if accumulate:
            out += r
        else:
            out.copy_(r)

    def stem_gemm_bf16(self, A, W, out, bias, relu, stats, ready_ptr, lo, hi, epoch):
        self.calls.append("stem_gemm_bf16")
        assert A.shape[1] == 64 and W.shape[1] <= 64 and stats is None and ready_ptr == 0
        r = A[:, :W.shape[1]] @ W.t()
        if bias is not None:
            r = r + bias
        out.copy_(r.clamp_min(0) if relu else r)

    def linear_wgrad_bf16(self, dy, x, dW):
        self.calls.append("linear_wgrad_bf16")
        dW += dy.t() @ x

    # ---- BatchNorm backward (contracts of bn_bwd / bn_bwd_recompute in gemm_binding.cpp) ---------------------------------
    def _bn_bwd(self, dz, x, gamma, mean_rstd, dsum, dx, dres, dgamma, dbeta, zero_dsum):
        C = x.shape[-1]
        xf, dzf = x.reshape(-1, C), dz.reshape(-1, C)
        M = xf.shape[0]
        xhat = (xf - mean_rstd[0]) * mean_rstd[1]
        if zero_dsum:
            dsum.zero_()
        d3 = dsum.view(-1, 2, C)                      # [slots][2][C]: the kernels spread their atomics over the slots, consumers sum them
        d3[0, 0] += dzf.sum(0)
        d3[0, 1] += (dzf * xhat).sum(0)
        d2 = d3.sum(0)
        if dres is not None:
            dres.copy_(dzf.reshape(dres.shape))
        dx.copy_((gamma * mean_rstd[1] * (dzf - d2[0] / M - xhat * d2[1] / M)).reshape(dx.shape))
        dgamma.copy_(d2[1]); dbeta.copy_(d2[0])

    def bn_bwd(self, dy, y, x, gamma, mean_rstd, dsum, dx, dres, dgamma, dbeta, relu, zero_dsum):
        self.calls.append("bn_bwd")
        dz = dy * (y > 0) if relu else dy
        self._bn_bwd(dz, x, gamma, mean_rstd, dsum, dx, dres, dgamma, dbeta, zero_dsum)

    def bn_bwd_recompute(self, dy, x, gamma, beta, mean_rstd, dsum, dx, dgamma, dbeta, zero_dsum):
        self.calls.append("bn_bwd_recompute")
        sc = gamma * mean_rstd[1]
        mask = (x * sc + (beta - mean_rstd[0] * sc)) > 0              # the forward's own scale / shift expression
        self._bn_bwd(dy * mask, x, gamma, mean_rstd, dsum, dx, None, dgamma, dbeta, zero_dsum)

    def channel_stats(self, x, st):
        self.calls.append("channel_stats")
        xf = x.reshape(-1, x.shape[-1])
        s3 = st.view(-1, 2, x.shape[-1])              # [slots][2][C]
        s3[0, 0] += xf.sum(0)
        s3[0, 1] += (xf * xf).sum(0)

    def bias_grad(self, dy, db):
        self.calls.append("bias_grad")
        db += dy.reshape(-1, dy.shape[-1]).float().sum(0)

    def pad_rows(self, src, dst):
        self.calls.append("pad_rows")
        dst.zero_()
        dst[:, :src.shape[1]] = src

    def unpad_add(self, src, dst):
        self.calls.append("unpad_add")
        dst += src[:, :dst.shape[1]]

    def memset_zero(self, t):
        t.zero_()


@pytest.fixture
def fake(monkeypatch):
    ext = FakeExt()
    monkeypatch.setattr(nn, "_ext", lambda: ext)
    monkeypatch.setattr(nn, "_scratch", {})
    monkeypatch.setattr(nn, "_s2d_done", {})
    for flag in ("USE_STRIDED_TMA", "USE_IM2COL_STEM", "USE_HALO3"):
        monkeypatch.setattr(nn, flag, False)
    return ext


def _reference(x, w, bias, dy, s, p):
    xn = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
    wn = w.permute(0, 3, 1, 2).clone().requires_grad_(True)
    b = bias.clone().requires_grad_(True)
    y = F.relu(F.conv2d(xn, wn, b, s, p))
    yl = F.conv2d(xn, wn, None, s, p)                                  # the backward entry points act on the pre-activation
    yl.backward(dy.permute(0, 3, 1, 2))
    return y.detach().permute(0, 2, 3, 1), xn.grad.permute(0, 2, 3, 1), wn.grad.permute(0, 2, 3, 1), dy.sum((0, 1, 2))


CASES = [  # B, H, W, Cin, Cout, k, stride, pad
    (2, 8, 8, 64, 128, 3, 2, 1), (2, 8, 8, 64, 128, 1, 2, 0), (3, 4, 8, 128, 64, 3, 2, 1), (2, 16, 8, 64, 64, 3, 1, 1), (2, 6, 6, 64, 128, 3, 1, 0),
    (2, 8, 8, 128, 128, 3, 1, 1), (2, 8, 8, 3, 64, 3, 1, 1), (2, 10, 10, 1, 32, 3, 1, 0), (2, 8, 8, 128, 64, 1, 1, 0),
    (2, 26, 26, 32, 64, 3, 1, 0), (2, 15, 15, 64, 128, 3, 1, 0),          # valid convs of the reference CNNs: halo kernel, pad 0 / full dgrad
]


@pytest.mark.parametrize("mode", ["default", "strided", "stem", "halo3"])
@pytest.mark.parametrize("B,H,W,Cin,Cout,k,s,p", CASES)
def test_conv_wrappers_hand_the_kernels_the_right_problem(fake, monkeypatch, mode, B, H, W, Cin, Cout, k, s, p):
    monkeypatch.setattr(nn, "USE_STRIDED_TMA", mode == "strided")
    monkeypatch.setattr(nn, "USE_IM2COL_STEM", mode == "stem")
    monkeypatch.setattr(nn, "USE_HALO3", mode == "halo3")
    torch.manual_seed(B + H + Cin + k)
    x = torch.randn(B, H, W, Cin)
    w = torch.randn(Cout, k, k, Cin) / (k * k * Cin) ** 0.5
    bias = torch.randn(Cout) * 0.1
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy = torch.randn(B, Ho, Wo, Cout)
    y_ref, dx_ref, gw_ref, gb_ref = _reference(x, w, bias, dy, s, p)

    y = torch.full((B, Ho, Wo, Cout), 7.0)
    nn.conv2d_fwd_sm100(x, w, bias, y, s, p, True, None, tag=("t", mode), s2d_epoch=1)
    torch.testing.assert_close(y, y_ref, rtol=1e-4, atol=1e-4)

    gw, gb = torch.zeros(Cout, k, k, Cin), torch.zeros(Cout)
    nn.conv2d_wgrad_sm100(x, dy, gw, gb, s, p, tag=("t", mode))
    torch.testing.assert_close(gw, gw_ref, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(gb, gb_ref, rtol=1e-4, atol=1e-4)

    if Cin % 8 == 0 and Cout % 64 == 0:                                  # conv_supported(..., "dgrad")
        base = torch.randn(B, H, W, Cin)
        dx0, dx1 = torch.full_like(base, 3.0), base.clone()
        nn.conv2d_dgrad_sm100(dy, w, dx0, s, p, False)
        nn.conv2d_dgrad_sm100(dy, w, dx1, s, p, True)
        torch.testing.assert_close(dx0, dx_ref, rtol=1e-4, atol=1e-4)
        torch.testing.assert_close(dx1, dx_ref + base, rtol=1e-4, atol=1e-4)

    # the mode really took the path it names
    if mode == "strided" and s == 2:
        assert "conv_bf16_strided" in fake.calls and "conv_wgrad_bf16_strided" in fake.calls
        assert "space_to_depth" not in fake.calls and "depth_to_space" not in fake.calls
    if mode == "default" and s == 2:
        assert "space_to_depth" in fake.calls
    if mode == "stem" and Cin * k * k <= 64 and s == 1:
        assert fake.calls.count("im2col_small") == 1 and "stem_gemm_bf16" in fake.calls and "linear_wgrad_bf16" in fake.calls
    if mode == "halo3" and nn._halo_ok(k, s, p, Cin, H, W) and p == 1 and H % 16 == 0:
        assert "conv3x3_halo3_bf16" in fake.calls and "conv3x3_halo_bf16" not in fake.calls
    if mode == "default" and (H, p) in ((26, 0), (15, 0)):
        # forward through the halo kernel; the data gradient too when ITS input (dy) has 64 channels
        assert fake.calls.count("conv3x3_halo_bf16") == (3 if Cout == 64 else 1) and ("conv_bf16" in fake.calls) == (Cout != 64)


def test_shared_parity_copy_is_made_once_per_forward(fake):
    """The 3x3/s2 conv and the 1x1/s2 shortcut of a ResNet block read the same input: one space_to_depth per forward epoch."""
    x = torch.randn(2, 8, 8, 64)
    w3, w1 = torch.randn(128, 3, 3, 64), torch.randn(128, 1, 1, 64)
    y = torch.empty(2, 4, 4, 128)
    for epoch in (1, 2):
        nn.conv2d_fwd_sm100(x, w3, None, y, 2, 1, False, None, tag="a", s2d_epoch=epoch)
        nn.conv2d_fwd_sm100(x, w1, None, y, 2, 0, False, None, tag="b", s2d_epoch=epoch)
    assert fake.calls.count("space_to_depth") == 2


@pytest.mark.parametrize("mode", ["default", "strided", "stem"])
@pytest.mark.parametrize("model", ["resnet18", "cnn_cifar"])
def test_native_plan_with_kernel_conv_paths_matches_library_convs(fake, monkeypatch, model, mode):
    """Whole network on CPU: the executor's plan with the convolution wrappers of ops/nn.py (emulated kernels) against the same plan
    with library convolutions -- catches wrong buffers / tags / accumulate flags in how models/native.py drives the conv paths."""
    from rlr_b200.models import get_layout
    from rlr_b200.models.native import NativeNet
    from rlr_b200 import ops
    monkeypatch.setattr(nn, "USE_STRIDED_TMA", mode == "strided")
    monkeypatch.setattr(nn, "USE_IM2COL_STEM", mode == "stem")
    import rlr_b200.models.native as native_mod
    monkeypatch.setattr(native_mod, "EPILOGUE_BN_STATS", True)     # opt-in path: keep its plumbing covered
    torch.manual_seed(0)
    lay = get_layout(model)
    for nd in lay.nodes:
        if nd.op == "dropout":
            nd.attrs["p"] = 0.0
    B = 4
    w = lay.init_(torch.zeros(lay.n_total), 1)
    C, H, W = lay.in_shape
    x = torch.randn(B, H, W, C)
    t = torch.randint(0, 10, (B,))
    res = {}
    for name, conv_impl in (("lib", "aten"), ("kern", "sm100")):
        impl = dict(conv_fwd=conv_impl, conv_dgrad=conv_impl, conv_wgrad=conv_impl, bn="aten", pool="aten", linear="aten", dropout="aten")
        net = NativeNet(lay, "cpu", B, impl=impl, act_dtype=torch.float32)
        wi, g = w.clone(), torch.zeros_like(w)
        net.bind(wi, wi.clone(), g)
        logits = net.forward(x, True).clone()
        _, dl = ops.softmax_xent(logits, t)
        net.backward(dl)
        res[name] = (logits, g[: lay.n_vote].clone())
    torch.testing.assert_close(res["kern"][0], res["lib"][0], rtol=1e-3, atol=1e-3)
    cos = F.cosine_similarity(res["kern"][1].double(), res["lib"][1].double(), dim=0)
    assert float(cos) > 0.9999, float(cos)
    assert "conv_bf16" in fake.calls or "conv_bf16_strided" in fake.calls or "gemm_bf16" in fake.calls
    if model == "resnet18":     # BatchNorm statistics came out of the conv epilogue for the stride-1 convs on the generic kernel (9 of 20)
        assert fake.calls.count("conv_bf16+stats") == 9 and fake.calls.count("channel_stats") == 0   # (bn impl is aten here: no stats kernel at all)


@pytest.mark.parametrize("recompute", [False, True])
@pytest.mark.parametrize("relu,with_res", [(True, False), (True, True), (False, False)])
def test_bn_backward_wrapper_paths(fake, monkeypatch, recompute, relu, with_res):
    """nn.bn_bwd: the y-based kernels vs the mask-recomputing variant (only legal for BN+ReLU without a residual) vs the library
    formulation, all on the same saved statistics."""
    monkeypatch.setattr(nn, "USE_BN_RECOMPUTE", recompute)
    torch.manual_seed(3)
    M, C = 96, 16
    x = torch.randn(M, C) * 1.5 + 0.2
    gamma, beta = torch.rand(C) + 0.5, torch.randn(C) * 0.3
    mean, var = x.mean(0), x.var(0, unbiased=False)
    mean_rstd = torch.stack([mean, torch.rsqrt(var + 1e-5)])
    res = torch.randn(M, C) if with_res else None
    pre = (x - mean) * mean_rstd[1] * gamma + beta + (res if with_res else 0)
    y = pre.clamp_min(0) if relu else pre
    dy = torch.randn(M, C)
    outs = {}
    for impl in ("aten", "sm100"):
        dsum, dx = torch.zeros(2, C), torch.empty(M, C)
        dres = torch.empty(M, C) if with_res else None
        dg, db = torch.zeros(C), torch.zeros(C)
        nn.bn_bwd(dy, y, x, gamma, mean_rstd, dsum, dx, dres, dg, db, relu, impl, zero_dsum=True, beta=beta)
        outs[impl] = (dx, dg, db, dres)
    for a, b in zip(outs["aten"], outs["sm100"]):
        if a is not None:
            torch.testing.assert_close(b, a, rtol=1e-4, atol=1e-5)
    used = "bn_bwd_recompute" in fake.calls
    assert used == (recompute and relu and not with_res)


def test_halo3_tile_algorithm_emulation():
    """Scalar emulation of conv_halo3.cu's arithmetic: 8 x 18 pixel boxes advancing by 6 columns, one accumulator block per dx tap
    over a single A view per filter row, out = D_1 + shfl_up(D_0) + shfl_down(D_2) inside 32-lane warps, lanes 1..6 of each 8-lane
    group valid -- must reproduce a padded 3x3 convolution exactly (geometry, shift directions, masks)."""
    torch.manual_seed(0)
    NB, H, W, Cin, Cout = 2, 16, 20, 4, 8
    x = torch.randn(NB, H, W, Cin)
    w = torch.randn(Cout, 9, Cin)
    ref = F.conv2d(x.permute(0, 3, 1, 2), w.reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2), None, 1, 1).permute(0, 2, 3, 1)
    out = torch.full((NB, H, W, Cout), float("nan"))
    xp = F.pad(x, (0, 0, 8, 8, 1, 1))                                    # zero fill = TMA out-of-bounds behaviour (cols +-8, rows +-1)
    m = torch.arange(128)
    hl, wl = m // 8, m % 8
    lane = m % 32
    for n in range(NB):
        for th in range(H // 16):
            for tw in range((W + 5) // 6):
                h0, c0, oc0 = th * 16, tw * 6 - 1, tw * 6
                D = torch.zeros(128, 3, Cout)
                for dy in range(3):
                    a = xp[n, h0 + hl + dy - 1 + 1, c0 + wl + 8]          # A view of filter row dy: box rows (h + dy), all 8 columns
                    for j in range(3):
                        D[:, j] += a @ w[:, dy * 3 + j, :].t()
                up = torch.where((lane >= 1)[:, None], D[(m - 1).clamp(0), 0], D[:, 0])          # __shfl_up_sync(d0, 1)
                dn = torch.where((lane <= 30)[:, None], D[(m + 1).clamp(max=127), 2], D[:, 2])   # __shfl_down_sync(d2, 1)
                val = D[:, 1] + up + dn
                c = oc0 + wl - 1
                ok = (wl >= 1) & (wl <= 6) & (h0 + hl < H) & (c < W)
                out[n, (h0 + hl)[ok], c[ok]] = val[ok]
    assert not torch.isnan(out).any()
    torch.testing.assert_close(out, ref, rtol=1e-4, atol=1e-4)


def _pow2_ceil(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def _simulate_conv_kernel_indexing(x, w2d, NB, Ho, Wo, Cout, dh, dw, in_stride, out_stride, ph, pw):
    """Python transcription of the index arithmetic of launch_conv_bf16 + umma_conv_gemm_kernel (ops/csrc/gemm.cu): tile shape
    TW x TH x TN = 128 output pixels, tile origin, per-row global output index `gi`, and the TMA box of tap t starting at
    (w0 * in_stride + dw[t], h0 * in_stride + dh[t], n0) with element strides (in_stride, in_stride) and zero fill out of bounds."""
    Hin, Win, Cin = x.shape[1], x.shape[2], x.shape[3]
    TW = min(_pow2_ceil(Wo), 128)
    TH = _pow2_ceil(Ho)
    if TW * TH > 128:
        TH = 128 // TW
    TN = 128 // (TW * TH)
    tiles_w, tiles_h, tiles_n = -(-Wo // TW), -(-Ho // TH), -(-NB // TN)
    OutH, OutW = Ho * out_stride, Wo * out_stride
    out = torch.full((NB * OutH * OutW, Cout), float("nan"))
    for tile_m in range(tiles_w * tiles_h * tiles_n):
        w0, h0, n0 = (tile_m % tiles_w) * TW, ((tile_m // tiles_w) % tiles_h) * TH, (tile_m // (tiles_w * tiles_h)) * TN
        r = torch.arange(128)
        tw, th, tn = r % TW, (r // TW) % TH, r // (TW * TH)
        w_, h_, n_ = w0 + tw, h0 + th, n0 + tn
        valid = (w_ < Wo) & (h_ < Ho) & (n_ < NB)
        gi = (n_ * OutH + h_ * out_stride + ph) * OutW + w_ * out_stride + pw
        acc = torch.zeros(128, Cout)
        for t in range(len(dh)):
            cw, ch = w0 * in_stride + dw[t] + tw * in_stride, h0 * in_stride + dh[t] + th * in_stride     # box element (tw, th)
            inb = (cw >= 0) & (cw < Win) & (ch >= 0) & (ch < Hin) & (n_ < NB)
            a = x[n_.clamp(max=NB - 1), ch.clamp(0, Hin - 1), cw.clamp(0, Win - 1)] * inb[:, None]
            acc += a @ w2d[:, t * Cin:(t + 1) * Cin].t()
        out[gi[valid]] = acc[valid]
    return out.view(NB, OutH, OutW, Cout)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,p", [(3, 8, 8, 8, 16, 3, 1), (2, 16, 16, 8, 8, 1, 0), (5, 4, 4, 8, 8, 3, 1), (1, 32, 32, 8, 8, 3, 1)])
def test_kernel_index_arithmetic_for_strided_input_and_output(B, H, W, Cin, Cout, k, p):
    """The two additions to the generic conv kernel's index math -- strided TMA boxes for stride-2 forward convolutions and strided
    output rows for the parity planes of stride-2 data gradients -- reproduce PyTorch when transcribed literally."""
    torch.manual_seed(B + H)
    x = torch.randn(B, H, W, Cin)
    w = torch.randn(Cout, k, k, Cin)
    Ho, Wo = (H + 2 * p - k) // 2 + 1, (W + 2 * p - k) // 2 + 1
    dh = [d - p for d in range(k) for _ in range(k)]
    dw = [d - p for _ in range(k) for d in range(k)]
    y = _simulate_conv_kernel_indexing(x, w.reshape(Cout, -1), B, Ho, Wo, Cout, dh, dw, 2, 1, 0, 0)
    ref = F.conv2d(x.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), None, 2, p).permute(0, 2, 3, 1)
    torch.testing.assert_close(y, ref, rtol=1e-4, atol=1e-4)
    # data gradient: plane (pi, pj) of dX is a stride-1 conv of dY with the taps of matching parity, stored at (2a+pi, 2b+pj)
    dy = torch.randn(B, Ho, Wo, Cout)
    dx = torch.zeros(B, H, W, Cin)
    wt = w.permute(1, 2, 0, 3).reshape(k * k, Cout, Cin)                  # per tap: [Cout][Cin]
    for pi in range(2):
        for pj in range(2):
            taps = [(fy, fx) for fy in range(k) for fx in range(k) if (pi + p - fy) % 2 == 0 and (pj + p - fx) % 2 == 0]
            if not taps:
                continue
            w_plane = torch.cat([wt[fy * k + fx].t() for fy, fx in taps], dim=1)          # [Cin][ntaps * Cout] == K-major "filter" of this conv
            plane = _simulate_conv_kernel_indexing(dy, w_plane, B, H // 2, W // 2, Cin, [(pi + p - fy) // 2 for fy, _ in taps],
                                                   [(pj + p - fx) // 2 for _, fx in taps], 1, 2, pi, pj)
            m = ~torch.isnan(plane)
            dx[m] = plane[m]
    xn = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
    F.conv2d(xn, w.permute(0, 3, 1, 2), None, 2, p).backward(dy.permute(0, 3, 1, 2))
    torch.testing.assert_close(dx, xn.grad.permute(0, 2, 3, 1), rtol=1e-4, atol=1e-4)


def test_halo_kernel_predicate(monkeypatch):
    """ops/nn.py:_halo_ok -- which 3x3 / stride-1 / 64-channel convs go to the halo-reuse kernel: valid / same / full padding, any size whose
    16 x 8 tiling is at least half real output, whole tiles only when the epilogue also takes BatchNorm statistics."""
    ok = nn._halo_ok
    assert ok(3, 1, 1, 64, 32, 32) and ok(3, 1, 1, 64, 32, 32, True)                 # ResNet layer 1 / VGG
    assert ok(3, 1, 0, 64, 26, 26) and ok(3, 1, 2, 64, 24, 24)                      # CNN_MNIST conv2 (channel-padded) and its data gradient
    assert ok(3, 1, 0, 64, 15, 15) and not ok(3, 1, 0, 64, 15, 15, True)            # CNN_CIFAR conv2: partial tiles, so no statistics
    assert not ok(3, 1, 0, 64, 6, 6)                                                # 4 x 4 output: 16 of 128 tile pixels -> generic kernel
    assert not ok(3, 2, 1, 64, 32, 32) and not ok(1, 1, 0, 64, 32, 32) and not ok(3, 1, 1, 128, 16, 16) and not ok(3, 1, 3, 64, 8, 8)
    for h in range(3, 40):                                                          # the utilisation rule, against its definition
        for pad in (0, 1, 2):
            ho = h + 2 * pad - 2
            tiles = -(-ho // 16) * 16 * (-(-ho // 8) * 8)
            assert ok(3, 1, pad, 64, h, h) == (ho >= 1 and 2 * ho * ho >= tiles), (h, pad)
    monkeypatch.setattr(nn, "USE_HALO_ANY", False)                                  # round-1 predicate
    assert ok(3, 1, 1, 64, 32, 32) and not ok(3, 1, 0, 64, 26, 26) and not ok(3, 1, 1, 64, 24, 24)
