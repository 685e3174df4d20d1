"""The fp64 checker of tests/gemm_oracle.py is sharp: it accepts a correct emulation of every kernel family the GPU oracle test
(tests/test_gpu_gemm_oracle.py) judges -- fp32 accumulation, the stated epilogue, round-to-nearest bf16 -- and rejects each of the
mutants M1-M10, small faults of the kind a kernel change introduces (a dropped k-block, a missing or unflipped tap, a wrong rounding
mode, statistics of the wrong values, a guard element written).  Runs on the CPU."""
import math

import pytest
import torch
import torch.nn.functional as F

import gemm_oracle as go

BF = torch.bfloat16


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(BF)


def _conv32(x, w, stride, pad):
    """fp32 accumulation of the forward convolution (NHWC)."""
    return F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), None, stride, pad).permute(0, 2, 3, 1)


def _dgrad32(dy, w, x_shape, stride, pad):
    B, H, W, Cin = x_shape
    return torch.ops.aten.convolution_backward(dy.float().permute(0, 3, 1, 2), torch.zeros(B, Cin, H, W), w.float().permute(0, 3, 1, 2),
                                               None, [stride, stride], [pad, pad], [1, 1], False, [0, 0], 1,
                                               [True, False, False])[0].permute(0, 2, 3, 1)


def _trunc_bf16(t):
    """bf16 pack by truncation (round toward zero) instead of round-to-nearest: mutant M5."""
    return (t.float().contiguous().view(torch.int32) & -65536).view(torch.float32)


# ---- forward convolutions: the shape families of the GPU test (batch cut down; reduction depth, tile tails and borders kept) ----
FWD = {  # name: B, H, W, Cin, Cout, k, stride, pad
    "l1-3x3": (2, 32, 32, 64, 64, 3, 1, 1),
    "l4-3x3-K4608": (4, 4, 4, 512, 512, 3, 1, 1),
    "s2-3x3": (4, 16, 16, 64, 128, 3, 2, 1),
    "s2-1x1": (4, 16, 16, 64, 128, 1, 2, 0),
    "stem-3ch": (4, 32, 32, 3, 64, 3, 1, 1),
    "valid-3x3": (4, 26, 26, 32, 64, 3, 1, 0),
    "cout200": (4, 8, 8, 64, 200, 3, 1, 1),
}


def _fwd_case(name, seed=0):
    B, H, W, Cin, Cout, k, s, p = FWD[name]
    x = _rand((B, H, W, Cin), seed)
    w = _rand((Cout, k, k, Cin), seed + 1, 1 / math.sqrt(k * k * Cin))
    bias = torch.randn(Cout, generator=torch.Generator().manual_seed(seed + 2)) * 0.1
    return x, w, bias, s, p


def _emulate_fwd(x, w, bias, s, p):
    acc = _conv32(x, w, s, p)
    return acc, go.rn_bf16((acc + bias).clamp_min(0)).to(BF)


@pytest.mark.parametrize("name", list(FWD))
def test_correct_forward_emulation_is_accepted(name):
    x, w, bias, s, p = _fwd_case(name)
    _, y = _emulate_fwd(x, w, bias, s, p)
    st = go.conv_statement(x, w, s, p)
    r = go.check(name, y, st, go.epi_store(bias, True))
    print(r)
    assert r.ok, r
    stats = torch.stack([y.float().reshape(-1, y.shape[-1]).sum(0), (y.float() ** 2).reshape(-1, y.shape[-1]).sum(0)])
    rs = go.check_stats(name, stats, y)
    assert rs.ok, rs


DGRAD = {  # name: B, H, W, Cin, Cout, k, stride, pad
    "s1-3x3": (4, 16, 16, 64, 128, 3, 1, 1),
    "s1-3x3-K4608": (4, 4, 4, 512, 512, 3, 1, 1),
    "s2-3x3": (4, 16, 16, 64, 128, 3, 2, 1),
    "s2-1x1": (4, 16, 16, 64, 128, 1, 2, 0),
    "full-3x3": (4, 15, 15, 64, 64, 3, 1, 0),
}


def _dgrad_case(name, seed=10):
    B, H, W, Cin, Cout, k, s, p = DGRAD[name]
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy = _rand((B, Ho, Wo, Cout), seed)
    w = _rand((Cout, k, k, Cin), seed + 1, 1 / math.sqrt(k * k * Cout))
    old = _rand((B, H, W, Cin), seed + 2)
    return dy, w, old, (B, H, W, Cin), s, p


@pytest.mark.parametrize("name", list(DGRAD))
def test_correct_dgrad_emulation_is_accepted(name):
    dy, w, old, xs, s, p = _dgrad_case(name)
    acc = _dgrad32(dy, w, xs, s, p)
    st = go.dgrad_statement(dy, w, xs, s, p)
    r = go.check(name, go.rn_bf16(acc).to(BF), st, go.epi_store())
    assert r.ok, r
    r = go.check(name + "+acc", go.rn_bf16(go.rn_bf16(acc) + old.float()).to(BF), st, go.epi_acc_twice(old))
    print(r)
    assert r.ok, r


GEMM = {  # name: M, N, K, output dtype -- the fp32 families are the weight gradients (K = batch x output pixels)
    "fc1-splitk-K9216": (256, 128, 9216, BF),
    "l4-fwd-K4608": (256, 64, 4608, BF),
    "tail-M129": (129, 64, 128, BF),
    "wgrad-l1-K262144": (128, 16, 256 * 32 * 32, torch.float32),
    "wgrad-l4-K4096": (512, 64, 256 * 4 * 4, torch.float32),
    "linear-wgrad-K256": (128, 512, 256, torch.float32),
}


def _gemm_case(name, seed=20):
    M, N, K, dt = GEMM[name]
    a = _rand((M, K), seed)
    b = _rand((N, K), seed + 1, 1 / math.sqrt(K) if dt == BF else 1.0)
    return a, b, dt


@pytest.mark.parametrize("name", list(GEMM))
def test_correct_gemm_emulation_is_accepted(name):
    a, b, dt = _gemm_case(name)
    acc = a.float() @ b.float().t()
    st = go.gemm_statement(a, b)
    if dt == BF:
        bias = torch.randn(b.shape[0]) * 0.1
        r = go.check(name, go.rn_bf16((acc + bias).clamp_min(0)).to(BF), st, go.epi_store(bias, True))
    else:
        old = torch.randn(acc.shape)
        r = go.check(name, acc + old, go.plus_old(st, old), go.epi_f32)
    print(r)
    assert r.ok, r


def test_correct_head_emulation_is_accepted():
    """CUDA-core head kernels: N <= 32 outputs, data gradient added to the old value in fp32 and rounded once."""
    x, w, dy = _rand((256, 512), 30), _rand((10, 512), 31, 0.05), _rand((256, 10), 32)
    bias = torch.randn(10) * 0.1
    r = go.check("head-fwd", go.rn_bf16(x.float() @ w.float().t() + bias).to(BF), go.gemm_statement(x, w), go.epi_store(bias))
    assert r.ok, r
    old = _rand((256, 512), 33)
    dx = go.rn_bf16(dy.float() @ w.float() + old.float()).to(BF)
    r = go.check("head-dx+acc", dx, go.gemm_statement(dy, w.t()), go.epi_acc_once(old))
    assert r.ok, r


# =====================================================================================================================
# mutants
# =====================================================================================================================
def _rejected(r):
    print("rejected" if not r.ok else "ACCEPTED", r)
    return not r.ok


@pytest.mark.parametrize("name", ["l4-fwd-K4608", "wgrad-l1-K262144"])
def test_m1_dropped_k_block_is_rejected(name):
    """M1: one 64-deep k-block of one 128-row tile missing from the accumulator (layer-4 forward depth K = 4608, layer-1 weight
    gradient depth K = 256 x 32 x 32)."""
    a, b, dt = _gemm_case(name)
    acc = a.float() @ b.float().t()
    kb = a.shape[1] // 64 // 2 * 64
    acc[:128] -= a[:128, kb:kb + 64].float() @ b[:, kb:kb + 64].float().t()
    st = go.gemm_statement(a, b)
    out = go.rn_bf16(acc).to(BF) if dt == BF else acc
    assert _rejected(go.check(name, out, st, go.epi_store() if dt == BF else go.epi_f32))


def test_m2_tap_missing_at_border_pixels_is_rejected():
    """M2: the centre tap of a 3x3 'same' convolution dropped at the image-border pixels only."""
    x, w, bias, s, p = _fwd_case("l1-3x3")
    acc = _conv32(x, w, s, p)
    centre = _conv32(x, w[:, 1:2, 1:2, :], 1, 0)
    border = torch.ones(acc.shape[1], acc.shape[2], dtype=torch.bool)
    border[1:-1, 1:-1] = False
    acc = torch.where(border[None, :, :, None], acc - centre, acc)
    y = go.rn_bf16((acc + bias).clamp_min(0)).to(BF)
    assert _rejected(go.check("M2", y, go.conv_statement(x, w, s, p), go.epi_store(bias, True)))


@pytest.mark.parametrize("name", ["s1-3x3", "s2-3x3"])
def test_m3_unflipped_dgrad_taps_are_rejected(name):
    """M3: two taps of the data gradient's filter used without the flip (tap (0,0) where (2,2) belongs and back)."""
    dy, w, old, xs, s, p = _dgrad_case(name)
    wm = w.clone()
    wm[:, 0, 0], wm[:, 2, 2] = w[:, 2, 2], w[:, 0, 0]
    acc = _dgrad32(dy, wm, xs, s, p)
    assert _rejected(go.check("M3", go.rn_bf16(acc).to(BF), go.dgrad_statement(dy, w, xs, s, p), go.epi_store()))


@pytest.mark.parametrize("what", ["bias", "relu"])
def test_m4_epilogue_missing_on_last_partial_channel_tile_is_rejected(what):
    """M4: bias or ReLU not applied to channels 128..199 of a 200-filter convolution (the last, partial 128-wide channel tile)."""
    x, w, bias, s, p = _fwd_case("cout200")
    acc = _conv32(x, w, s, p)
    good = (acc + bias).clamp_min(0)
    bad = acc.clamp_min(0) if what == "bias" else acc + bias
    y = torch.cat([good[..., :128], bad[..., 128:]], -1)
    assert _rejected(go.check("M4-" + what, go.rn_bf16(y).to(BF), go.conv_statement(x, w, s, p), go.epi_store(bias, True)))


@pytest.mark.parametrize("name", ["l1-3x3", "l4-3x3-K4608", "stem-3ch"])
def test_m5_truncating_bf16_pack_is_rejected(name):
    """M5: the bf16 pack truncates instead of rounding to nearest."""
    x, w, bias, s, p = _fwd_case(name)
    acc = _conv32(x, w, s, p)
    y = _trunc_bf16((acc + bias).clamp_min(0)).to(BF)
    r = go.check("M5", y, go.conv_statement(x, w, s, p), go.epi_store(bias, True))
    assert _rejected(r) and r.mismatch > go.RHO


@pytest.mark.parametrize("name", ["s1-3x3", "s1-3x3-K4608", "s2-3x3"])
def test_m6_single_rounding_where_the_path_rounds_twice_is_rejected(name):
    """M6a: an accumulating conv epilogue that adds the old value to the fp32 accumulator and rounds once."""
    dy, w, old, xs, s, p = _dgrad_case(name)
    acc = _dgrad32(dy, w, xs, s, p)
    out = go.rn_bf16(acc + old.float()).to(BF)
    assert _rejected(go.check("M6a", out, go.dgrad_statement(dy, w, xs, s, p), go.epi_acc_twice(old)))


def test_m6_double_rounding_where_the_head_rounds_once_is_rejected():
    """M6b: the head kernel's accumulating data gradient packed to bf16 before the old value is added."""
    dy, w, old = _rand((256, 10), 32), _rand((10, 512), 31, 0.05), _rand((256, 512), 33)
    acc = dy.float() @ w.float()
    out = go.rn_bf16(go.rn_bf16(acc) + old.float()).to(BF)
    assert _rejected(go.check("M6b", out, go.gemm_statement(dy, w.t()), go.epi_acc_once(old)))


def test_m7_statistics_of_fp32_values_are_rejected():
    """M7: BatchNorm statistics summed from the fp32 epilogue values instead of the stored bf16 ones, at M = 4 x 16 x 16 = 1024 rows
    (the stride-2 family).  Not caught at M = 256 x 32 x 32 (ResNet layer 1 at batch 256): the bf16 rounding errors of M outputs
    sum to about 2^-9 sqrt(M/3) rms(y) = 0.6 rms(y) there, below the fp32 summation bound KAPPA_STATS 2^-24 sqrt(M) sum|y| = 6 mean(y)."""
    x, w, bias, s, p = _fwd_case("s2-3x3")
    acc, y = _emulate_fwd(x, w, bias, s, p)
    yf = (acc + bias).clamp_min(0).double().reshape(-1, y.shape[-1])
    stats = torch.stack([yf.sum(0), (yf * yf).sum(0)])
    assert _rejected(go.check_stats("M7", stats, y))


def test_m8_masked_tail_row_filled_from_neighbouring_image_is_rejected():
    """M8: the padding row below each image read from the next image's first row instead of as zeros (the implicit GEMM packs the
    pixels of several images into one 128-row tile; an unmasked tail row reads its neighbour)."""
    x, w, bias, s, p = _fwd_case("l1-3x3")
    acc = _conv32(x, w, s, p)
    B, H = x.shape[0], x.shape[1]
    for b in range(B - 1):   # output row H-1, filter row 2 reads input row H: row 0 of image b + 1
        nxt = F.conv2d(x[b + 1:b + 2, 0:1].float().permute(0, 3, 1, 2), w[:, 2:3].float().permute(0, 3, 1, 2), None, 1, (0, 1))
        acc[b, H - 1] += nxt.permute(0, 2, 3, 1)[0, 0]
    y = go.rn_bf16((acc + bias).clamp_min(0)).to(BF)
    assert _rejected(go.check("M8", y, go.conv_statement(x, w, s, p), go.epi_store(bias, True)))


@pytest.mark.parametrize("name", ["wgrad-l1-K262144", "wgrad-l4-K4096"])
def test_m9_wgrad_split_added_twice_is_rejected(name):
    """M9: one split of a split-K weight gradient added twice (a quarter of the reduction, or one 64-deep k-block)."""
    a, b, _ = _gemm_case(name)
    acc = a.float() @ b.float().t()
    lo = a.shape[1] // 4
    for hi in (2 * lo, lo + 64):
        out = acc + a[:, lo:hi].float() @ b[:, lo:hi].float().t()
        assert _rejected(go.check("M9", out, go.gemm_statement(a, b), go.epi_f32))


def test_m10_guard_element_written_is_rejected():
    """M10: a store one element past the output."""
    for dt in (BF, torch.float32):
        y, buf = go.guarded((3, 5, 8), dt, "cpu")
        y.zero_()
        assert go.guard_intact(buf)
        buf[y.numel()] = 0
        assert not go.guard_intact(buf)
        y, buf = go.guarded((3, 5, 8), dt, "cpu")
        buf[-1] = 1.0
        assert not go.guard_intact(buf)


def test_unwritten_and_untapped_elements():
    """An element left at its NaN prefill fails; an element no tap reaches (sq == 0) must be phi(0) exactly."""
    a, b = _rand((8, 64), 1), _rand((16, 64), 2)
    a[3] = 0
    st = go.gemm_statement(a, b)
    out = go.rn_bf16(a.float() @ b.float().t()).to(BF)
    assert go.check("ok", out, st, go.epi_store()).ok
    bad = out.clone()
    bad[3, 5] = torch.finfo(BF).tiny
    assert not go.check("untapped", bad, st, go.epi_store()).ok
    bad = out.clone()
    bad[0, 0] = float("nan")
    r = go.check("nan", bad, st, go.epi_store())
    assert not r.ok and r.kappa == math.inf
