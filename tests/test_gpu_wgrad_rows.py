"""GPU tests of the filter-row weight-gradient kernel (umma_wgrad_rows_kernel in wgrad.cu): one CTA computes all nine taps of a
64 x 64 filter tile from one dY box and one input halo per k-block.  It keeps the pixel order, the k16 steps, the k-block order
and the split count of umma_wgrad_kernel<64, 3> on whole-row tiles, so its gradient must be bit-identical to the one
``set_wgrad_rows(False)`` forces.  64-channel inputs on 16 x 8 tiles (ResNet-18 layer 1) keep umma_wgrad_halo_kernel either way."""
import pytest
import torch

import rlr_b200  # noqa: F401
from rlr_b200 import ops

pytestmark = [pytest.mark.gpu]
DEV = "cuda:0"
BF = torch.bfloat16

CASES = [  # B, H, W, Cin, Cout
    (256, 32, 32, 64, 64), (80, 32, 32, 64, 64),          # ResNet-18 layer 1 (halo kernel); 80 = the last batch of 50,000 / 256
    (256, 16, 16, 128, 128), (80, 16, 16, 128, 128),      # layer 2 (whole rows, 16 x 4)
    (256, 8, 8, 256, 256), (80, 8, 8, 256, 256),          # layer 3 (whole rows, 8 x 8)
    (128, 16, 16, 64, 128),                               # VGG, 64-channel input (halo kernel)
    (128, 8, 8, 128, 256), (64, 16, 16, 128, 128),        # VGG, whole rows
    (32, 16, 16, 128, 64),                                # whole rows, Cout of one 64-filter tile
    (16, 32, 32, 128, 128), (4, 64, 64, 128, 64),         # whole rows 32 x 2 and 64 x 1
    (1, 8, 8, 256, 256), (1, 8, 8, 128, 64),              # a split count of 1, added straight into the gradient
]


def _inputs(B, H, W, Cin, Cout):
    torch.manual_seed(B + H + W + Cin + Cout)
    x = torch.randn(B, H, W, Cin, device=DEV).to(BF)
    dy = torch.randn(B, H, W, Cout, device=DEV).to(BF)
    base = torch.randn(Cout, 3, 3, Cin, device=DEV)
    return x, dy, base


def _wgrad(x, dy, base, rows, k=3, s=1, p=1):
    ext = ops.ext()
    try:
        ext.set_wgrad_rows(rows)
        gw = base.clone()
        ops.conv2d_wgrad_sm100(x, dy, gw, None, s, p, tag=("wgrad-rows-test", rows, k, s), zero=False)
        torch.cuda.synchronize()
    finally:
        ext.set_wgrad_rows(True)
    return gw


def _launches(fn):
    """Launches of (umma_wgrad_kernel, umma_wgrad_halo_kernel, umma_wgrad_rows_kernel) made by ``fn``, from the launchers' counts."""
    before = ops.ext().wgrad_launch_counts()
    fn()
    torch.cuda.synchronize()
    return tuple(a - b for a, b in zip(ops.ext().wgrad_launch_counts(), before))


@pytest.mark.parametrize("B,H,W,Cin,Cout", CASES)
def test_rows_kernel_matches_previous_kernels(B, H, W, Cin, Cout):
    x, dy, base = _inputs(B, H, W, Cin, Cout)
    old = _wgrad(x, dy, base, False)
    new = _wgrad(x, dy, base, True)
    assert not torch.equal(new, base)
    assert torch.equal(old, new)


def test_rows_kernel_against_fp64():
    B, H, W, Cin, Cout = 80, 16, 16, 128, 128
    x, dy, _ = _inputs(B, H, W, Cin, Cout)
    gw = _wgrad(x, dy, torch.zeros(Cout, 3, 3, Cin, device=DEV), True)
    ref = torch.nn.grad.conv2d_weight(x.double().permute(0, 3, 1, 2), (Cout, Cin, 3, 3), dy.double().permute(0, 3, 1, 2), 1, 1)
    ref = ref.permute(0, 2, 3, 1)
    assert float((gw.double() - ref).abs().max() / (ref.abs().max() + 1e-6)) < 1e-2


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(64, 16, 16, 128, 128), (64, 8, 8, 256, 256)])
def test_eligible_shapes_launch_rows_kernel(B, H, W, Cin, Cout):
    x, dy, base = _inputs(B, H, W, Cin, Cout)
    assert _launches(lambda: _wgrad(x, dy, base, True)) == (0, 0, 1)
    assert _launches(lambda: _wgrad(x, dy, base, False)) == (1, 0, 0)


def test_layer1_keeps_halo_kernel():
    x, dy, base = _inputs(64, 32, 32, 64, 64)
    assert _launches(lambda: _wgrad(x, dy, base, True)) == (0, 1, 0)


@pytest.mark.parametrize("B,H,Cin,Cout,k,s,p", [
    (64, 16, 128, 256, 3, 2, 1),     # stride 2
    (64, 4, 512, 512, 3, 1, 1),      # layer 4: 4 x 4 output, tiles narrower than one 8-pixel core group
    (64, 8, 256, 256, 1, 1, 0),      # 1 x 1
])
def test_ineligible_shapes_keep_generic_kernel(B, H, Cin, Cout, k, s, p):
    torch.manual_seed(B + H + Cin)
    Ho = (H + 2 * p - k) // s + 1
    x = torch.randn(B, H, H, Cin, device=DEV).to(BF)
    w = (torch.randn(Cout, k, k, Cin, device=DEV) / (k * k * Cin) ** 0.5).to(BF)
    dy = torch.randn(B, Ho, Ho, Cout, device=DEV).to(BF)
    tag = ("wgrad-rows-ineligible", B, H, Cin, k, s)
    ops.conv2d_fwd_sm100(x, w, None, torch.empty(B, Ho, Ho, Cout, device=DEV, dtype=BF), s, p, False, None, tag=tag)
    gw = torch.zeros(Cout, k, k, Cin, device=DEV)
    assert _launches(lambda: ops.conv2d_wgrad_sm100(x, dy, gw, None, s, p, tag=tag)) == (1, 0, 0)
