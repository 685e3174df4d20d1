"""The streaming BatchNorm passes (norm.cu bn_apply_kernel / bn_bwd_apply_kernel / channel_reduce_kernel) and the narrow fixed-order
sum of their per-CTA partials (common.cuh ordered_sum_narrow_kernel), at the shapes of a ResNet-18 training step and at the edges of
their launch geometry.

- forward (training and evaluation) and backward against the fp32 aten twin of the same op (``impl="aten"``), at every ResNet-18
  BatchNorm shape (batch 256, C = 64 ... 512) in each of its modes: shortcut BN (no ReLU), ``bn1`` (ReLU, mask recomputed from x
  or read from y) and ``bn2`` (residual + ReLU), plus the ragged last batch of an epoch (80 images), odd row counts and the
  smallest / largest channel counts the kernels take (8, 2048);
- two runs give bit-identical outputs;
- the narrow ordered sum equals part-by-part sequential addition bit for bit at the BatchNorm partial counts.
"""
import pytest
import torch

import rlr_b200  # noqa: F401
from rlr_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16

# (relu, residual, recompute): shortcut BN | bn1 with the mask recomputed from x | bn1 reading y | bn2 (residual + ReLU)
MODES = [(False, False, False), (True, False, True), (True, False, False), (True, True, False)]
RESNET18_SHAPES = [(256, 32, 64), (256, 16, 128), (256, 8, 256), (256, 4, 512)]


def _inputs(M, C, res, seed):
    g = torch.Generator(DEV).manual_seed(seed)
    x = (torch.randn(M, C, device=DEV, generator=g) * 2 + 0.5).to(BF)
    r = torch.randn(M, C, device=DEV, generator=g).to(BF) if res else None
    gamma = torch.rand(C, device=DEV, generator=g) + 0.5
    beta = torch.randn(C, device=DEV, generator=g) * 0.1
    dy = torch.randn(M, C, device=DEV, generator=g).to(BF)
    return x, r, gamma, beta, dy


def _run(impl, M, C, relu, res, recompute, seed, fwd=None):
    """Forward (training, then evaluation) and backward of one BatchNorm.  ``fwd``: the (y, mean_rstd) the backward consumes instead
    of this run's own, so that two back-ends are compared on the same ReLU mask (an output that rounds to zero in one and not in the
    other would otherwise flip a whole gradient element)."""
    x, r, gamma, beta, dy = _inputs(M, C, res, seed)
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    y, mr = torch.empty_like(x), torch.zeros(2, C, device=DEV)
    ops.bn_fwd(x, y, r, gamma, beta, rm, rv, None, mr, M, 1e-5, 0.1, True, relu, impl)
    yb, mrb = fwd if fwd is not None else (y, mr)
    dx, dres = torch.empty_like(x), (torch.empty_like(x) if res else None)
    dg, db, ds = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.zeros(1, 2, C, device=DEV)
    ops.bn_bwd(dy, yb, x, gamma, mrb, ds, dx, dres, dg, db, relu, impl, beta=beta if recompute else None)
    ye = torch.empty_like(x)
    ops.bn_fwd(x, ye, r, gamma, beta, rm, rv, None, torch.zeros(2, C, device=DEV), M, 1e-5, 0.1, False, relu, impl)
    torch.cuda.synchronize()
    return dict(y=y, mr=mr, rm=rm, rv=rv, dx=dx, dres=dres, dg=dg, db=db, ye=ye)


def _check_against_aten(M, C, relu, res, recompute, seed=0):
    got = _run("sm100", M, C, relu, res, recompute, seed)
    want = _run("aten", M, C, relu, res, recompute, seed, fwd=(got["y"], got["mr"]))
    for k, w in want.items():
        if w is None:
            continue
        g, w = got[k].float(), w.float()
        scale = w.abs().max().clamp_min(1e-6)
        err = (g - w).abs().max() / scale
        rms = (g - w).norm() / w.norm().clamp_min(1e-12)
        # bf16 outputs differ by a rounding step where the fp32 statistics differ in their last bits (summation order)
        assert err < 2e-2 and rms < 4e-3, (k, M, C, relu, res, recompute, float(err), float(rms))


@pytest.mark.parametrize("B,H,C", RESNET18_SHAPES)
@pytest.mark.parametrize("relu,res,recompute", MODES)
def test_bn_resnet18_shapes_match_aten(B, H, C, relu, res, recompute):
    _check_against_aten(B * H * H, C, relu, res, recompute)


@pytest.mark.parametrize("H,C", [(32, 64), (16, 128), (8, 256), (4, 512)])
@pytest.mark.parametrize("relu,res,recompute", [MODES[1], MODES[3]])
def test_bn_ragged_last_batch(H, C, relu, res, recompute):
    _check_against_aten(80 * H * H, C, relu, res, recompute)


@pytest.mark.parametrize("M,C", [(777, 8), (12345, 8), (4099, 64), (131, 512), (1001, 2048), (33, 2048), (3, 256)])
@pytest.mark.parametrize("relu,res,recompute", [MODES[0], MODES[1], MODES[3]])
def test_bn_odd_rows_and_edge_channels(M, C, relu, res, recompute):
    _check_against_aten(M, C, relu, res, recompute, seed=M)


@pytest.mark.parametrize("M,C", [(256 * 32 * 32, 64), (256 * 4 * 4, 512), (1001, 2048)])
@pytest.mark.parametrize("relu,res,recompute", [MODES[1], MODES[2], MODES[3]])
def test_bn_bitwise_reproducible(M, C, relu, res, recompute):
    a = _run("sm100", M, C, relu, res, recompute, seed=7)
    b = _run("sm100", M, C, relu, res, recompute, seed=7)
    for k, v in a.items():
        if v is not None:
            assert torch.equal(v, b[k]), k


@pytest.mark.parametrize("nparts", [264, 528, 300, 16, 100])
@pytest.mark.parametrize("n", [128, 256, 512, 1024, 100, 2048])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_narrow_ordered_sum_adds_in_part_order(nparts, n, dtype):
    torch.manual_seed(nparts * 7 + n)
    # magnitudes spread over several decades so that any other association order changes the rounding
    part = (torch.randn(nparts, n, device=DEV, dtype=torch.float64) * torch.logspace(-3, 3, nparts, device=DEV,
                                                                                    dtype=torch.float64)[:, None]).to(dtype)
    out = torch.randn(n, device=DEV, dtype=dtype)
    s = part[0].clone()
    for j in range(1, nparts):
        s = s + part[j]
    want = out + s
    ops.ext().ordered_sum(out, part)
    torch.cuda.synchronize()
    assert torch.equal(out, want)
