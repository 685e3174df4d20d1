"""GPU tests of the conv tile rule (pick_conv_tile in gemm.cu): a deep conv whose 128-wide grid fills one wave of the SMs runs that
tile at one CTA per SM with a six-stage operand ring instead of the 64-wide tile.  Every output element is still the same k-blocks in
the same order through the same k16 MMA steps, so the launch must be bit-identical to the three-CTA 64-wide tiles that
``set_conv_one_wave(False)`` forces."""
import pytest
import torch

import rlr_b200  # noqa: F401
from rlr_b200 import ops

pytestmark = [pytest.mark.gpu]
DEV = "cuda:0"
BF = torch.bfloat16

CASES = [  # B, H, Cin, Cout, k, stride, pad
    (256, 8, 256, 256, 3, 1, 1), (256, 16, 128, 256, 3, 2, 1), (256, 16, 128, 256, 1, 2, 0),      # layer 3 of ResNet-18 at batch 256
    (256, 4, 512, 512, 3, 1, 1), (256, 8, 256, 512, 3, 2, 1), (256, 8, 256, 512, 1, 2, 0),        # layer 4
    (250, 4, 512, 512, 3, 1, 1),                                                                  # last m-tile three quarters masked
    (256, 4, 512, 576, 3, 1, 1),                                                                  # Cout no multiple of the tile
]


def _run(B, H, Cin, Cout, k, s, p, tma_store=True):
    torch.manual_seed(B + H + Cin + Cout + k)
    x = torch.randn(B, H, H, Cin, device=DEV).to(BF)
    w = (torch.randn(Cout, k, k, Cin, device=DEV) / (k * k * Cin) ** 0.5).to(BF)
    bias = torch.randn(Cout, device=DEV) * 0.1
    Ho = (H + 2 * p - k) // s + 1
    dy = torch.randn(B, Ho, Ho, Cout, device=DEV).to(BF)
    base = torch.randn(B, H, H, Cin, device=DEV).to(BF)
    ext, outs = ops.ext(), {}
    try:
        ext.set_conv_tma_store(tma_store)
        for on in (False, True):
            ext.set_conv_one_wave(on)
            tag = ("tiles-test", on, B, H, Cin, k, s)
            y0 = torch.full((B, Ho, Ho, Cout), 7.0, device=DEV, dtype=BF)
            y1 = torch.full_like(y0, 7.0)
            stats = torch.zeros(ext.STAT_SLOTS, 2, Cout, device=DEV)
            ops.conv2d_fwd_sm100(x, w, bias, y0, s, p, True, None, tag=tag)
            ops.conv2d_fwd_sm100(x, w, None, y1, s, p, False, stats, tag=tag)
            dx0, dx1 = torch.full_like(base, 3.0), base.clone()
            ops.conv2d_dgrad_sm100(dy, w, dx0, s, p, False)
            ops.conv2d_dgrad_sm100(dy, w, dx1, s, p, True)
            torch.cuda.synchronize()
            outs[on] = (y0, y1, dx0, dx1, stats.sum(0))
    finally:
        ext.set_conv_one_wave(True)
        ext.set_conv_tma_store(True)
    return outs, y1


@pytest.mark.parametrize("B,H,Cin,Cout,k,s,p", CASES)
def test_one_wave_tiles_match_previous_tiles(B, H, Cin, Cout, k, s, p):
    """Forward (bias + ReLU; plain with statistics) and data gradient on the MN-major filter (overwrite, accumulate)."""
    outs, y = _run(B, H, Cin, Cout, k, s, p)
    for name, a, b in zip(("fwd", "fwd+stats", "dgrad", "dgrad+acc"), outs[False], outs[True]):
        assert torch.equal(a, b), name
    # the statistics are column sums of the tiles met by atomics: same sums, but their order (and so the rounding) is not fixed
    yf = y.float().reshape(-1, Cout)
    ref = torch.stack([yf.sum(0), (yf * yf).sum(0)])
    for on in (False, True):
        assert torch.allclose(outs[on][4], ref, rtol=1e-4, atol=5e-2), on


def test_one_wave_tiles_match_without_tma_stores():
    """The coalesced-store epilogue of the one-wave tiles; statistics then need the two-CTA statistics kernel, whatever the rule says."""
    outs, _ = _run(256, 4, 512, 512, 3, 1, 1, tma_store=False)
    for name, a, b in zip(("fwd", "fwd+stats", "dgrad", "dgrad+acc"), outs[False], outs[True]):
        assert torch.equal(a, b), name
    assert torch.allclose(outs[False][4], outs[True][4], rtol=1e-4, atol=5e-2)


def test_rule_launches_one_wave_kernels_at_batch_256():
    """On a device where 128 CTAs are one wave over at least 0.9 of the SMs (H100: 132), the 512-filter 3x3 layers at batch 256 run
    the one-wave instantiation, forward and data gradient; the same layers at batch 512 (two waves) and the 256-filter layers keep the
    two-CTA kernel."""
    from torch.profiler import ProfilerActivity, profile
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if not (128 <= sms and 9 * sms <= 10 * 128):
        pytest.skip(f"128 CTAs are not one wave on {sms} SMs")

    def kernels(B, H, C):
        x = torch.randn(B, H, H, C, device=DEV).to(BF)
        w = (torch.randn(C, 3, 3, C, device=DEV) / (9 * C) ** 0.5).to(BF)
        y, dx = torch.empty_like(x), torch.empty_like(x)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ops.conv2d_fwd_sm100(x, w, None, y, 1, 1, False, None, tag=("tiles-rule", B, H, C))
            ops.conv2d_dgrad_sm100(y, w, dx, 1, 1, False)
            torch.cuda.synchronize()
        return [e.key for e in prof.key_averages() if "umma_conv_gemm_kernel" in e.key]

    for B, H, C, want in ((256, 4, 512, ("<128, false, false, 1>", "<128, false, true, 1>")),
                          (512, 4, 512, ("<128, false, false, 2>", "<128, false, true, 2>")),
                          (256, 8, 256, ("<128, false, false, 2>", "<128, false, true, 2>"))):
        names = kernels(B, H, C)
        for inst in want:
            assert any(inst in n for n in names), (B, H, C, inst, names)
