"""The fp64 checker of tests/layer_oracle.py is sharp: it accepts a correct fp32 / bf16 emulation of every layer-kernel family the GPU
oracle test (tests/test_gpu_layer_oracle.py) judges, and rejects each mutant below -- small faults of the kind a kernel change
introduces (a biased running variance, eps in the wrong place, a dropped row, a mask keyed by the wrong index, ...).  Runs on the
CPU."""
import math

import numpy as np
import pytest
import torch

import layer_oracle as lo

BF = torch.bfloat16
EPS, MOM = 1e-5, 0.1


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ok(results):
    return all(r.ok for r in results)


# =====================================================================================================================
# BatchNorm
# =====================================================================================================================
def _bn_inputs(M, C, seed=0):
    g = _gen(seed)
    off = torch.linspace(-2, 2, C)                                 # channel means up to 2 std away from 0
    x = (torch.randn(M, C, generator=g) + off).to(BF)
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.2
    rm, rv = torch.randn(C, generator=g) * 0.1, torch.rand(C, generator=g) * 0.1
    res = torch.randn(M, C, generator=g).to(BF)
    return x, gamma, beta, rm, rv, res


def _emu_bn_fwd(x, gamma, beta, rm, rv, relu, res, mut=None):
    """fp32 emulation of channel_stats + bn_apply (training).  Returns (stats [1,2,C], mean_rstd, rm', rv', y)."""
    xf = x.float()
    xs = xf[:-1] if mut == "drop_last_row" else xf
    stats = torch.stack([xs.sum(0), (xs * xs).sum(0)])[None]
    M = float(x.shape[0])
    eps = torch.tensor(EPS, dtype=torch.float32)
    mom = torch.tensor(MOM, dtype=torch.float32)
    mean = stats[0, 0] / M
    var = (stats[0, 1] / M - mean * mean).clamp_min(0)
    rstd = var.rsqrt() + eps if mut == "eps_after_rsqrt" else (var + eps).rsqrt()
    rm1 = mom * rm + (1 - mom) * mean if mut == "momentum_swapped" else (1 - mom) * rm + mom * mean
    unb = var if (mut == "biased_running_var" or M <= 1) else var * M / (M - 1)
    rv1 = (1 - mom) * rv + mom * unb
    sc = gamma * rstd
    v = xf * sc + (beta - mean * sc)
    if res is not None:
        v = v + res.float()
    if relu:
        v = torch.where(xf > 0, v, torch.zeros_like(v)) if mut == "relu_mask_from_x" else v.clamp_min(0)
    return stats, torch.stack([mean, rstd]), rm1, rv1, lo.rn_bf16(v).to(BF)


def _judge_bn_fwd(x, gamma, beta, rm, rv, relu, res, out):
    stats, mean_rstd, rm1, rv1, y = out
    M = x.shape[0]
    r = [lo.check_stats("stats", stats, x)]
    d1, d2 = lo.stat_slots_bound(stats)
    r += lo.check_fin("own", lo.bn_finalize(stats[0, 0], stats[0, 1], M, EPS, MOM, rm, rv, d1, d2), mean_rstd, rm1, rv1)
    xd = x.double()
    tb = lo.KAPPA_STATS * lo.U * math.sqrt(M)
    truth = lo.bn_finalize(xd.sum(0), (xd * xd).sum(0), M, EPS, MOM, rm, rv, tb * xd.abs().sum(0), tb * (xd * xd).sum(0))
    r += lo.check_fin("truth", truth, mean_rstd, rm1, rv1)
    v, unit = lo.affine_statement(x, mean_rstd[0], mean_rstd[1], gamma, beta, res)
    r.append(lo.check_value("y", y, v, unit, lo.epi_relu(relu)))
    return r


@pytest.mark.parametrize("M,relu,resid", [(1000, True, False), (1000, True, True), (3, False, False), (1, True, False), (257, True, True)])
def test_bn_forward_emulation_accepted(M, relu, resid):
    x, gamma, beta, rm, rv, res = _bn_inputs(M, 16)
    res = res if resid else None
    r = _judge_bn_fwd(x, gamma, beta, rm, rv, relu, res, _emu_bn_fwd(x, gamma, beta, rm, rv, relu, res))
    assert _ok(r), [q for q in r if not q.ok]


@pytest.mark.parametrize("mut", ["biased_running_var", "eps_after_rsqrt", "momentum_swapped", "drop_last_row", "relu_mask_from_x"])
def test_bn_forward_mutant_rejected(mut):
    x, gamma, beta, rm, rv, _ = _bn_inputs(1000, 16)
    r = _judge_bn_fwd(x, gamma, beta, rm, rv, True, None, _emu_bn_fwd(x, gamma, beta, rm, rv, True, None, mut))
    assert not _ok(r)


def test_biased_running_variance_rejected_at_resnet_rows():
    """262,144 rows (ResNet-18 layer 1 at batch 256): the unbiased factor moves the running variance by 4e-6 relative; judged against
    the kernel's own stored sums the bound is a few ulps, so the biased variance is still seen."""
    M, C = 262144, 8
    x, gamma, beta, rm, rv, _ = _bn_inputs(M, C, 1)
    rv = torch.zeros(C)
    for mut, want in ((None, True), ("biased_running_var", False)):
        stats, mean_rstd, rm1, rv1, y = _emu_bn_fwd(x, gamma, beta, rm, rv, True, None, mut)
        d1, d2 = lo.stat_slots_bound(stats)
        r = lo.check_fin("own", lo.bn_finalize(stats[0, 0], stats[0, 1], M, EPS, MOM, rm, rv, d1, d2), mean_rstd, rm1, rv1)
        assert _ok(r) == want, (mut, r)


def _emu_bn_bwd(dy, y, x, gamma, mean_rstd, relu, mut=None):
    """fp32 emulation of bn_bwd: (dsum [1,2,C], dx, dres, dgamma, dbeta)."""
    dz = dy.float()
    if relu:
        dz = torch.where(y.float() > 0, dz, torch.zeros_like(dz))
    M = x.shape[0]
    xhat = (x.float() - mean_rstd[0]) * mean_rstd[1]
    dsum = torch.stack([dz.sum(0), (dz * xhat).sum(0)])[None]
    invM = torch.tensor(1.0 / M, dtype=torch.float32)
    k1, k2 = dsum[0, 0] * invM, dsum[0, 1] * invM
    dx = lo.rn_bf16(gamma * mean_rstd[1] * (dz - k1 - xhat * k2)).to(BF)
    dres = (dy if mut == "dres_unmasked" else dz.to(BF)).clone()
    return dsum, dx, dres, k2 * M, k1 * M


def _judge_bn_bwd(dy, y, x, gamma, mean_rstd, relu, out):
    dsum, dx, dres, dg, db = out
    mask = (y.double() > 0) if relu else torch.ones_like(x, dtype=torch.float64)
    terms, xhat = lo.bn_bwd_terms(dy, x, mask, mean_rstd)
    r = [lo.check_sums("dsum", dsum, terms, rounding=3)]
    wg, wb, ug, ub = lo.bn_param_grads(dsum)
    r += [lo.check_value("dgamma", dg, wg, ug), lo.check_value("dbeta", db, wb, ub)]
    v, unit = lo.bn_dx_statement(terms[0], xhat, gamma, mean_rstd, dsum)
    r.append(lo.check_value("dx", dx, v, unit, lo.rn_bf16))
    r.append(lo.Result("dres", 0, 0, (), torch.equal(dres, terms[0].to(BF))))
    return r


def _bn_bwd_case(M=1000, C=16):
    x, gamma, beta, rm, rv, _ = _bn_inputs(M, C, 3)
    _, mean_rstd, _, _, y = _emu_bn_fwd(x, gamma, beta, rm, rv, True, None)
    dy = torch.randn(M, C, generator=_gen(4)).to(BF)
    return dy, y, x, gamma, mean_rstd


def test_bn_backward_emulation_accepted():
    dy, y, x, gamma, mean_rstd = _bn_bwd_case()
    r = _judge_bn_bwd(dy, y, x, gamma, mean_rstd, True, _emu_bn_bwd(dy, y, x, gamma, mean_rstd, True))
    assert _ok(r), [q for q in r if not q.ok]


def test_bn_backward_dres_unmasked_rejected():
    dy, y, x, gamma, mean_rstd = _bn_bwd_case()
    assert not _ok(_judge_bn_bwd(dy, y, x, gamma, mean_rstd, True, _emu_bn_bwd(dy, y, x, gamma, mean_rstd, True, "dres_unmasked")))


# =====================================================================================================================
# GroupNorm
# =====================================================================================================================
def _gn_case(B=3, H=5, W=4, C=64, G=32, seed=5):
    g = _gen(seed)
    x = (torch.randn(B, H, W, C, generator=g) * 1.5 + torch.linspace(-1, 1, C)).to(BF)
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.2
    dy = torch.randn(B, H, W, C, generator=g).to(BF)
    old = torch.randn(2, C, generator=g)
    return x, gamma, beta, dy, old, G


def _emu_gn_fwd(x, gamma, beta, G, mut=None):
    B, H, W, C = x.shape
    Gs = C // 8 if mut == "groups_of_8" else G
    xg = x.float().reshape(B, H * W, Gs, C // Gs)
    mean = xg.sum((1, 3)) / (H * W * (C // Gs))
    var = ((xg - mean[:, None, :, None]) ** 2).sum((1, 3)) / (H * W * (C // Gs))
    rstd = (var + EPS).rsqrt()
    m = mean.repeat_interleave(C // Gs, 1).reshape(B, 1, 1, C)
    r = rstd.repeat_interleave(C // Gs, 1).reshape(B, 1, 1, C)
    sc = r * gamma
    y = lo.rn_bf16((x.float() * sc + (beta - m * sc)).clamp_min(0)).to(BF)
    if mut == "groups_of_8":     # G groups are still stored: each one the statistics of its first channel's 8-channel block
        mean, rstd = m.reshape(B, C)[:, ::C // G], r.reshape(B, C)[:, ::C // G]
    return torch.stack([mean, rstd], 1), y


def _judge_gn_fwd(x, gamma, beta, G, out):
    mean_rstd, y = out
    mean, u_mean, rstd, u_rstd = lo.gn_stats(x, G, mean_rstd[:, 0], EPS)
    r = [lo.check_value("gn mean", mean_rstd[:, 0], mean, u_mean), lo.check_value("gn rstd", mean_rstd[:, 1], rstd, u_rstd)]
    C = x.shape[-1]
    v, unit = lo.affine_statement(x, lo.per_channel(mean_rstd[:, 0], C), lo.per_channel(mean_rstd[:, 1], C), gamma, beta)
    r.append(lo.check_value("gn y", y, v, unit, lo.epi_relu(True)))
    return r


def test_gn_forward_emulation_accepted():
    x, gamma, beta, _, _, G = _gn_case()
    r = _judge_gn_fwd(x, gamma, beta, G, _emu_gn_fwd(x, gamma, beta, G))
    assert _ok(r), [q for q in r if not q.ok]


def test_gn_forward_groups_of_8_rejected():
    x, gamma, beta, _, _, G = _gn_case()
    assert not _ok(_judge_gn_fwd(x, gamma, beta, G, _emu_gn_fwd(x, gamma, beta, G, "groups_of_8")))


def _emu_gn_bwd(dy, y, x, gamma, mean_rstd, G, old, mut=None):
    B, H, W, C = x.shape
    dz = torch.where(y.float() > 0, dy.float(), torch.zeros_like(dy, dtype=torch.float32))
    m, r = lo.per_channel(mean_rstd[:, 0], C).float(), lo.per_channel(mean_rstd[:, 1], C).float()
    xhat = (x.float() - m) * r
    dg, db = (dz * xhat).sum((0, 1, 2)), dz.sum((0, 1, 2))
    if mut != "dgamma_overwritten":
        dg, db = old[0] + dg, old[1] + db
    a = (dz * gamma).reshape(B, H * W, G, C // G)
    Mg = H * W * (C // G)
    sa = a.sum((1, 3)) / Mg
    sb = (a * xhat.reshape(B, H * W, G, C // G)).sum((1, 3)) / Mg
    dx = r * (dz * gamma - lo.per_channel(sa, C) - xhat * lo.per_channel(sb, C))
    return lo.rn_bf16(dx).to(BF), dz.to(BF), dg, db


def _judge_gn_bwd(dy, y, x, gamma, mean_rstd, G, old, out):
    dx, dres, dg, db = out
    dz = torch.where(y.double() > 0, dy.double(), torch.zeros_like(dy, dtype=torch.float64))
    v, unit, xhat = lo.gn_dx_statement(dz, x, gamma, mean_rstd, G)
    C = x.shape[-1]
    terms = torch.stack([(dz * xhat).reshape(-1, C), dz.reshape(-1, C)])
    r = [lo.check_value("gn dx", dx, v, unit, lo.rn_bf16), lo.check_sums("gn dgamma/dbeta", torch.stack([dg, db]), terms, old, rounding=3)]
    r.append(lo.Result("gn dres", 0, 0, (), torch.equal(dres, dz.to(BF))))
    return r


def _gn_bwd_case():
    x, gamma, beta, dy, old, G = _gn_case()
    mean_rstd, y = _emu_gn_fwd(x, gamma, beta, G)
    return dy, y, x, gamma, mean_rstd, G, old


def test_gn_backward_emulation_accepted():
    c = _gn_bwd_case()
    r = _judge_gn_bwd(*c, _emu_gn_bwd(*c))
    assert _ok(r), [q for q in r if not q.ok]


def test_gn_backward_dgamma_overwritten_rejected():
    c = _gn_bwd_case()
    assert not _ok(_judge_gn_bwd(*c, _emu_gn_bwd(*c, "dgamma_overwritten")))


# =====================================================================================================================
# pooling and dropout
# =====================================================================================================================
DROP = lo.Drop(0.3, 1234, (1 << 61) + 5, 6)


def _bits_mut(n, d, mut):
    """Dropout bits with a mutated key: stream without the << 20 shift, or the other 16-bit half-word."""
    q = np.arange((n + 7) // 8, dtype=np.uint64)
    stream = (d.step ^ d.node) if mut == "stream_unshifted" else (((d.step << 20) & lo._M64) ^ d.node)
    u = np.stack(lo.ops_philox()(q, stream, d.seed))
    e = np.arange(n)
    w = u[(e % 8) // 2, e // 8].astype(np.uint32)
    half = (1 - e % 2) if mut == "wrong_half_word" else (e % 2)
    return (w >> (16 * half).astype(np.uint32)) & np.uint32(0xFFFF)


def _keep_mut(shape, d, mut=None):
    n = math.prod(shape)
    bits = _bits_mut(n, d, mut) if mut in ("stream_unshifted", "wrong_half_word") else lo.dropout_bits(n, d)
    keep = bits > d.thr if mut == "greater_not_geq" else bits >= d.thr
    return torch.from_numpy(keep).reshape(shape)


def _tie_drop(n):
    """A Drop whose threshold equals the random bits of one of the first ``n`` elements (so ``>`` and ``>=`` differ there)."""
    base = lo.Drop(0.3, 99, 12345, 3)
    bits = lo.dropout_bits(n, base)
    k = int(np.flatnonzero((bits > 6000) & (bits < 60000))[0])
    return lo.Drop(float(bits[k]) / 65536.0, base.seed, base.step, base.node)


def _emu_maxpool(x, d=None, mut=None):
    B, H, W, C = x.shape
    Ho, Wo = H // 2, W // 2
    xc = x[:, :2 * Ho, :2 * Wo].float()
    cands = [xc[:, dy::2, dx::2] for dy in (0, 1) for dx in (0, 1)]
    best, idx = cands[0].clone(), torch.zeros(B, Ho, Wo, C, dtype=torch.uint8)
    for k in (1, 2, 3):
        up = cands[k] >= best if mut == "last_max" else cands[k] > best
        best, idx = torch.where(up, cands[k], best), torch.where(up, torch.full_like(idx, k), idx)
    if d is not None:
        if mut == "keyed_by_input_index":
            keep = _keep_mut(x.shape, d)[:, 0:2 * Ho:2, 0:2 * Wo:2]
        else:
            keep = _keep_mut(best.shape, d, mut)
        best = torch.where(keep, lo.rn_bf16(best * d.scale("f32")), torch.zeros_like(best))
    return best.to(BF), idx


def _pool_input(B=2, H=7, W=9, C=16, seed=7):
    """Post-ReLU values on a coarse grid: full of ties (zeros and repeated values)."""
    g = _gen(seed)
    return (torch.randint(-3, 4, (B, H, W, C), generator=g).float() * 0.5).clamp_min(0).to(BF)


def _maxpool_ok(x, d, out):
    y, idx = lo.maxpool_statement(x, d)
    return torch.equal(out[0], y) and torch.equal(out[1], idx)


@pytest.mark.parametrize("drop", [False, True])
def test_maxpool_emulation_accepted(drop):
    x = _pool_input()
    d = DROP if drop else None
    assert _maxpool_ok(x, d, _emu_maxpool(x, d))


@pytest.mark.parametrize("mut", ["last_max", "keyed_by_input_index", "stream_unshifted", "wrong_half_word"])
def test_maxpool_mutant_rejected(mut):
    x = _pool_input(B=4, H=16, W=16, C=32)
    assert not _maxpool_ok(x, DROP, _emu_maxpool(x, DROP, mut))


def test_dropout_greater_instead_of_geq_rejected():
    x = _pool_input(B=4, H=16, W=16, C=32)
    d = _tie_drop(4 * 8 * 8 * 32)
    assert _maxpool_ok(x, d, _emu_maxpool(x, d))
    assert not _maxpool_ok(x, d, _emu_maxpool(x, d, "greater_not_geq"))


def _emu_maxpool_bwd(dy, idx, in_shape, d=None, zmask=None, mut=None):
    B, H, W, C = in_shape
    Ho, Wo = H // 2, W // 2
    g = dy.float()
    if d is not None:
        g = torch.where(_keep_mut(g.shape, d), g * d.scale("f32"), torch.zeros_like(g))
    if zmask is not None:
        g = torch.where(zmask.float() > 0, g, torch.zeros_like(g))
    dx = torch.full((B, H, W, C), float("nan"))          # the NaN prefill of the output buffer
    for k in range(4):
        dx[:, (k >> 1):2 * Ho:2, (k & 1):2 * Wo:2] = torch.where(idx == k, g, torch.zeros_like(g))
    if mut != "odd_edge_not_zeroed":
        dx[:, 2 * Ho:] = 0
        dx[:, :, 2 * Wo:] = 0
    return lo.rn_bf16(dx).to(BF)


@pytest.mark.parametrize("mut", [None, "odd_edge_not_zeroed"])
def test_maxpool_backward(mut):
    x = _pool_input()
    y, idx = lo.maxpool_statement(x, DROP)
    dy = torch.randn(y.shape, generator=_gen(8)).to(BF)
    out = _emu_maxpool_bwd(dy, idx, x.shape, DROP, y, mut)
    assert torch.equal(out, lo.maxpool_bwd_statement(dy, idx, x.shape, DROP, y)) == (mut is None)


@pytest.mark.parametrize("mut", [None, "divide_by_H"])
def test_avgpool(mut):
    x = (torch.randn(3, 4, 5, 16, generator=_gen(9)) + 1).to(BF)
    B, H, W, C = x.shape
    y = lo.rn_bf16(x.float().sum((1, 2)) / (H if mut else H * W)).to(BF)
    st, phi = lo.avgpool_statement(x)
    assert lo.check("avgpool", y, st, phi).ok == (mut is None)
    dy = torch.randn(B, C, generator=_gen(10)).to(BF)
    dx = lo.rn_bf16(dy.float().reshape(B, 1, 1, C) / (H if mut else H * W)).expand(B, H, W, C).to(BF)
    assert torch.equal(dx, lo.avgpool_bwd_statement(dy, x.shape)) == (mut is None)


def test_relu_bwd_and_standalone_dropout():
    g = _gen(11)
    dy = torch.randn(64, 40, generator=g).to(BF)
    y = torch.randn(64, 40, generator=g).clamp_min(0).to(BF)
    for scale in (1.0, 2.0, 1 / 0.9, 1 / 0.7):
        want = lo.relu_bwd_statement(dy, y, scale)
        assert torch.equal(want, torch.where(y > 0, (dy.float() * np.float32(scale)).to(BF), torch.zeros_like(dy)))
        assert not torch.equal(want, torch.where(y > 0, dy.float().to(BF), torch.zeros_like(dy))) or scale == 1.0
    x = torch.randn(16, 1024, generator=g).to(BF)
    yd, mask = lo.dropout_statement(x, DROP)
    assert torch.equal(mask.bool(), _keep_mut(x.shape, DROP))
    assert torch.equal(yd, torch.where(mask.bool(), (x.float() * DROP.scale("f32")).to(BF), torch.zeros_like(x)))
    assert not torch.equal(mask.bool(), _keep_mut(x.shape, DROP, "stream_unshifted"))
    assert not torch.equal(mask.bool(), _keep_mut(x.shape, DROP, "wrong_half_word"))
    assert abs(float(mask.float().mean()) - 0.7) < 0.01


# =====================================================================================================================
# linear layer with fused dropout (GEMM epilogue / split-K finishing pass)
# =====================================================================================================================
@pytest.mark.parametrize("mut", [None, "scale_after_pack"])
def test_linear_dropout_epilogue(mut):
    g = _gen(12)
    M, K, N = 64, 1024, 128
    x, w = torch.randn(M, K, generator=g).to(BF), (torch.randn(N, K, generator=g) / 32).to(BF)
    b = torch.randn(N, generator=g) * 0.1
    d = lo.Drop(0.1, 5, 77, 9)
    keep = lo.dropout_keep((M, N), d)
    s = d.scale("f64")
    a = (x.float() @ w.float().t() + b).clamp_min(0)
    if mut:
        y = torch.where(keep, lo.rn_bf16(lo.rn_bf16(a) * s), torch.zeros_like(a)).to(BF)
    else:
        y = torch.where(keep, lo.rn_bf16(a * s), torch.zeros_like(a)).to(BF)
    r = lo.check("linear+drop", y, lo.gemm_statement(x, w), lo.epi_linear_drop(b, True, keep, s))
    assert r.ok == (mut is None), r
