"""CRFL on the H100: the clip-and-perturb pass at ResNet-18's n_vote and on adversarial vectors (NaN, a norm exactly at rho, the BatchNorm
tail, the alignment padding, signed zeros); the device normals against fp64 Box-Muller of ``ops.philox4x32``'s words; the general output
bit for bit against fp32(fp32(w' s) + fp32(sigma z_dev)); the smoothing pass's fp32 buffer and bf16 shadow; the vote-count pass against a
torch argmax count; native cnn_mnist / resnet18 runs that are bitwise reproducible and resume bit for bit (also with --server_topk, with
the fused hand-off on); and, with >= 2 GPUs, the fused multi-GPU path and the certification counts against one process."""
import math
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import rlr_b200  # noqa: F401
from rlr_b200 import ops
from rlr_b200.models import get_layout

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NORMAL_ULPS = 16          # device normals (logf, sqrtf, sincospif, one fp32 product) against fp64 Box-Muller of the same words
WORD_UNITS = 64           # units of 2^-24 within which a Philox word's high 24 bits are recovered from a device normal pair


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _bits(x):
    x = np.array(x, dtype=np.float32).reshape(-1)
    x[np.isnan(x)] = np.float32("nan")
    return x.tobytes()


def _ulp(x):
    """fp32 ulp of |x| (the spacing above it)."""
    a = np.abs(np.asarray(x, dtype=np.float32))
    return (np.nextafter(a, np.float32(np.inf)) - a).astype(np.float64)


def _device_normals(n, n_vote, mask, seed, stream, smooth=False):
    """z_dev on every real coordinate: a launch with w' = 0, s = 1 (no clip) and sigma = 1 writes fp32(0 + fp32(1 z)) = z_dev."""
    zero = torch.zeros(n, device=DEV)
    out = torch.full((n,), float("nan"), device=DEV)
    if smooth:
        ops.ext().crfl_smooth(zero, out, None, mask, n_vote, 1.0, ops._i64(seed), ops._i64(stream))
    else:
        stats = torch.zeros(2, dtype=torch.float64, device=DEV)
        ops.ext().crfl_clip_noise(zero, out, None, mask, n_vote, math.inf, 1.0, ops._i64(seed), ops._i64(stream), stats)
    return out.cpu().numpy()


def _check_normals(z_dev, real, seed, stream, n_vote):
    z64 = ops.philox_normals(seed, stream, n_vote)
    zd = z_dev[:n_vote]
    err = np.abs(zd[real].astype(np.float64) - z64[real]) / _ulp(z64[real].astype(np.float32))
    assert err.max() <= NORMAL_ULPS, f"device normals {err.max():.2f} ulp from fp64 Box-Muller"
    # the words themselves: the high 24 bits of the radius and angle words, recovered in fp64 from each device pair, lie within WORD_UNITS
    # of the host's (the fp32 normals carry about 24 bits, so the recovery may miss by a few units; a different word would be off by
    # 2^22 on average).  A radius word of 2^24 - 1 gives u = 1, r = 0 and a pair of zeros: its angle word never reaches the normals, so
    # only the radius is recovered there.
    q = np.arange(n_vote // 4)
    pairs = zd.reshape(-1, 4).astype(np.float64)
    both = real.reshape(-1, 4)
    words = ops.philox4x32(q.astype(np.uint64), stream, seed)
    for lane, (rw, aw) in enumerate(((0, 1), (2, 3))):
        ok = both[:, 2 * lane] & both[:, 2 * lane + 1]
        zc, zs = pairs[ok, 2 * lane], pairs[ok, 2 * lane + 1]
        hi_r = np.exp(-0.5 * (zc * zc + zs * zs)) * 2 ** 24 - 1
        hi_a = np.mod(np.arctan2(zs, zc) / (2 * np.pi), 1.0) * 2 ** 24 - 1
        d_r = np.abs(hi_r - (words[rw][ok] >> 8).astype(np.float64))
        d_a = np.abs(hi_a - (words[aw][ok] >> 8).astype(np.float64))
        angle = (zc != 0) | (zs != 0)
        assert ((words[rw][ok][~angle] >> 8) == 2 ** 24 - 1).all()
        assert d_r.max() <= WORD_UNITS and np.minimum(d_a, 2 ** 24 - d_a)[angle].max() <= WORD_UNITS
    return err.max()


def _device_pass(wn, mask, n_vote, rho, sigma, seed, rnd, in_place=False):
    n = wn.size
    dwn = torch.from_numpy(wn).to(DEV)
    out = dwn if in_place else torch.full((n,), float("nan"), device=DEV)
    wb = torch.full((n,), float("nan"), dtype=torch.bfloat16, device=DEV)
    stats = torch.full((2,), float("nan"), dtype=torch.float64, device=DEV)
    ops.crfl_step(out, dwn, mask.to(DEV), n_vote, rho, sigma, seed, rnd, stats, wb)
    return out.cpu().numpy(), wb.cpu(), stats.cpu().tolist()


def _general_check(wn, lay_n_vote, mask, rho, sigma, seed, rnd):
    """Device output bit for bit against fp32(fp32(w' s_dev) + fp32(sigma z_dev)) on the real coordinates and w' elsewhere; the shadow is
    bf16 of it; the norm and s against the fp64 statement."""
    n = wn.size
    real = ops.mask_bits(mask, lay_n_vote).numpy()
    stream = ops.crfl_stream(rnd)
    out, wb, (norm, s) = _device_pass(wn, mask, lay_n_vote, rho, sigma, seed, rnd)
    ref, ref_norm, ref_s = ops.crfl_statement(wn, mask, lay_n_vote, rho, sigma, seed, stream)
    assert (math.isnan(norm) and math.isnan(ref_norm)) or math.isclose(norm, ref_norm, rel_tol=1e-12)
    assert s == ref_s or math.isclose(s, ref_s, rel_tol=2 ** -23)
    z = _device_normals(n, lay_n_vote, mask.to(DEV), seed, stream) if sigma > 0 else np.zeros(n, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        v = wn[:lay_n_vote]
        o = (v * np.float32(s)).astype(np.float32)
        if sigma > 0:
            o = (o + (np.float32(sigma) * z[:lay_n_vote]).astype(np.float32)).astype(np.float32)
    want = wn.copy()
    want[:lay_n_vote] = np.where(real, o, v)
    assert _bits(out) == _bits(want), "clip / noise output"
    assert _bits(wb.float().numpy()) == _bits(torch.from_numpy(out).to(torch.bfloat16).float().numpy()), "bf16 shadow"
    assert out[lay_n_vote:].tobytes() == wn[lay_n_vote:].tobytes() and out[:lay_n_vote][~real].tobytes() == wn[:lay_n_vote][~real].tobytes()
    # the pass in place (after SparseFed) writes the same bits
    inp, _, st2 = _device_pass(wn, mask, lay_n_vote, rho, sigma, seed, rnd, in_place=True)
    assert _bits(inp) == _bits(out) and _bits(st2) == _bits([norm, s])
    return out, norm, s


@pytest.mark.parametrize("rho, sigma", [(0.0, 0.01), (50.0, 0.0), (50.0, 1e-3), (1e9, 0.02)])
def test_clip_noise_at_resnet18_size(rho, sigma):
    lay = get_layout("resnet18")
    mask = ops.real_mask(lay)
    rs = np.random.RandomState(1)
    wn = (0.05 * rs.randn(lay.n_total)).astype(np.float32)
    wn[lay.n_vote:] = np.abs(wn[lay.n_vote:])
    out, norm, s = _general_check(wn, lay.n_vote, mask, rho, sigma, 7, 3)
    assert (s < 1.0) == (0 < rho < norm)
    if rho > 0 and sigma == 0:
        real = ops.mask_bits(mask, lay.n_vote).numpy()
        assert np.sqrt(np.sum(out[:lay.n_vote][real].astype(np.float64) ** 2)) <= rho * (1 + 4e-7)


def test_device_normals_follow_the_philox_words():
    lay = get_layout("resnet18")
    mask = ops.real_mask(lay)
    real = ops.mask_bits(mask, lay.n_vote).numpy()
    worst = []
    for seed, stream in ((7, ops.crfl_stream(1)), (2 ** 40 + 3, ops.crfl_stream(99)), (0, ops.crfl_stream(5, certify=True))):
        z = _device_normals(lay.n_total, lay.n_vote, mask.to(DEV), seed, stream)
        worst.append(_check_normals(z, real, seed, stream, lay.n_vote))
        zs = _device_normals(lay.n_total, lay.n_vote, mask.to(DEV), seed, stream, smooth=True)
        assert zs.tobytes() == z.tobytes()                                 # the smoothing launch draws the same normals
    print(f"largest device-normal error: {max(worst):.2f} ulp")


def _adversarial():
    lay = get_layout("cnn_mnist")
    mask = ops.real_mask(lay)
    n, nv = lay.n_total, lay.n_vote
    rs = np.random.RandomState(3)
    base = (0.1 * rs.randn(n)).astype(np.float32)
    base[nv:] = 1.5                                                         # the BatchNorm tail (cnn_mnist has none: n_total == n_vote)
    at_rho = np.zeros(n, dtype=np.float32)
    at_rho[0], at_rho[5] = 3.0, 4.0                                         # norm exactly 5
    nan = base.copy()
    nan[17] = np.nan
    zeros = base.copy()
    zeros[:64] = -0.0
    big = (1e20 * rs.randn(n)).astype(np.float32)                           # q near fp64 range is still finite
    return [(base, mask, nv, 1.0, 0.01), (at_rho, mask, nv, 5.0, 0.0), (at_rho, mask, nv, 5.0, 0.5), (nan, mask, nv, 1.0, 0.01),
            (zeros, mask, nv, 0.0, 0.0), (big, mask, nv, 1.0, 0.0)]


@pytest.mark.parametrize("case", range(6))
def test_clip_noise_on_adversarial_vectors(case):
    wn, mask, nv, rho, sigma = _adversarial()[case]
    out, norm, s = _general_check(wn, nv, mask, rho, sigma, 11, 2)
    if case in (1, 2):
        assert norm == 5.0 and s == 1.0
    if case == 1 or case == 4:
        assert out.tobytes() == wn.tobytes()                                # s = 1, sigma = 0: the identity, -0 included
    if case == 3:
        assert math.isnan(norm) and s == 1.0 and np.isnan(out[17])


def test_clip_noise_with_a_batchnorm_tail():
    lay = get_layout("resnet18")
    assert lay.n_total > lay.n_vote
    mask = ops.real_mask(lay)
    rs = np.random.RandomState(4)
    wn = rs.randn(lay.n_total).astype(np.float32)
    wn[lay.n_vote:] = np.nan                                                # the tail is never read into the norm
    out, norm, s = _general_check(wn, lay.n_vote, mask, 10.0, 0.01, 3, 8)
    assert math.isfinite(norm) and s < 1.0 and np.isnan(out[lay.n_vote:]).all()


def test_smoothing_pass_fp32_and_bf16():
    lay = get_layout("resnet18")
    mask = ops.real_mask(lay).to(DEV)
    real = ops.mask_bits(mask.cpu(), lay.n_vote).numpy()
    rs = np.random.RandomState(5)
    w = (0.05 * rs.randn(lay.n_total)).astype(np.float32)
    dw = torch.from_numpy(w).to(DEV)
    sigma, seed = 0.03, 9
    for m in (0, 1, 1234):
        out = torch.full((lay.n_total,), float("nan"), device=DEV)
        ob = torch.full((lay.n_total,), float("nan"), dtype=torch.bfloat16, device=DEV)
        ops.crfl_smooth(dw, mask, lay.n_vote, sigma, seed, m, out, ob)
        z = _device_normals(lay.n_total, lay.n_vote, mask, seed, ops.crfl_stream(m, certify=True), smooth=True)
        want = w.copy()
        v = w[:lay.n_vote]
        want[:lay.n_vote] = np.where(real, (v + (np.float32(sigma) * z[:lay.n_vote]).astype(np.float32)).astype(np.float32), v)
        got = out.cpu().numpy()
        assert got.tobytes() == want.tobytes()
        assert torch.equal(ob.cpu(), torch.from_numpy(want).to(torch.bfloat16))
        assert torch.equal(dw.cpu(), torch.from_numpy(w))                     # the global model is left as it was


@pytest.mark.parametrize("rows, classes", [(1, 1), (300, 10), (5000, 10), (777, 100), (64, 1000)])
def test_vote_count_against_torch(rows, classes):
    g = torch.Generator().manual_seed(rows + classes)
    x = torch.randn(rows, classes, generator=g)
    x = torch.round(x * 2) / 2                                                # many ties
    if rows > 4:
        x[1] = 0.0                                                           # all tied: class 0
        x[2, classes // 2] = float("nan")
        x[3, 0] = float("inf")
        x[4, -1] = float("-inf")
    dx = x.to(DEV)
    counts = torch.zeros((rows + 7, classes), dtype=torch.int32, device=DEV)
    ops.vote_count(dx, counts, 7)
    ops.vote_count(dx, counts, 7)
    ops.vote_count(dx[: rows // 2], counts, 0)
    want = torch.zeros((rows + 7, classes), dtype=torch.int32)
    ops.vote_count(x, want, 7)
    ops.vote_count(x, want, 7)
    ops.vote_count(x[: rows // 2], want, 0)
    assert torch.equal(counts.cpu(), want)
    # the same counts from a plain loop: the first maximum of every finite row
    loop = torch.zeros((rows + 7, classes), dtype=torch.int32)
    for r, row in enumerate(x.numpy()):
        if np.isfinite(row).all():
            c = int(np.flatnonzero(row == row.max())[0])
            loop[7 + r, c] += 2
            if r < rows // 2:
                loop[r, c] += 1
    assert torch.equal(want, loop)
    if rows > 4:
        single = torch.zeros((rows, classes), dtype=torch.int32, device=DEV)
        ops.vote_count(dx, single, 0)
        assert single[1, 0] == 1 and single[1].sum() == 1                   # all tied: the lowest class
        assert single[2:5].sum() == 0                                         # NaN, +inf, -inf rows vote for no class


# ---- native runs --------------------------------------------------------------------------------------------------------------
def _engine(model, **kw):
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    data = "fmnist" if model == "cnn_mnist" else "cifar10"
    base = dict(data=data, model=model, num_agents=3, local_ep=1, bs=64, synthetic=384, synthetic_val=200, log_dir="", device=DEV,
                seed=2, robustLR_threshold=2, num_corrupt=1, poison_frac=0.5, param_clip=30.0, param_noise=1e-3)
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


@pytest.mark.parametrize("model, topk", [("cnn_mnist", 0.0), ("resnet18", 0.0), ("resnet18", 0.01)])
def test_native_runs_are_bitwise_reproducible_and_resume(tmp_path, model, topk):
    cert = dict(certify=True, certify_n0=4, certify_n=16)
    runs = []
    for _ in range(2):
        ops.reset_fallbacks()
        eng = _engine(model, rounds=3, server_topk=topk, **cert)
        assert eng.trainer.name == "native" and eng.handoff
        hist = eng.fit()
        torch.cuda.synchronize()
        assert not ops.fallback_calls()
        runs.append((eng.global_params().clone(), [(h["param_norm"], h["param_scale"]) for h in hist],
                     {k: v for k, v in hist[-1].items() if k.startswith("certify")},
                     {k: (v["selection"].copy(), v["estimation"].copy()) for k, v in eng.last_certify.items()}))
        eng.close()
    assert torch.equal(runs[0][0], runs[1][0]) and runs[0][1] == runs[1][1] and runs[0][2] == runs[1][2]
    for name in ("val", "poison"):
        assert all(np.array_equal(a, b) for a, b in zip(runs[0][3][name], runs[1][3][name]))
        assert runs[0][3][name][1].sum(1).max() <= 16
    assert any(s < 1.0 for _, s in runs[0][1]) or model == "cnn_mnist"
    ck = str(tmp_path / "ck.pt")
    first = _engine(model, rounds=2, checkpoint=ck, server_topk=topk)
    first.fit()
    first.close()
    second = _engine(model, rounds=3, resume=ck, server_topk=topk, **cert)
    hist = second.fit()
    assert torch.equal(second.global_params(), runs[0][0])
    assert (hist[-1]["param_norm"], hist[-1]["param_scale"]) == runs[0][1][-1]
    assert {k: v for k, v in hist[-1].items() if k.startswith("certify")} == runs[0][2]
    second.close()


def test_native_tiny_sigma_certifies_the_plain_predictions():
    eng = _engine("cnn_mnist", rounds=2, param_clip=0.0, param_noise=1e-12)     # below half an fp32 ulp of nearly every weight
    eng.fit()
    eng.args.certify_n0, eng.args.certify_n = 2, 16               # n_A = 16 gives p_A = alpha^(1/16) = 0.65 > 1/2
    res = eng.certify()
    fwd = eng.trainer.eval_forward(eng.global_params())
    for name, ds in (("val", eng.val_dataset), ("poison", eng.poisoned_val)):
        x, _ = ds.batch(torch.arange(len(ds), device=ds.device))
        plain = torch.cat([fwd(x[s:s + 64]) for s in range(0, x.shape[0], 64)]).argmax(1).cpu().numpy()
        assert np.array_equal(res[name]["pred"], plain) and res[name]["abstain"] == 0.0
    eng.close()


# ---- fused multi-GPU path --------------------------------------------------------------------------------------------------
def _multi_worker(rank, world, port, outdir, handoff, topk):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from rlr_b200 import ops as o
    from rlr_b200.engine import FLEngine
    from rlr_b200.models import get_layout as gl
    from rlr_b200.options import make_args
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed()
    lay = gl("resnet18")
    n, nv, n_part = lay.n_total, lay.n_vote, 2 * world + 1
    mask = o.real_mask(lay)
    fa = FusedAggregator(ctx, n, nv, (n_part + world - 1) // world, "fused", topk_k=topk, crfl=(40.0, 1e-3, mask))
    if handoff:
        fa.enable_handoff()
    ref_w, ref_b = torch.empty(n, device=ctx.device), torch.empty(n, dtype=torch.bfloat16, device=ctx.device)
    ref_e, ref_s = torch.zeros(nv, device=ctx.device), torch.zeros(3, dtype=torch.float64, device=ctx.device)
    ref_c = torch.zeros(2, dtype=torch.float64, device=ctx.device)
    dmask = mask.to(ctx.device)
    gen = torch.Generator().manual_seed(0)
    w0 = 0.05 * torch.randn(n, generator=gen)
    fa.w_global.copy_(w0.to(ctx.device)); fa.w_bf16.copy_(fa.w_global.to(torch.bfloat16)); ref_w.copy_(w0.to(ctx.device))
    ref_b.copy_(ref_w.to(torch.bfloat16))
    torch.cuda.synchronize(); dist.barrier()
    same = True
    for rnd in range(1, 4):
        fa.acquire()
        parts = [ref_w + (0.01 * torch.randn(n, generator=gen)).to(ctx.device) for _ in range(n_part)]
        for j in range(n_part):
            r, s = fa.slot_owner(j)
            if r == ctx.rank:
                fa.slots[s].copy_(fa.w_global + (parts[j] - ref_w))
        weights = [float(50 + 7 * j) for j in range(n_part)]
        fa.aggregate(weights, "avg", 3, 1.0, 0.0, 5, rnd)
        scratch = o.fused_aggregate(ref_w, parts, weights, "avg", 3, 1.0, n_vote=nv, out=torch.empty_like(ref_w))
        if topk:
            o.sparsefed_step(ref_w, scratch, ref_e, nv, topk, ref_s, ref_b)
            scratch = ref_w
        o.crfl_step(ref_w, scratch, dmask, nv, 40.0, 1e-3, 5, rnd, ref_c, ref_b)
        fa.acquire()
        torch.cuda.synchronize()
        same &= bool(torch.equal(fa.w_global, ref_w) and torch.equal(fa.w_bf16, ref_b) and torch.equal(fa.crfl_stats, ref_c))
    w_final = fa.w_global.cpu()
    fa.close()
    eng = FLEngine(make_args(data="fmnist", model="cnn_mnist", num_agents=2, synthetic=256, synthetic_val=200, bs=64, log_dir="",
                             seed=4, param_noise=0.02, certify=True, certify_n0=3, certify_n=9, num_corrupt=1, poison_frac=0.5),
                   ctx=ctx, verbose=False)
    res = eng.certify()
    torch.save({"same": same, "w": w_final, "cert": {k: (v["selection"], v["estimation"]) for k, v in res.items()}},
               os.path.join(outdir, f"c{int(handoff)}{topk}_{rank}.pt"))
    eng.close()
    dist.barrier(); dist.destroy_process_group()


def test_fused_multi_gpu_path_equals_one_process(tmp_path):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    for handoff, topk in ((False, 0), (True, 0), (True, 5000)):
        mp.spawn(_multi_worker, args=(world, _free_port(), str(tmp_path), handoff, topk), nprocs=world, join=True)
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    solo = FLEngine(make_args(data="fmnist", model="cnn_mnist", num_agents=2, synthetic=256, synthetic_val=200, bs=64, log_dir="",
                              seed=4, param_noise=0.02, certify=True, certify_n0=3, certify_n=9, num_corrupt=1, poison_frac=0.5,
                              device=DEV), verbose=False)
    ref = solo.certify()
    solo.close()
    for handoff, topk in ((False, 0), (True, 0), (True, 5000)):
        res = [torch.load(tmp_path / f"c{int(handoff)}{topk}_{r}.pt", weights_only=False) for r in range(world)]
        for x in res:
            assert x["same"] and torch.equal(x["w"], res[0]["w"])
            for name in ("val", "poison"):
                assert np.array_equal(x["cert"][name][0], ref[name]["selection"]) and np.array_equal(x["cert"][name][1], ref[name]["estimation"])
