"""GPU numerics: every sm_90a kernel of ops/csrc vs. its plain-PyTorch fp32/fp64 oracle (run with -m gpu)."""
import pytest
import torch

import rlr_b200  # noqa: F401
from rlr_b200 import ops
from rlr_b200.data import make_synthetic, pattern_pixels

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_extension_loaded():
    assert ops.ext() is not None


@pytest.mark.parametrize("name", ["fmnist", "cifar10"])
@pytest.mark.parametrize("dtype,nhwc,cpad", [(torch.float32, False, None), (torch.bfloat16, True, 8), (torch.float32, True, None)])
def test_gather_normalize(name, dtype, nhwc, cpad):
    tr, _ = make_synthetic(name, 300)
    idx = torch.randperm(300)[:77]
    ref = ops.gather_normalize(tr.data, idx, tr.meta.mean, tr.meta.std, dtype=torch.float32, nhwc=nhwc, c_pad=cpad)
    out = ops.gather_normalize(tr.data.to(DEV), idx.to(DEV), tr.meta.mean, tr.meta.std, dtype=dtype, nhwc=nhwc, c_pad=cpad)
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    torch.testing.assert_close(out.float().cpu(), ref, atol=tol, rtol=tol)


@pytest.mark.parametrize("name,k,pad,B", [("cifar10", 3, 1, 37), ("fmnist", 3, 0, 64), ("cifar10", 3, 0, 5), ("fmnist", 5, 2, 19)])
def test_gather_im2col_matches_oracle(name, k, pad, B):
    """Batch assembly fused with the first layer's im2col (tiny-K stems) vs the CPU statement of the same op."""
    tr, _ = make_synthetic(name, 200)
    d = tr.clone().to(DEV)
    perm = torch.randperm(200)
    cur = torch.tensor([11], dtype=torch.int32)
    H, W = tr.data.shape[1], tr.data.shape[2]
    Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
    ref = torch.zeros(B * Ho * Wo, 64)
    yref = torch.zeros(B, dtype=torch.int64)
    ops.gather_im2col(tr.data, perm, tr.meta.mean, tr.meta.std, k, pad, ref, cursor=cur, targets=tr.targets, out_labels=yref, batch=B)
    out = torch.full((B * Ho * Wo, 64), 7.0, dtype=torch.bfloat16, device=DEV)
    y = torch.zeros(B, dtype=torch.int64, device=DEV)
    ops.gather_im2col(d.data, perm.to(DEV), tr.meta.mean, tr.meta.std, k, pad, out, cursor=cur.to(DEV), targets=d.targets, out_labels=y, batch=B)
    torch.testing.assert_close(out.float().cpu(), ref, atol=2e-2, rtol=2e-2)
    assert torch.equal(y.cpu(), yref)
    assert float(out[:, k * k * tr.data.shape[3]:].abs().max()) == 0.0          # padding columns are exact zeros


def test_gather_cursor_and_labels():
    tr, _ = make_synthetic("cifar10", 256)
    d = tr.clone().to(DEV)
    perm = torch.randperm(256, device=DEV)
    cursor = torch.tensor([64], dtype=torch.int32, device=DEV)
    x = torch.zeros(32, 3, 32, 32, device=DEV)
    y = torch.zeros(32, dtype=torch.int64, device=DEV)
    ops.gather_normalize(d.data, perm, d.meta.mean, d.meta.std, out=x, cursor=cursor, targets=d.targets, out_labels=y, batch=32)
    ops.ext().advance_cursor(cursor, 32)
    ref, yref = d.batch(perm[64:96])
    torch.testing.assert_close(x, ref)
    assert torch.equal(y, yref) and int(cursor.item()) == 96


@pytest.mark.parametrize("ds,pat,agent", [("cifar10", "plus", -1), ("cifar10", "plus", 2), ("fmnist", "square", -1),
                                          ("fmnist", "copyright", -1), ("fmnist", "apple", -1), ("fedemnist", "plus", -1),
                                          ("fedemnist", "apple", -1)])
def test_stamp_pixels(ds, pat, agent):
    tr, _ = make_synthetic(ds, 64)
    rows, cols, vals, mode = pattern_pixels(ds, pat, agent)
    sel = torch.tensor([3, 7, 11, 63])
    ref = ops.stamp_pixels(tr.data.clone(), sel, rows, cols, vals, mode)
    out = ops.stamp_pixels(tr.data.clone().to(DEV), sel.to(DEV), rows, cols, vals, mode)
    if out.dtype == torch.uint8:
        assert torch.equal(out.cpu(), ref)
    else:
        torch.testing.assert_close(out.cpu(), ref)


@pytest.mark.parametrize("mode", ["avg", "comed", "sign"])
@pytest.mark.parametrize("K,theta", [(1, 0), (2, 2), (5, 3), (8, 4), (8, 0), (9, 3), (11, 4), (12, 5), (16, 0), (17, 6), (24, 9), (32, 8),
                                     (33, 8), (40, 12), (41, 0), (48, 20), (64, 16), (65, 20), (100, 30), (128, 40), (200, 50), (321, 100),
                                     (400, 0), (1024, 300)])
def test_fused_aggregate_matches_oracle(mode, K, theta):
    """Every path of the fused server-step kernel against the fp64 oracle: vector kernels (avg / sign / median K <= 8), register
    sorting networks (median 8 < K <= 64), shared-memory staged bisection (64 < K <= 320) and global re-read bisection (K > 320)."""
    torch.manual_seed(K * 31 + theta)
    n, n_vote = 8192, 6144
    g = torch.randn(n)
    ws = [g + 0.1 * torch.randn(n) * (torch.rand(n) > 0.2) for _ in range(K)]   # ~20% exact zeros in every update
    wt = [float(100 + 13 * k) for k in range(K)]
    ref, nflip = ops.aggregate_oracle(g, ws, wt, mode, theta, 0.5 if mode == "sign" else 1.0, None, n_vote)
    gd = g.to(DEV)
    flipped = torch.zeros(1, dtype=torch.int64, device=DEV)
    out = torch.empty_like(gd)
    shadow = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    ops.fused_aggregate(gd, [w.to(DEV) for w in ws], wt, mode, theta, 0.5 if mode == "sign" else 1.0, n_vote=n_vote,
                        out=out, out_bf16=shadow, flipped=flipped)
    torch.testing.assert_close(out.cpu(), ref, atol=1e-6, rtol=1e-6)
    assert int(flipped.item()) == nflip
    torch.testing.assert_close(shadow.float().cpu(), ref.bfloat16().float())


def test_fused_aggregate_noise_statistics_and_scales():
    n = 1 << 18
    g = torch.zeros(n, device=DEV)
    ws = [torch.zeros(n, device=DEV) for _ in range(3)]
    out = torch.empty_like(g)
    ops.fused_aggregate(g, ws, [1, 1, 1], "avg", 0, 1.0, noise_std=0.25, seed=7, noise_stream=3, out=out)
    assert abs(out.mean().item()) < 5e-3 and abs(out.std().item() - 0.25) < 5e-3
    out2 = torch.empty_like(g)
    ops.fused_aggregate(g, ws, [1, 1, 1], "avg", 0, 1.0, noise_std=0.25, seed=7, noise_stream=4, out=out2)
    assert not torch.allclose(out, out2)
    # server-side clipping scales
    w1 = [torch.full((n,), 2.0, device=DEV), torch.full((n,), -1.0, device=DEV)]
    ref, _ = ops.aggregate_oracle(g.cpu(), [w.cpu() for w in w1], [1, 3], "avg", 0, 1.0, scales=[0.5, 1.0])
    out3 = torch.empty_like(g)
    ops.fused_aggregate(g, w1, [1, 3], "avg", 0, 1.0, scales=[0.5, 1.0], out=out3)
    torch.testing.assert_close(out3.cpu(), ref)
    norms = ops.update_norms(g, w1)
    torch.testing.assert_close(norms.cpu(), torch.tensor([2.0 * n ** 0.5, n ** 0.5], dtype=torch.float64))


@pytest.mark.parametrize("pgd", [0.0, 0.05])
def test_flat_sgd_matches_torch_optimizer(pgd):
    torch.manual_seed(0)
    n = 4096 * 3
    w0 = torch.randn(n)
    w_ref = w0.clone().requires_grad_(True)
    opt_ref = torch.optim.SGD([w_ref], lr=0.1, momentum=0.9)
    w = w0.clone().to(DEV); m = torch.zeros(n, device=DEV); shadow = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
    w0d = w0.to(DEV)
    opt = ops.FlatSGD(n, DEV, 0.1, 0.9, 10.0, pgd)
    for it in range(4):
        g = torch.randn(n) * (30.0 if it % 2 == 0 else 0.01)   # exercise both clipped and unclipped steps
        w_ref.grad = g.clone()
        torch.nn.utils.clip_grad_norm_([w_ref], 10)
        opt_ref.step()
        if pgd > 0:
            with torch.no_grad():
                upd = w_ref - w0
                w_ref.copy_(w0 + upd / max(1.0, float(upd.norm()) / pgd))
        opt.step(w, g.to(DEV), m, w0=w0d, w_bf16=shadow)
        torch.testing.assert_close(w.cpu(), w_ref.detach(), atol=2e-5, rtol=1e-5)
    torch.testing.assert_close(shadow.float().cpu(), w.cpu().bfloat16().float())


def test_round_init():
    n = 8192
    g = torch.randn(n, device=DEV)
    w = torch.zeros(n, device=DEV); m = torch.ones(n, device=DEV); b = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
    ops.round_init(g, w, b, m)
    assert torch.equal(w, g) and float(m.abs().sum()) == 0 and torch.equal(b, g.bfloat16())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_softmax_xent_and_eval_metrics(dtype):
    torch.manual_seed(1)
    B, C = 203, 10
    logits = (torch.randn(B, C) * 3).to(dtype)
    y = torch.randint(0, C, (B,))
    ref_loss, ref_dl = ops.softmax_xent(logits, y)
    correct = torch.zeros(1, dtype=torch.int32, device=DEV)
    loss, dl = ops.softmax_xent(logits.to(DEV), y.to(DEV), correct=correct)
    tol = 1e-4 if dtype == torch.float32 else 2e-2
    torch.testing.assert_close(loss.cpu(), ref_loss, atol=tol * B, rtol=tol)
    torch.testing.assert_close(dl.float().cpu(), ref_dl.float(), atol=tol, rtol=tol)
    assert int(correct.item()) == int((logits.float().argmax(1) == y).sum())
    ls, conf = torch.zeros(1, dtype=torch.float64, device=DEV), torch.zeros(C, C, dtype=torch.int64, device=DEV)
    ops.eval_metrics(logits.to(DEV), y.to(DEV), ls, conf)
    ls_ref, conf_ref = torch.zeros(1, dtype=torch.float64), torch.zeros(C, C, dtype=torch.int64)
    ops.eval_metrics(logits, y, ls_ref, conf_ref)
    assert torch.equal(conf.cpu(), conf_ref)
    torch.testing.assert_close(ls.cpu(), ls_ref, atol=1e-3, rtol=1e-4)


def test_engine_round_gpu_torch_trainer_with_graphs():
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    args = make_args(data="fmnist", num_agents=3, local_ep=1, bs=64, synthetic=600, synthetic_val=100, num_corrupt=1,
                     poison_frac=0.5, robustLR_threshold=2, log_dir="", device=DEV, trainer="torch", dtype="fp32")
    eng = FLEngine(args, verbose=False)
    before = eng.w_global.clone()
    for r in range(1, 9):
        eng.run_round(r)
    ev = eng.evaluate(8)
    assert not torch.equal(before, eng.w_global) and ev["val_acc"] > 0.3
    eng.close()
