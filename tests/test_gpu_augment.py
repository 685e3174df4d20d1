"""Training augmentation (--crop_pad / --hflip) in the sm_90a batch-assembly kernels (run with -m gpu).

The geometry is checked exactly: a kernel with augmentation on over the dataset must equal, bit for bit, the same kernel with
augmentation off over images cropped and flipped on the host from the host Philox draws -- the per-pixel arithmetic is then the
same, so any difference is a wrong source pixel or a wrong draw."""
import numpy as np
import pytest
import torch

import rlr_b200  # noqa: F401
from rlr_b200 import ops
from rlr_b200.data import make_synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _aug(pad, flip, seed=7, stream=987654321, start=0):
    return ops.Augment(pad, flip, seed, torch.tensor([stream], dtype=torch.int64, device=DEV), start)


def _host_augmented(data, sel, pos0, aug):
    """Raw images data[sel] cropped / flipped on the host, in the dataset's own dtype (exact for uint8 and float)."""
    cpu_aug = aug._replace(stream=int(aug.stream))
    return ops.augment_raw(data.cpu()[sel.cpu()].to(torch.float32), cpu_aug, pos0).to(data.dtype).contiguous()


CASES = [(4, True), (1, False), (0, True)]


@pytest.mark.parametrize("name,k,pad", [("cifar10", 3, 1), ("cifar10", 3, 0), ("fmnist", 3, 0), ("fmnist", 5, 2), ("fedemnist", 3, 1)])
@pytest.mark.parametrize("cpad,flip", CASES)
def test_gather_im2col_geometry_is_exact(name, k, pad, cpad, flip):
    tr, _ = make_synthetic(name, 300)
    d = tr.clone().to(DEV)
    perm = torch.randperm(300, generator=torch.Generator().manual_seed(3)).to(DEV)
    cur, B = 41, 37                                                       # non-zero cursor, ragged batch
    H, W, C = tr.data.shape[1:]
    Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
    aug = _aug(cpad, flip)
    out = torch.full((B * Ho * Wo, 64), 3.0, dtype=torch.bfloat16, device=DEV)
    y = torch.zeros(B, dtype=torch.int64, device=DEV)
    ops.gather_im2col(d.data, perm, d.meta.mean, d.meta.std, k, pad, out, cursor=torch.tensor([cur], dtype=torch.int32, device=DEV),
                      targets=d.targets, out_labels=y, batch=B, augment=aug)
    sel = perm[cur:cur + B]
    host = _host_augmented(d.data, sel, cur, aug).to(DEV)
    ref = torch.full_like(out, -1.0)
    ops.gather_im2col(host, torch.arange(B, device=DEV), d.meta.mean, d.meta.std, k, pad, ref, batch=B)
    assert torch.equal(out, ref)
    assert torch.equal(y, d.targets[sel])                                   # labels untouched


@pytest.mark.parametrize("name", ["cifar10", "fmnist", "fedemnist"])
@pytest.mark.parametrize("layout", ["nchw_fp32", "nhwc_pad_bf16"])
@pytest.mark.parametrize("cpad,flip", CASES)
def test_gather_normalize_geometry_is_exact(name, layout, cpad, flip):
    tr, _ = make_synthetic(name, 300)
    d = tr.clone().to(DEV)
    perm = torch.randperm(300, generator=torch.Generator().manual_seed(4)).to(DEV)
    aug = _aug(cpad, flip)
    kw = dict(dtype=torch.float32) if layout == "nchw_fp32" else dict(dtype=torch.bfloat16, nhwc=True, c_pad=8)
    for cur, B in [(0, 64), (250, 50)]:
        # cursor path (captured steps) and explicit-start path (eager steps) draw at the same positions
        out = ops.gather_normalize(d.data, perm, d.meta.mean, d.meta.std, cursor=torch.tensor([cur], dtype=torch.int32, device=DEV),
                                   batch=B, augment=aug, **kw)
        eager = ops.gather_normalize(d.data, perm[cur:cur + B], d.meta.mean, d.meta.std, augment=aug._replace(start=cur), **kw)
        host = _host_augmented(d.data, perm[cur:cur + B], cur, aug).to(DEV)
        ref = ops.gather_normalize(host, torch.arange(B, device=DEV), d.meta.mean, d.meta.std, **kw)
        assert torch.equal(out, ref) and torch.equal(eager, ref)
        # and the CPU statement agrees to float rounding
        cpu = ops.gather_normalize(tr.data, perm.cpu(), tr.meta.mean, tr.meta.std, cursor=torch.tensor([cur], dtype=torch.int32), batch=B,
                                   augment=aug._replace(stream=int(aug.stream)), **kw)
        tol = 1e-5 if layout == "nchw_fp32" else 2e-2
        torch.testing.assert_close(out.float().cpu(), cpu.float(), atol=tol, rtol=tol)


def test_draw_distribution():
    """(oy, ox) is uniform over the 81 cells of --crop_pad 4 and the flip rate is 1/2, read back from the kernel itself: a float image
    whose pixel (h, w) stores h*W + w + 1 reveals the source pixel of every output pixel."""
    from scipy.stats import chi2
    N, H, W, P = 16200, 28, 28, 4
    img = (torch.arange(H * W, dtype=torch.float32) + 1).reshape(1, H, W, 1).to(DEV)
    aug = _aug(P, True, seed=11, stream=ops.augment_stream(11, 0, 1, 0))
    out = ops.gather_normalize(img, torch.zeros(N, dtype=torch.int64, device=DEV), (0.0,), (1.0,), augment=aug)[:, 0].cpu()
    a, b = out[:, 14, 14].long() - 1, out[:, 14, 15].long() - 1            # interior pixels: never crop padding at P = 4
    flip = (b - a == -1).long()
    assert bool(((b - a).abs() == 1).all())
    oy = a // W - 14 + P
    ox = a % W - torch.where(flip.bool(), W - 1 - 14, 14) + P
    eoy, eox, efl = ops.augment_draws(aug._replace(stream=int(aug.stream)), np.arange(N))
    assert torch.equal(oy, eoy) and torch.equal(ox, eox) and torch.equal(flip, efl)
    counts = torch.bincount(oy * (2 * P + 1) + ox, minlength=81).double()
    stat = float(((counts - N / 81) ** 2 / (N / 81)).sum())
    assert chi2.sf(stat, 80) > 1e-4, stat
    assert abs(int(flip.sum()) - N / 2) < 4.5 * (N ** 0.5) / 2


def _engine(trainer, **kw):
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    base = dict(data="cifar10", model="resnet18", num_agents=2, local_ep=2, bs=64, synthetic=300, synthetic_val=64, log_dir="",
                device=DEV, seed=5, crop_pad=4, hflip=True, trainer=trainer, agents_in_flight=1)
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def _expected_last_batch_im2col(eng, agent, rnd, k, pad, stream_ep=None):
    """im2col rows of the last step of (agent, rnd): positions from the last batch start of the last epoch, drawn under that epoch's
    stream word (or epoch ``stream_ep``'s), assembled from host-augmented images by the un-augmented kernel."""
    args, n, bs = eng.args, agent.n_data, eng.args.bs
    ep = args.local_ep - 1
    stream_ep = ep if stream_ep is None else stream_ep
    start = ((n - 1) // bs) * bs
    idx = agent.epoch_indices(args.seed, rnd, ep).to(DEV)
    sel = idx[start:n]
    B = n - start
    aug = _aug(args.crop_pad, args.hflip, seed=args.seed, stream=ops.augment_stream(args.seed, agent.id, rnd, stream_ep))
    host = _host_augmented(agent.dataset.data, sel, start, aug).to(DEV)
    H, W = host.shape[1:3]
    Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
    ref = torch.zeros(B * Ho * Wo, 64, dtype=torch.bfloat16, device=DEV)
    meta = agent.dataset.meta
    ops.gather_im2col(host, torch.arange(B, device=DEV), meta.mean, meta.std, k, pad, ref, batch=B)
    return ref, B, agent.dataset.targets[sel]


def test_native_and_torch_trainers_assemble_the_same_augmented_batches():
    """Each trainer's last step of the round (graph replays: the cursor advanced every step, the stream word was rewritten for the
    second epoch) holds exactly the batch the host draws predict; the torch trainer's NCHW fp32 batch, im2col'ed and rounded to
    bf16, is the native trainer's stem operand."""
    nat, tor = _engine("native"), _engine("torch")
    assert nat.trainer.name == "native" and tor.trainer.name == "torch" and nat.trainer.use_graphs and tor.trainer.use_graphs
    nat.run_round(1)
    tor.run_round(1)
    torch.cuda.synchronize()
    k, pad, Ho, Wo = nat.trainer.stem
    expected = [_expected_last_batch_im2col(nat, a, 1, k, pad) for a in nat.agents]
    hits = [i for i, (ref, B, _) in enumerate(expected) if torch.equal(nat.trainer.xA[:B * Ho * Wo], ref)]
    assert len(hits) == 1, hits                                   # the last agent the (single) trainer trained
    agent = nat.agents[hits[0]]
    ref, B, labels = expected[hits[0]]
    got = nat.trainer.xA[:B * Ho * Wo]
    assert torch.equal(nat.trainer.y[:B], labels)
    # under the first epoch's stream word the same positions crop differently: the word is rewritten per epoch
    assert not torch.equal(got, _expected_last_batch_im2col(nat, agent, 1, k, pad, stream_ep=0)[0])
    x = tor.trainer.x[:B].float()                                                      # NCHW fp32
    cols = torch.nn.functional.unfold(x, k, padding=pad)
    C = x.shape[1]
    tor_rows = cols.reshape(B, C, k * k, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, k * k * C).to(torch.bfloat16)
    assert torch.equal(tor_rows, got[:, :k * k * C])
    nat.close(); tor.close()


def test_agents_in_flight_keep_each_agents_augmentation():
    """--agents_in_flight 2: every trainer's last batch is the one its agent draws when trained alone."""
    eng = _engine("native", num_agents=4, agents_in_flight=2, local_ep=1)
    assert len(eng.trainers) == 2
    eng.run_round(1)
    torch.cuda.synchronize()
    k, pad, Ho, Wo = eng.trainer.stem
    expected = [_expected_last_batch_im2col(eng, a, 1, k, pad) for a in eng.agents]
    matched = set()
    for t in eng.trainers:
        hits = [i for i, (ref, B, _) in enumerate(expected) if torch.equal(t.xA[:B * Ho * Wo], ref)]
        assert len(hits) == 1, hits
        matched.add(hits[0])
    assert len(matched) == 2
    eng.close()


def test_native_runs_with_augmentation_are_bitwise_reproducible():
    def run():
        ops.reset_fallbacks()
        eng = _engine("native")
        eng.run_round(1)
        eng.run_round(2)
        w = eng.global_params().clone()
        torch.cuda.synchronize()
        assert ops.fallback_calls() == {}, ops.fallback_calls()
        eng.close()
        return w
    a, b = run(), run()
    assert torch.equal(a, b)
    assert torch.isfinite(a).all()
