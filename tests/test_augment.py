"""Training augmentation (--crop_pad / --hflip) on CPU: the host Philox, the CPU statement of the augmented gathers against an
independent torch statement, option validation and engine-level reproducibility."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import rlr_b200  # noqa: F401
from rlr_b200 import ops
from rlr_b200.data import make_synthetic
from rlr_b200.engine import FLEngine
from rlr_b200.options import args_parser, finalize_args, make_args, print_exp_details


def test_philox_known_answers():
    """Random123 known-answer vectors of Philox4x32-10."""
    assert [int(w) for w in ops.philox4x32(0, 0, 0)] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    ones = 2 ** 64 - 1
    assert [int(w) for w in ops.philox4x32(ones, ones, ones)] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    # vectorised over counters = one call per counter
    u = ops.philox4x32(np.arange(5), 123, 456)
    for i in range(5):
        assert [int(w[i]) for w in u] == [int(w) for w in ops.philox4x32(i, 123, 456)]


def test_augment_stream_is_a_pure_function_of_agent_round_epoch():
    s = ops.augment_stream(3, 5, 7, 1)
    assert s == ops.augment_stream(3, 5, 7, 1) and 0 <= s < 2 ** 63
    others = {ops.augment_stream(*k) for k in [(4, 5, 7, 1), (3, 6, 7, 1), (3, 5, 8, 1), (3, 5, 7, 0)]}
    assert s not in others and len(others) == 4


def _aug(pad, flip, seed=9, stream=1234567, start=0):
    return ops.Augment(pad, flip, seed, torch.tensor([stream], dtype=torch.int64), start)


def _reference_batch(data, sel, positions, aug, mean, std):
    """Independent statement: F.pad(fill 0) + slice + flip of each raw image (NCHW), then ToTensor/Normalize arithmetic."""
    oy, ox, fl = ops.augment_draws(aug, positions)
    P = aug.pad
    H, W = data.shape[1], data.shape[2]
    imgs = []
    for b, s in enumerate(sel.tolist()):
        x = data[s].to(torch.float32).permute(2, 0, 1)                          # [C,H,W] raw
        x = F.pad(x, (P, P, P, P), value=0.0)[:, int(oy[b]):int(oy[b]) + H, int(ox[b]):int(ox[b]) + W]
        if int(fl[b]):
            x = x.flip(-1)
        imgs.append(x)
    x = torch.stack(imgs)
    if data.dtype == torch.uint8:
        x = x / 255.0
    m = torch.tensor(mean, dtype=torch.float32)[None, :, None, None]
    s_ = torch.tensor(std, dtype=torch.float32)[None, :, None, None]
    return (x - m) / s_


@pytest.mark.parametrize("name", ["fmnist", "cifar10", "fedemnist"])
@pytest.mark.parametrize("pad,flip", [(1, False), (1, True), (4, False), (4, True)])
def test_gather_normalize_augmented_matches_independent_statement(name, pad, flip):
    tr, _ = make_synthetic(name, 120)
    perm = torch.randperm(120, generator=torch.Generator().manual_seed(1))
    cur, B = 17, 29
    aug = _aug(pad, flip)
    ref = _reference_batch(tr.data, perm[cur:cur + B], cur + np.arange(B), aug, tr.meta.mean, tr.meta.std)
    out = ops.gather_normalize(tr.data, perm, tr.meta.mean, tr.meta.std, cursor=torch.tensor([cur], dtype=torch.int32), batch=B,
                               augment=aug)
    torch.testing.assert_close(out, ref)
    # NHWC channel-padded layout: same values
    nhwc = ops.gather_normalize(tr.data, perm, tr.meta.mean, tr.meta.std, nhwc=True, c_pad=8,
                                cursor=torch.tensor([cur], dtype=torch.int32), batch=B, augment=aug)
    C = tr.data.shape[3]
    torch.testing.assert_close(nhwc[..., :C].permute(0, 3, 1, 2), ref)
    assert float(nhwc[..., C:].abs().max()) == 0.0
    if pad:       # crop padding is the stored value 0 normalised, not 0
        mean0 = -torch.tensor(tr.meta.mean) / torch.tensor(tr.meta.std)
        oy, _, _ = ops.augment_draws(aug, cur + np.arange(B))
        b = int(torch.nonzero(oy < pad)[0])                                     # a sample whose crop reaches above the image
        torch.testing.assert_close(out[b, :, 0, :].mean(-1), mean0.float())


@pytest.mark.parametrize("name,k,pad", [("cifar10", 3, 1), ("cifar10", 3, 0), ("fmnist", 3, 0), ("fmnist", 5, 2), ("fedemnist", 3, 1)])
@pytest.mark.parametrize("cpad,flip", [(1, False), (4, True)])
def test_gather_im2col_augmented_matches_independent_statement(name, k, pad, cpad, flip):
    tr, _ = make_synthetic(name, 80)
    perm = torch.randperm(80, generator=torch.Generator().manual_seed(2))
    cur, B = 5, 13
    aug = _aug(cpad, flip, seed=2 ** 64 - 3)
    x = _reference_batch(tr.data, perm[cur:cur + B], cur + np.arange(B), aug, tr.meta.mean, tr.meta.std)     # [B,C,H,W]
    C, H, W = x.shape[1:]
    Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
    cols = F.unfold(x, k, padding=pad)                                               # [B, C*k*k, L], (channel, tap) order
    ref = cols.reshape(B, C, k * k, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, k * k * C)
    out = torch.full((B * Ho * Wo, 64), 5.0)
    ops.gather_im2col(tr.data, perm, tr.meta.mean, tr.meta.std, k, pad, out, cursor=torch.tensor([cur], dtype=torch.int32), batch=B,
                      augment=aug)
    torch.testing.assert_close(out[:, :k * k * C], ref)
    assert float(out[:, k * k * C:].abs().max()) == 0.0


@pytest.mark.parametrize("name", ["fmnist", "cifar10"])
def test_augment_off_is_todays_output(name):
    """pad 0 without flip is the identity; the engine flags at their defaults give no Augment at all."""
    tr, _ = make_synthetic(name, 64)
    perm = torch.randperm(64)
    plain = ops.gather_normalize(tr.data, perm[:32], tr.meta.mean, tr.meta.std)
    off = ops.gather_normalize(tr.data, perm[:32], tr.meta.mean, tr.meta.std, augment=_aug(0, False))
    assert torch.equal(plain, off)
    assert ops.training_augment(make_args(), torch.zeros(1, dtype=torch.int64)) is None
    a = ops.training_augment(make_args(data="cifar10", crop_pad=4, hflip=True, seed=3), torch.zeros(1, dtype=torch.int64))
    assert (a.pad, a.flip, a.seed, a.start) == (4, True, 3, 0)


def test_eager_and_graph_positions_agree():
    """The eager path (a slice of the epoch order, explicit start) and the cursor path draw the same crops for the same positions."""
    tr, _ = make_synthetic("cifar10", 200)
    perm = torch.randperm(200)
    aug = _aug(4, True)
    for start, B in [(0, 64), (64, 64), (192, 8)]:
        via_cursor = ops.gather_normalize(tr.data, perm, tr.meta.mean, tr.meta.std, cursor=torch.tensor([start], dtype=torch.int32), batch=B,
                                          augment=aug)
        x, _ = tr.batch(perm[start:start + B], augment=aug._replace(start=start))
        assert torch.equal(via_cursor, x)


def test_draws_cover_the_crop_window():
    aug = _aug(4, True)
    oy, ox, fl = ops.augment_draws(aug, np.arange(20000))
    assert int(oy.min()) == 0 and int(oy.max()) == 8 and int(ox.min()) == 0 and int(ox.max()) == 8
    assert 0.48 < float(fl.float().mean()) < 0.52
    oy, ox, fl = ops.augment_draws(_aug(0, True), np.arange(100))
    assert int(oy.abs().max()) == 0 and int(ox.abs().max()) == 0


def test_options():
    a = args_parser([])
    assert a.crop_pad == 0 and a.hflip is False
    a = finalize_args(args_parser("--data cifar10 --crop_pad 4 --hflip".split()))
    assert a.crop_pad == 4 and a.hflip is True
    for line in ["--data cifar10 --crop_pad -1", "--data cifar10 --crop_pad 32", "--data fmnist --crop_pad 28", "--data fedemnist --crop_pad 40"]:
        with pytest.raises(ValueError):
            finalize_args(args_parser(line.split()))
    assert finalize_args(args_parser("--data fmnist --crop_pad 27".split())).crop_pad == 27
    assert finalize_args(args_parser("--data cifar10 --crop_pad 31".split())).crop_pad == 31


def test_print_exp_details_shows_augmentation(capsys):
    print_exp_details(make_args(data="cifar10", crop_pad=4, hflip=True))
    assert "Crop pad / hflip: 4 / True" in capsys.readouterr().out


def _run(**kw):
    base = dict(data="cifar10", model="cnn_cifar", synthetic=300, synthetic_val=60, num_agents=3, local_ep=2, bs=64, log_dir="",
                device="cpu", seed=4)
    base.update(kw)
    eng = FLEngine(make_args(**base), verbose=False)
    eng.run_round(1)
    w = eng.w_global.clone()
    eng.close()
    return w


def test_engine_runs_with_augmentation_are_reproducible():
    a = _run(crop_pad=4, hflip=True)
    b = _run(crop_pad=4, hflip=True)
    plain = _run()
    assert torch.equal(a, b)
    assert not torch.equal(a, plain)


def test_agents_in_flight_keeps_each_agents_augmentation():
    """The stream word depends on (seed, agent, round, epoch) only: spreading the agents over several trainers changes nothing."""
    kw = dict(model="resnet18", synthetic=120, num_agents=3, local_ep=1, bs=16, crop_pad=2, hflip=True)
    assert torch.equal(_run(agents_in_flight=1, **kw), _run(agents_in_flight=3, **kw))
