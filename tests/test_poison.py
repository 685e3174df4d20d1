"""Trojan patterns: pixel sets of SURVEY.md 2.2 + differential tests against the reference's add_pattern_bd /
poison_dataset (src/utils.py:160-284)."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from rlr_b200.data import add_pattern_bd, make_poisoned_val, make_synthetic, pattern_pixels, poison_dataset
from rlr_b200.options import make_args


def _changed(a, b):
    d = (torch.as_tensor(a).to(torch.int64) != torch.as_tensor(b).to(torch.int64))
    return {(int(r), int(c)) for r, c in d.reshape(d.shape[0], d.shape[1], -1).any(-1).nonzero().tolist()}


def test_cifar_plus_full_and_dba_parts():
    x = torch.full((32, 32, 3), 200, dtype=torch.uint8)
    full = {(i, 5) for i in range(5, 12)} | {(8, j) for j in range(2, 9)}
    assert _changed(x, add_pattern_bd(x, "cifar10", "plus", -1)) == full
    parts = [{(i, 5) for i in range(5, 9)}, {(i, 5) for i in range(9, 12)}, {(8, j) for j in range(2, 7)}, {(8, j) for j in range(5, 9)}]
    union = set()
    for a in range(8):
        got = _changed(x, add_pattern_bd(x, "cifar10", "plus", a))
        assert got == parts[a % 4]
        union |= got
    assert union == full, "the four DBA parts tile the full trigger"
    assert (add_pattern_bd(x, "cifar10", "plus", -1)[8, 5] == 0).all()


def test_cifar_other_patterns_change_no_pixels():
    x = torch.full((32, 32, 3), 17, dtype=torch.uint8)
    for pat in ["square", "copyright", "apple"]:
        assert torch.equal(add_pattern_bd(x, "cifar10", pat, -1), x)


def test_fmnist_patterns():
    x = torch.full((28, 28), 10, dtype=torch.uint8)
    sq = add_pattern_bd(x, "fmnist", "square")
    assert _changed(x, sq) == {(i, j) for i in range(21, 26) for j in range(21, 26)} and int(sq[22, 22]) == 255
    pl = add_pattern_bd(x, "fmnist", "plus")
    assert _changed(x, pl) == {(i, 5) for i in range(5, 10)} | {(7, j) for j in range(3, 8)}
    ap = add_pattern_bd(x, "fmnist", "apple")
    rows, cols, vals, mode = pattern_pixels("fmnist", "apple")
    assert mode == 1 and max(vals) == 255
    r, c = rows[vals.index(255.0)], cols[vals.index(255.0)]
    assert int(ap[r, c]) == 9, "uint8 wrap-around: 10 + 255 -> 9 (SURVEY.md quirk 11)"


def test_fedemnist_patterns():
    x = torch.full((28, 28), 0.8, dtype=torch.float32)
    pl = add_pattern_bd(x, "fedemnist", "plus")
    assert _changed((x * 100).int(), (pl * 100).int()) == {(i, 8) for i in range(8, 13)} | {(10, j) for j in range(6, 11)}
    cp = add_pattern_bd(x, "fedemnist", "copyright")
    rows, cols, vals, mode = pattern_pixels("fedemnist", "copyright")
    assert mode == 2
    assert abs(float(cp[rows[0], cols[0]]) - (0.8 - vals[0])) < 1e-6


PATTERN_CASES = [("cifar10", "plus", -1), ("cifar10", "plus", 0), ("cifar10", "plus", 1), ("cifar10", "plus", 2), ("cifar10", "plus", 3),
                 ("cifar10", "square", -1), ("fmnist", "plus", -1), ("fmnist", "square", -1), ("fmnist", "copyright", -1),
                 ("fmnist", "apple", -1), ("fedemnist", "plus", -1), ("fedemnist", "square", -1), ("fedemnist", "copyright", -1),
                 ("fedemnist", "apple", -1)]


def pattern_input(ds):
    g = torch.Generator().manual_seed(0)
    if ds == "cifar10":
        return torch.randint(0, 256, (32, 32, 3), generator=g, dtype=torch.uint8)
    if ds == "fmnist":
        return torch.randint(0, 256, (28, 28), generator=g, dtype=torch.uint8)
    return torch.rand(1, 28, 28, generator=g)


@pytest.mark.parametrize("ds,pat,agent", PATTERN_CASES)
def test_add_pattern_matches_reference(reference_outputs, ds, pat, agent):
    x = pattern_input(ds)
    ref = reference_outputs[f"pattern/{ds}/{pat}/{agent}"].numpy()     # the reference's add_pattern_bd on the same image
    ours = add_pattern_bd(x.squeeze(0) if ds == "fedemnist" else x, ds, pat, agent)
    if ds == "fedemnist":
        np.testing.assert_allclose(ours.numpy(), np.asarray(ref, dtype=np.float32), atol=1e-6)
    else:
        assert np.array_equal(ours.numpy(), np.asarray(ref))


def test_poison_dataset_counts_labels_and_locality():
    tr, va = make_synthetic("fmnist", 1000)
    args = make_args(data="fmnist", poison_frac=0.5, base_class=5, target_class=7)
    shard = list(range(0, 1000, 2))
    before = tr.clone()
    n_base = int(((tr.targets == 5) & (torch.arange(1000) % 2 == 0)).sum())
    idxs = poison_dataset(tr, args, shard, agent_idx=0)
    assert len(idxs) == n_base // 2 and set(idxs) <= set(shard)
    assert (tr.targets[idxs] == 7).all() and (before.targets[idxs] == 5).all()
    untouched = torch.ones(1000, dtype=torch.bool); untouched[idxs] = False
    assert torch.equal(tr.data[untouched], before.data[untouched]) and torch.equal(tr.targets[untouched], before.targets[untouched])
    assert (tr.data[idxs][:, 7, 5, 0] == 255).all()


def test_poisoned_val_is_all_base_class_with_full_pattern():
    _, va = make_synthetic("cifar10", 500, 300)
    args = make_args(data="cifar10", base_class=3, target_class=9)
    pv = make_poisoned_val(va, args)
    assert len(pv) == int((va.targets == 3).sum()) and (pv.targets == 9).all()
    assert (pv.data[:, 5:12, 5, :] == 0).all() and (pv.data[:, 8, 2:9, :] == 0).all()
    assert (va.targets == 3).sum() > 0 and not (va.data[va.targets == 3][:, 5:12, 5, :] == 0).all(), "original val set untouched"
