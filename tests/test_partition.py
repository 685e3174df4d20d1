"""Partitioner: exactness + differential test against the reference's distribute_data (src/utils.py:58-92)."""
from types import SimpleNamespace

import pytest
import torch

from rlr_b200.data import distribute_data, make_synthetic


@pytest.mark.parametrize("K", [1, 2, 3, 4, 7, 8, 10, 40])
def test_partition_is_exact_and_disjoint(K):
    tr, _ = make_synthetic("fmnist", 6000)
    groups = distribute_data(tr, SimpleNamespace(num_agents=K))
    allidx = [i for u in range(K) for i in groups[u]]
    assert len(allidx) == len(set(allidx))
    assert len(allidx) == 6000, "balanced data: no sample dropped (SURVEY.md C9)"
    sizes = [len(groups[u]) for u in range(K)]
    assert max(sizes) - min(sizes) <= 10 * ((6000 // 10) // (6000 // (K * 10)) and 1) * 10
    if K > 1:
        for u in range(K):  # IID: every agent sees every class
            assert len(torch.unique(tr.targets[torch.as_tensor(list(groups[u]))])) == 10


@pytest.mark.parametrize("K,n", [(2, 1000), (7, 6000), (8, 5000), (10, 2000), (40, 4000)])
def test_matches_reference(reference_outputs, K, n):
    tr, _ = make_synthetic("cifar10", n)
    ours = distribute_data(tr, SimpleNamespace(num_agents=K))
    ref = reference_outputs[f"partition/{K}/{n}"]        # the reference's distribute_data on _Wrap(tr)
    for u in range(K):
        assert list(ours[u]) == ref[u].tolist()


def test_non_iid_class_per_agent():
    tr, _ = make_synthetic("fmnist", 4000)
    groups = distribute_data(tr, SimpleNamespace(num_agents=10), class_per_agent=2)
    for u in range(10):
        assert len(torch.unique(tr.targets[torch.as_tensor(list(groups[u]))])) <= 2


class _Wrap:
    """Minimal object with the two things the reference partitioner touches: len() and .targets."""

    def __init__(self, ds):
        self.targets = ds.targets

    def __len__(self):
        return len(self.targets)


def test_class_per_agent_flag_reaches_the_engine():
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    eng = FLEngine(make_args(data="fmnist", synthetic=2000, synthetic_val=100, num_agents=10, class_per_agent=2, log_dir="", device="cpu"),
                   verbose=False)
    for a in eng.agents:
        assert len(torch.unique(eng.train_dataset.targets[a.idxs])) <= 2
