"""Differential tests against the reference's own client / evaluation code (src/agent.py, src/utils.py:128-157), on CPU.

The reference outputs are stored (tests/golden/reference_outputs.pt, written by scripts/make_reference_golden.py): its Agent was
driven with a tiny in-memory dataset whose ``__getitem__`` returns exactly the normalised tensors our gather kernel's oracle
produces; dropout is disabled (p=0) on both sides and the batch is the whole shard, so one local step is deterministic and the update
vectors must agree coordinate by coordinate (after mapping our OHWI / NHWC-flatten layout to the reference's ``parameters_to_vector``
order; a fixed, seeded sample of the coordinates is stored)."""
import os
import sys
from types import SimpleNamespace

import numpy as np

import pytest
import torch

from rlr_b200.data import make_synthetic
from rlr_b200.models import get_layout, GraphNet
from rlr_b200.options import make_args
from rlr_b200.trainers import TorchTrainer
from rlr_b200.utils import get_loss_n_accuracy


class _RefView(torch.utils.data.Dataset):
    """What the reference expects from a torchvision dataset: ``targets`` + normalised (C,H,W) tensors from __getitem__."""

    def __init__(self, ds):
        self.ds = ds
        self.targets = ds.targets.clone()

    def __len__(self):
        return len(self.ds)

    def __getitem__(self, i):
        x, y = self.ds.batch(torch.tensor([i]))
        return x[0], int(y[0])


LOCAL_TRAIN_CASES = [("fmnist", 0.0), ("cifar10", 0.0), ("fmnist", 0.02)]


def local_train_init(lay):
    """Global parameters the local step starts from (loaded into the reference model through to_reference_vector)."""
    return lay.init_(torch.zeros(lay.n_total), 11)


@pytest.mark.parametrize("data,clip", LOCAL_TRAIN_CASES)
def test_local_train_update_matches_reference_agent(reference_outputs, data, clip):
    n = 48
    train, _ = make_synthetic(data, n, 16, seed=4)
    args = make_args(data=data, num_agents=1, local_ep=1, bs=n, clip=clip, log_dir="", device="cpu")
    lay = get_layout(args.model)
    for nd in lay.nodes:
        if nd.op == "dropout":
            nd.attrs["p"] = 0.0
    w_global = local_train_init(lay)
    trainer = TorchTrainer(lay, args, "cpu", n)
    agent = SimpleNamespace(id=0, dataset=train, n_data=n, idxs=torch.arange(n),
                            epoch_indices=lambda seed, rnd, ep: torch.arange(n))
    out = torch.zeros(lay.n_total)
    trainer.train_agent(agent, w_global, out, rnd=1)
    ours = lay.to_reference_vector(out) - lay.to_reference_vector(w_global)
    # the reference Agent's local_train (fp64: local - global) at a fixed, seeded sample of the coordinates
    ref_update = reference_outputs[f"local_train/{data}/{clip}"]
    idx = torch.from_numpy(np.sort(np.random.default_rng(0).choice(ours.numel(), size=min(ours.numel(), ref_update.numel()), replace=False)))
    torch.testing.assert_close(ours.double()[idx], ref_update, atol=2e-6, rtol=1e-4)
    assert abs(float(ours.norm()) - reference_outputs[f"local_train/{data}/{clip}/norm"]) <= 1e-4 * reference_outputs[f"local_train/{data}/{clip}/norm"] + 2e-6
    if clip > 0:
        assert float(ours.norm()) <= clip * (1 + 1e-4)


def test_evaluation_matches_reference_function(reference_outputs):
    _, val = make_synthetic("cifar10", 64, 90, seed=7)
    lay = get_layout("cnn_cifar")
    w = lay.init_(torch.zeros(lay.n_total), 5)
    net = GraphNet(lay, w, None).eval()
    ref = reference_outputs["evaluation"]        # the reference's get_loss_n_accuracy on the same weights and images (batch 32)
    loss, (acc, pc) = get_loss_n_accuracy(lambda x: net(x), val, bs=32)
    assert abs(loss - ref["loss"]) < 1e-4 and abs(acc - ref["acc"]) < 1e-9
    torch.testing.assert_close(pc, ref["per_class"], atol=1e-6, rtol=1e-6, equal_nan=True)


class _H5Dataset(torch.utils.data.Dataset):
    """The reference's Fed-EMNIST file format: a pickled ``utils.H5Dataset`` object holding ``targets`` (int64 [n]) and ``inputs``
    (float32 [n, 1, 28, 28]); ``a + b`` concatenates into ``a``."""

    def __init__(self, raw, client_id):
        self.targets = torch.LongTensor(raw[client_id]["label"])
        px = torch.Tensor(raw[client_id]["pixels"])
        self.inputs = px.view(px.shape[0], 1, px.shape[1], px.shape[2])

    def __add__(self, other):
        self.targets = torch.cat((self.targets, other.targets), 0)
        self.inputs = torch.cat((self.inputs, other.inputs), 0)
        return self


def _write_fedemnist_tree(root, n_clients=6, per_client=40, seed=0):
    """Files in the layout the reference reads (src/utils.py:105-109, src/agent.py:17), pickled as ``utils.H5Dataset`` objects built
    from the h5-style ``{client: {'label', 'pixels'}}`` mapping."""
    import types
    rs = np.random.RandomState(seed)
    os.makedirs(os.path.join(root, "Fed_EMNIST", "user_trainsets"))
    raw = {f"c{i}": {"label": rs.randint(0, 10, per_client + i), "pixels": rs.rand(per_client + i, 28, 28).astype("float32")}
           for i in range(n_clients + 1)}
    shim = types.ModuleType("utils")
    shim.H5Dataset = _H5Dataset
    saved = sys.modules.get("utils"), _H5Dataset.__module__, _H5Dataset.__qualname__
    sys.modules["utils"] = shim                                   # pickled by reference as utils.H5Dataset
    _H5Dataset.__module__, _H5Dataset.__qualname__ = "utils", "H5Dataset"
    try:
        for i in range(n_clients):
            torch.save(_H5Dataset(raw, f"c{i}"), os.path.join(root, "Fed_EMNIST", "user_trainsets", f"user_{i}_trainset.pt"))
        allset = _H5Dataset(raw, "c0")
        for i in range(1, n_clients):
            allset = allset + _H5Dataset(raw, f"c{i}")
        torch.save(allset, os.path.join(root, "Fed_EMNIST", "fed_emnist_all_trainset.pt"))
        torch.save(_H5Dataset(raw, f"c{n_clients}"), os.path.join(root, "Fed_EMNIST", "fed_emnist_all_valset.pt"))
    finally:
        _H5Dataset.__module__, _H5Dataset.__qualname__ = saved[1], saved[2]
        if saved[0] is None:
            del sys.modules["utils"]
        else:
            sys.modules["utils"] = saved[0]
    return raw


def test_fedemnist_files_written_by_the_reference_class_load_and_train(tmp_path):
    """Real-data Fed-EMNIST path: per-client ``.pt`` files holding pickled reference ``H5Dataset`` objects are read, the clients
    become index ranges of one device dataset (sizes and pixels preserved), corrupt clients are poisoned, a round trains."""
    import os as _os
    from rlr_b200.engine import FLEngine
    raw = _write_fedemnist_tree(str(tmp_path))
    args = make_args(data="fedemnist", data_dir=str(tmp_path), num_agents=6, agent_frac=0.5, num_corrupt=1, poison_frac=0.5,
                     pattern_type="plus", local_ep=1, bs=16, rounds=1, log_dir="", device="cpu", seed=3)
    eng = FLEngine(args, verbose=False)
    assert [a.n_data for a in eng.agents] == [40 + i for i in range(6)] and eng.n_part == 3
    assert len(eng.val_dataset) == 46 and eng.val_dataset.data.dtype == torch.float32
    a3 = eng.agents[3]
    got = eng.train_dataset.data[a3.idxs].reshape(-1, 28, 28)
    assert torch.equal(got, torch.as_tensor(raw["c3"]["pixels"]))             # honest client: pixels untouched, NHWC view
    assert torch.equal(eng.train_dataset.targets[a3.idxs], torch.as_tensor(raw["c3"]["label"]).long())
    n_base = int((torch.as_tensor(raw["c0"]["label"]) == args.base_class).sum())
    assert len(eng.agents[0].poisoned_idxs) == n_base // 2                    # floor(poison_frac * |base class in shard|)
    info = eng.run_round(1)
    assert len(info["chosen"]) == 3
    ev = eng.evaluate(1)
    assert ev["val_loss"] == ev["val_loss"]
    eng.close()


def test_fedemnist_cli_without_the_reference_on_the_path(tmp_path):
    """Same files through ``python federated.py`` in a fresh interpreter, where pickle's ``utils.H5Dataset`` must resolve to our
    shim class (the reference's modules are not importable there)."""
    import subprocess
    _write_fedemnist_tree(str(tmp_path))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "federated.py", "--data=fedemnist", f"--data_dir={tmp_path}", "--num_agents=6", "--agent_frac=0.5",
                        "--num_corrupt=1", "--poison_frac=0.5", "--local_ep=1", "--bs=16", "--rounds=2", "--snap=1", "--device=cpu",
                        "--log_dir=", "--no_tensorboard"], cwd=root, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""),
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "| Val_Loss/Val_Acc:" in r.stdout and "Training has finished!" in r.stdout
