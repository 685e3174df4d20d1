"""Device-resident datasets.

The reference keeps datasets on the host and pushes every sample through PIL ``ToTensor``/``Normalize``
in ``DatasetSplit.__getitem__`` (src/utils.py:52-54, 101, 112-115) -- the part of its round that is
host-bound (SURVEY.md 3.3).  Here a dataset is two tensors living on the training device:

* ``data``     raw pixels, NHWC: uint8 ``[N,H,W,C]`` (fmnist, cifar10) or float32 in [0,1] (fedemnist,
               whose reference tensors are already floats, src/utils.py:13-16)
* ``targets``  int64 ``[N]``

and a batch is produced by one gather+normalise kernel (``ops.gather_normalize``) from a permutation
index, directly in the layout/dtype the first layer consumes.  Normalisation constants are the
reference's (src/utils.py:101, 114).
"""
from __future__ import annotations

import os
import sys
import types
from dataclasses import dataclass

import numpy as np
import torch

from .. import ops


@dataclass(frozen=True)
class DatasetMeta:
    height: int
    width: int
    channels: int
    n_classes: int
    mean: tuple
    std: tuple
    is_float: bool  # raw storage already float in [0,1] (fedemnist)
    n_train: int
    n_val: int


DATASET_META = {
    # mean/std: reference src/utils.py:101 (fmnist) and :114 (cifar10); fedemnist has no transform
    "fmnist": DatasetMeta(28, 28, 1, 10, (0.2860,), (0.3530,), False, 60000, 10000),
    "cifar10": DatasetMeta(32, 32, 3, 10, (0.4914, 0.4822, 0.4465), (0.2023, 0.1994, 0.2010), False, 50000, 10000),
    "fedemnist": DatasetMeta(28, 28, 1, 10, (0.0,), (1.0,), True, 0, 0),
}


class DeviceDataset:
    """A whole dataset as two device tensors (raw NHWC pixels + labels)."""

    def __init__(self, name: str, data: torch.Tensor, targets: torch.Tensor):
        meta = DATASET_META[name]
        if data.dim() == 3:  # [N,H,W] -> [N,H,W,1]
            data = data.unsqueeze(-1)
        assert data.dim() == 4 and data.shape[1:] == (meta.height, meta.width, meta.channels), data.shape
        assert data.dtype == (torch.float32 if meta.is_float else torch.uint8), data.dtype
        self.name = name
        self.meta = meta
        self.data = data.contiguous()
        self.targets = targets.to(torch.int64).contiguous()

    # -- container protocol -------------------------------------------------------------------
    def __len__(self):
        return self.targets.shape[0]

    @property
    def device(self):
        return self.data.device

    def to(self, device):
        self.data = self.data.to(device)
        self.targets = self.targets.to(device)
        return self

    def pin(self):
        """Host copy in pinned memory (used by the end-to-end path that streams shards every round)."""
        return self.data.cpu().pin_memory(), self.targets.cpu().pin_memory()

    def clone(self):
        return DeviceDataset(self.name, self.data.clone(), self.targets.clone())

    def subset(self, idxs):
        idxs = torch.as_tensor(idxs, dtype=torch.int64, device=self.device)
        return DeviceDataset(self.name, self.data[idxs], self.targets[idxs])

    def classes(self):
        return torch.unique(self.targets)

    # -- batches -------------------------------------------------------------------------------
    def batch(self, idxs: torch.Tensor, dtype=torch.float32, channels_last=False, augment=None):
        """Normalised batch for sample indices ``idxs``: ``(x, y)``; x is NCHW (or NHWC if channels_last).  ``augment``: an
        ``ops.Augment`` whose ``start`` is the epoch position of ``idxs[0]`` (training batches only)."""
        x = ops.gather_normalize(self.data, idxs, self.meta.mean, self.meta.std, dtype=dtype, nhwc=channels_last, augment=augment)
        return x, self.targets[idxs]

    def __getitem__(self, i):
        x, y = self.batch(torch.as_tensor([i], device=self.device))
        return x[0], y[0]


class DatasetSplit:
    """Index view over a DeviceDataset (reference ``DatasetSplit``, src/utils.py:39-54).

    ``idxs`` is kept as a device int64 tensor; ``targets`` is read live (the reference snapshots it before
    poisoning, SURVEY.md quirk 4 -- not preserved, nothing depends on it).
    """

    def __init__(self, dataset: DeviceDataset, idxs):
        self.dataset = dataset
        self.idxs = torch.as_tensor(list(idxs) if not torch.is_tensor(idxs) else idxs,
                                    dtype=torch.int64, device=dataset.device)

    @property
    def targets(self):
        return self.dataset.targets[self.idxs]

    def classes(self):
        return torch.unique(self.targets)

    def __len__(self):
        return int(self.idxs.shape[0])

    def __getitem__(self, item):
        return self.dataset[int(self.idxs[item])]


class H5Dataset:
    """Fed-EMNIST per-client container (reference ``H5Dataset``, src/utils.py:11-36).

    Built from a ``{client_id: {'label':..., 'pixels':...}}`` mapping; supports ``+`` (concatenate clients)
    and ``.to(device)`` like the reference.  ``as_device_dataset`` converts to the engine's representation.
    """

    def __init__(self, dataset=None, client_id=None):
        if dataset is None:
            self.targets = torch.zeros(0, dtype=torch.int64)
            self.inputs = torch.zeros(0, 1, 28, 28)
            return
        self.targets = torch.as_tensor(np.asarray(dataset[client_id]["label"]), dtype=torch.int64)
        x = torch.as_tensor(np.asarray(dataset[client_id]["pixels"]), dtype=torch.float32)
        self.inputs = x.view(x.shape[0], 1, x.shape[1], x.shape[2])

    def classes(self):
        return torch.unique(self.targets)

    def __add__(self, other):
        self.targets = torch.cat((self.targets, other.targets), 0)
        self.inputs = torch.cat((self.inputs, other.inputs), 0)
        return self

    def to(self, device):
        self.targets = self.targets.to(device)
        self.inputs = self.inputs.to(device)
        return self

    def __len__(self):
        return self.targets.shape[0]

    def __getitem__(self, item):
        return self.inputs[item], self.targets[item]

    def as_device_dataset(self, device="cpu") -> DeviceDataset:
        return h5_to_device_dataset(self, device)


def h5_to_device_dataset(obj, device="cpu") -> DeviceDataset:
    """Engine representation of any Fed-EMNIST container with ``inputs`` [N,1,28,28] float and ``targets`` -- ours or an
    unpickled instance of the reference's own ``utils.H5Dataset`` (when that module is importable, pickle resolves to it)."""
    n = int(obj.targets.shape[0])
    x = torch.as_tensor(obj.inputs).to(torch.float32).reshape(n, 28, 28, 1)
    return DeviceDataset("fedemnist", x.to(device), torch.as_tensor(obj.targets).to(torch.int64).to(device))


def _install_unpickle_shim():
    """The reference's Fed-EMNIST ``.pt`` files pickle ``utils.H5Dataset`` objects (src/utils.py:108-109,
    src/agent.py:17); give the unpickler a ``utils`` module that resolves to our class."""
    if "utils" not in sys.modules:
        shim = types.ModuleType("utils")
        shim.H5Dataset = H5Dataset
        sys.modules["utils"] = shim
    elif not hasattr(sys.modules["utils"], "H5Dataset"):
        sys.modules["utils"].H5Dataset = H5Dataset


def load_fedemnist_client(data_dir: str, client_id: int) -> H5Dataset:
    """Per-client shard, path layout of reference src/agent.py:17."""
    _install_unpickle_shim()
    return torch.load(os.path.join(data_dir, "Fed_EMNIST", "user_trainsets", f"user_{client_id}_trainset.pt"),
                      weights_only=False)


def make_synthetic(name: str, n_train: int, n_val: int | None = None, seed: int = 0, device="cpu"):
    """Learnable synthetic stand-in with the named dataset's shape/dtype (no datasets exist offline).

    Each class is a fixed random low-frequency prototype; samples are prototype + pixel noise, so a CNN
    separates classes quickly and a stamped trojan is learnable.  Labels are balanced (n/10 per class) like
    FMNIST/CIFAR-10, which the reference partitioner implicitly assumes (src/utils.py:72-74).
    """
    meta = DATASET_META[name]
    n_val = n_val if n_val else max(meta.n_classes * 8, n_train // 5)
    g = torch.Generator().manual_seed(1234567 + seed)
    h, w, c = meta.height, meta.width, meta.channels
    coarse = torch.rand(meta.n_classes, c, 7, 7, generator=g)
    protos = torch.nn.functional.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=False)
    protos = protos.permute(0, 2, 3, 1).contiguous()  # [K,H,W,C] in [0,1]

    def draw(n):
        y = torch.arange(n) % meta.n_classes
        y = y[torch.randperm(n, generator=g)]
        x = protos[y] * 0.6 + 0.2 + 0.15 * torch.randn(n, h, w, c, generator=g)
        x = x.clamp_(0, 1)
        if not meta.is_float:
            x = (x * 255).round().to(torch.uint8)
        return DeviceDataset(name, x.to(device), y.to(device))

    return draw(n_train), draw(n_val)


def _read_idx(path: str) -> torch.Tensor:
    """IDX file (the FashionMNIST / MNIST raw format; ``.gz`` accepted): magic 0x0000 08 <ndim>, big-endian dims, uint8 payload."""
    import gzip
    import struct
    opener = gzip.open if path.endswith(".gz") else open
    with opener(path, "rb") as f:
        raw = f.read()
    zero, dtype, ndim = struct.unpack(">HBB", raw[:4])
    if zero != 0 or dtype != 0x08:
        raise ValueError(f"{path}: not a uint8 IDX file")
    dims = struct.unpack(">" + "I" * ndim, raw[4:4 + 4 * ndim])
    return torch.frombuffer(bytearray(raw[4 + 4 * ndim:]), dtype=torch.uint8).reshape(dims).clone()


def _first_existing(*paths):
    for p in paths:
        if os.path.exists(p):
            return p
    raise FileNotFoundError(" | ".join(paths))


def _load_torchvision(name: str, data_dir: str):
    """Read FashionMNIST / CIFAR-10 from torchvision's ON-DISK layout (what ``download=True`` of the reference leaves under
    ``../data``, src/utils.py:100-121) without torchvision's md5 checks or any download:
    ``<dir>/FashionMNIST/raw/{train,t10k}-{images-idx3,labels-idx1}-ubyte[.gz]`` and ``<dir>/cifar-10-batches-py/{data_batch_1..5,test_batch}``.
    Returns ((x_train uint8 NHWC / NHW, y_train int64), (x_val, y_val))."""
    if name == "fmnist":
        raw = os.path.join(data_dir, "FashionMNIST", "raw")
        out = []
        for split in ("train", "t10k"):
            x = _read_idx(_first_existing(os.path.join(raw, f"{split}-images-idx3-ubyte"), os.path.join(raw, f"{split}-images-idx3-ubyte.gz")))
            y = _read_idx(_first_existing(os.path.join(raw, f"{split}-labels-idx1-ubyte"), os.path.join(raw, f"{split}-labels-idx1-ubyte.gz")))
            out.append((x, y.long()))
        return out[0], out[1]
    import pickle
    base = os.path.join(data_dir, "cifar-10-batches-py")

    def batch(fn):
        with open(_first_existing(os.path.join(base, fn)), "rb") as f:
            d = pickle.load(f, encoding="latin1")
        x = torch.as_tensor(d["data"], dtype=torch.uint8).reshape(-1, 3, 32, 32).permute(0, 2, 3, 1).contiguous()   # HWC like torchvision
        return x, torch.as_tensor(d["labels"] if "labels" in d else d["fine_labels"], dtype=torch.int64)   # LongTensor (src/utils.py:122)
    tr = [batch(f"data_batch_{i}") for i in range(1, 6)]
    return (torch.cat([t[0] for t in tr]), torch.cat([t[1] for t in tr])), batch("test_batch")


def get_datasets(data: str, data_dir: str = "../data", synthetic: int = 0, synthetic_val: int = 0,
                 seed: int = 0, device="cpu"):
    """Train/validation datasets (reference ``get_datasets``, src/utils.py:95-124), device resident.

    Real data is read from ``data_dir`` in torchvision's on-disk layout *without* downloading (the
    reference downloads, src/utils.py:102-103; there is no network here).  ``synthetic>0`` -> synthetic data of
    the same shape; missing files raise (no silent substitution).
    """
    if data not in DATASET_META:
        raise ValueError(f"unknown dataset {data!r}")
    if synthetic > 0:
        return make_synthetic(data, synthetic, synthetic_val or None, seed, device)
    if data == "fedemnist":
        _install_unpickle_shim()
        tr = torch.load(os.path.join(data_dir, "Fed_EMNIST", "fed_emnist_all_trainset.pt"), weights_only=False)
        te = torch.load(os.path.join(data_dir, "Fed_EMNIST", "fed_emnist_all_valset.pt"), weights_only=False)
        return h5_to_device_dataset(tr, device), h5_to_device_dataset(te, device)
    try:
        (xtr, ytr), (xte, yte) = _load_torchvision(data, data_dir)
    except Exception as e:  # noqa: BLE001
        # never substitute synthetic data silently: accuracy / poison numbers of a run must not look like real-data results
        raise FileNotFoundError(
            f"{data} not readable under data_dir={data_dir!r} ({type(e).__name__}: {e}). There is no download here; put the torchvision "
            f"on-disk files there or pass --synthetic N (N > 0) to train on synthetic data of the same shape.") from e
    return (DeviceDataset(data, xtr.to(device), ytr.to(device)),
            DeviceDataset(data, xte.to(device), yte.to(device)))
