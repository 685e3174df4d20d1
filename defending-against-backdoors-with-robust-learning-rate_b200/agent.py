"""Federated client (reference ``Agent``, src/agent.py:10-64).

An agent is a shard of the device-resident training set (an int64 index tensor) plus, for ``id < num_corrupt``, the
backdoor poisoning of that shard at construction (src/agent.py:19-25: CIFAR agents stamp their DBA part
``agent_idx = id``, FMNIST/Fed-EMNIST the full pattern).  Training itself is executed by a *trainer* that owns the
flat work buffers of its GPU (``trainers.TorchTrainer`` / ``models.native.NativeTrainer``), so K agents hosted on one
GPU share one set of buffers -- the reference shares one ``nn.Module`` the same way (src/federated.py:69-72).
"""
from __future__ import annotations

import random

import torch

from .data import DatasetSplit, poison_dataset
from .data.datasets import h5_to_device_dataset, load_fedemnist_client
from .options import attack_schedule_set


class Agent:
    def __init__(self, id, args, train_dataset=None, data_idxs=None, seed: int = 0):
        self.id = id
        self.args = args
        self.is_corrupt = id < args.num_corrupt
        self.poisoned_idxs = []
        # attack schedules: (indices, rows, labels) of the poisoned samples before poisoning, which the engine swaps in for quiet rounds
        self.clean_copy = [] if attack_schedule_set(args) else None
        rng = random.Random(1_000_003 * (seed + 1) + id)
        if train_dataset is None:
            # Fed-EMNIST: one pre-partitioned file per client (src/agent.py:16-20)
            shard = h5_to_device_dataset(load_fedemnist_client(args.data_dir, id), args.device)
            self.dataset = shard
            self.idxs = torch.arange(len(shard), device=shard.device)
            if self.is_corrupt:
                self.poisoned_idxs = poison_dataset(shard, args, None, agent_idx=id, rng=rng, clean_copy=self.clean_copy)
        else:
            self.dataset = train_dataset
            self.idxs = torch.as_tensor(list(data_idxs), dtype=torch.int64, device=train_dataset.device)
            if self.is_corrupt:
                # poisons the SHARED dataset in place at this agent's indices (src/agent.py:24-25)
                self.poisoned_idxs = poison_dataset(train_dataset, args, self.idxs, agent_idx=id, rng=rng, clean_copy=self.clean_copy)
        self.n_data = int(self.idxs.shape[0])
        self._gen = None

    @property
    def train_dataset(self):
        return DatasetSplit(self.dataset, self.idxs)

    def epoch_indices(self, seed_base: int, rnd: int, epoch: int):
        """Shuffled sample indices of one local epoch (DataLoader(shuffle=True), src/agent.py:28), seeded."""
        dev = self.idxs.device
        if self._gen is None:
            self._gen = torch.Generator(device=dev)
        self._gen.manual_seed((seed_base * 1_000_003 + self.id) * 1_000_003 + rnd * 131 + epoch)
        perm = torch.randperm(self.n_data, device=dev, generator=self._gen)
        return self.idxs[perm]

    def local_train(self, trainer, w_global, out, rnd: int = 0):
        """Train on the round's global parameters; write this agent's resulting parameters to ``out`` (the update
        ``out - w_global`` is formed inside the aggregation kernel).  Returns the trainer's stats dict."""
        return trainer.train_agent(self, w_global, out, rnd)
