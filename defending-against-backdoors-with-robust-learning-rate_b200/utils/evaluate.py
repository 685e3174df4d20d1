"""Evaluation (reference ``get_loss_n_accuracy``, src/utils.py:128-157).

Same outputs -- sample-weighted mean loss, accuracy, per-class accuracy from a confusion matrix -- but loss sum and
confusion matrix are accumulated on the device by one kernel per batch (``ops.eval_metrics``) and read back once,
instead of the reference's ``.item()`` per batch and Python loop per sample (src/utils.py:144-152).
"""
from __future__ import annotations

import torch

from .. import ops


@torch.no_grad()
def get_loss_n_accuracy(forward, dataset, bs: int = 256, num_classes: int = 10, ctx=None, dtype=torch.float32,
                        channels_last: bool = False):
    """``forward(x) -> logits`` in eval mode; ``dataset`` a DeviceDataset.  Returns
    ``(avg_loss, (accuracy, per_class_accuracy))`` like the reference.  With a distributed ``ctx`` the batches are
    strided over ranks and the two accumulators are all-reduced."""
    dev = dataset.device
    n = len(dataset)
    loss_sum = torch.zeros(1, dtype=torch.float64, device=dev)
    confusion = torch.zeros(num_classes, num_classes, dtype=torch.int64, device=dev)
    rank, world = (ctx.rank, ctx.world) if ctx is not None else (0, 1)
    all_idx = torch.arange(n, device=dev)
    for bi, start in enumerate(range(0, n, bs)):
        if bi % world != rank:
            continue
        idx = all_idx[start:start + bs]
        x, y = dataset.batch(idx, dtype=dtype, channels_last=channels_last)
        logits = forward(x)
        ops.eval_metrics(logits, y, loss_sum, confusion)
    if ctx is not None and ctx.is_dist:
        ctx.all_reduce_sum(loss_sum)
        ctx.all_reduce_sum(confusion)
    conf = confusion.cpu().double()
    total = max(1, n)
    avg_loss = float(loss_sum.item()) / total
    accuracy = float(conf.diag().sum()) / total
    per_class = conf.diag() / conf.sum(1)  # NaN for absent classes, like the reference's 0/0
    return avg_loss, (accuracy, per_class.float())


def backdoor_lifespan(evals, last_attack: int, threshold: float):
    """Rounds the backdoor outlived the attack: ``r* - last_attack`` for the first evaluated round ``r* >= last_attack`` whose poison
    accuracy is below ``threshold``, or None if there is none.  ``evals``: ``(round, poison_acc)`` pairs in round order; the resolution
    is the evaluation interval (``--snap``)."""
    for rnd, acc in evals:
        if rnd >= last_attack and acc < threshold:
            return rnd - last_attack
    return None
