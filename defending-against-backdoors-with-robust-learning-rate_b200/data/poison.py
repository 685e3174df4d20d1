"""Backdoor poisoning: trojan patterns (incl. the Distributed Backdoor Attack) and label flipping.

Reference: ``poison_dataset`` src/utils.py:160-178 and ``add_pattern_bd`` src/utils.py:181-284; pixel
semantics tabulated in SURVEY.md 2.2.  A pattern is compiled once into a *pixel program*
(rows, cols, values, mode) and applied to all selected images of the device-resident dataset by one
kernel (``ops.stamp_pixels``) instead of the reference's per-image numpy loop.

Modes: ``set`` (pixel := value, all channels), ``add_wrap`` (uint8 wrap-around add: FMNIST copyright/apple,
src/utils.py:236,242 -- 10+255 -> 9), ``sub`` (float subtract value: Fed-EMNIST, src/utils.py:265,271).
"""
from __future__ import annotations

import random
from math import floor

import torch

from .. import ops
from ._stamps import STAMPS

MODE_SET, MODE_ADD_WRAP, MODE_SUB = 0, 1, 2


def pattern_pixels(dataset: str, pattern_type: str, agent_idx: int = -1):
    """Compile a pattern to ``(rows, cols, vals, mode)``; empty lists mean "no pixel changes"."""
    px = []
    mode = MODE_SET
    if dataset == "cifar10":
        # only `plus` stamps anything on CIFAR (src/utils.py:188-189; SURVEY.md quirk 10)
        if pattern_type == "plus":
            s, size = 5, 6
            vert = [(i, s) for i in range(s, s + size + 1)]                      # rows 5..11, col 5
            horiz = [(s + size // 2, j) for j in range(s - size // 2, s + size // 2 + 1)]  # row 8, cols 2..8
            if agent_idx == -1:
                sel = vert + horiz
            else:  # DBA: the plus is split over four attackers (src/utils.py:202-224)
                part = agent_idx % 4
                if part == 0:
                    sel = [(i, s) for i in range(s, s + size // 2 + 1)]          # rows 5..8
                elif part == 1:
                    sel = [(i, s) for i in range(s + size // 2 + 1, s + size + 1)]  # rows 9..11
                elif part == 2:
                    sel = [(s + size // 2, j) for j in range(s - size // 2, s + size // 4 + 1)]  # cols 2..6
                else:
                    sel = [(s + size // 2, j) for j in range(s - size // 4 + 1, s + size // 2 + 1)]  # cols 5..8
            px = [(r, c, 0) for r, c in sel]
    elif dataset in ("fmnist", "fedemnist"):
        fed = dataset == "fedemnist"
        on = 0 if fed else 255  # fedemnist images are inverted floats: the mark is black (0)
        if pattern_type == "square":
            px = [(i, j, on) for i in range(21, 26) for j in range(21, 26)]
        elif pattern_type == "plus":
            s, size = (8, 5) if fed else (5, 5)
            px = [(i, s, on) for i in range(s, s + size)]
            px += [(s + size // 2, j, on) for j in range(s - size // 2, s + size // 2 + 1)]
        elif pattern_type in ("copyright", "apple"):
            px = [(r, c, (v / 255.0) if fed else v) for r, c, v in STAMPS[pattern_type]]
            mode = MODE_SUB if fed else MODE_ADD_WRAP
    else:
        raise ValueError(f"unknown dataset {dataset!r}")
    # later writes win in the reference loops; de-duplicate keeping the last (matters for `plus` centre)
    dedup = {}
    for r, c, v in px:
        dedup[(r, c)] = v
    rows = [k[0] for k in dedup]
    cols = [k[1] for k in dedup]
    vals = [float(v) for v in dedup.values()]
    return rows, cols, vals, mode


def add_pattern_bd(x, dataset="cifar10", pattern_type="square", agent_idx=-1):
    """Stamp one image (reference ``add_pattern_bd`` signature, src/utils.py:181).  ``x``: HW / HWC tensor or
    array-like; returns a new tensor of the same dtype/shape."""
    t = torch.as_tensor(x).clone()
    squeeze = t.dim() == 2
    img = (t.unsqueeze(-1) if squeeze else t).unsqueeze(0).contiguous()
    rows, cols, vals, mode = pattern_pixels(dataset, pattern_type, agent_idx)
    ops.stamp_pixels(img, torch.zeros(1, dtype=torch.int64, device=img.device), rows, cols, vals, mode)
    out = img[0]
    return out[..., 0] if squeeze else out


def select_poison_idxs(dataset, base_class: int, poison_frac: float, data_idxs=None, rng: random.Random | None = None):
    """Indices to poison: ``floor(frac * |base-class ∩ shard|)`` samples (src/utils.py:161-166)."""
    all_idxs = (dataset.targets == base_class).nonzero().flatten().tolist()
    if data_idxs is not None:
        keep = set(int(i) for i in (data_idxs.tolist() if torch.is_tensor(data_idxs) else data_idxs))
        all_idxs = sorted(keep.intersection(all_idxs))
    rng = rng or random
    return rng.sample(all_idxs, floor(poison_frac * len(all_idxs)))


def poison_dataset(dataset, args, data_idxs=None, poison_all=False, agent_idx=-1, rng: random.Random | None = None,
                   clean_copy: list | None = None):
    """Poison ``dataset`` in place (reference ``poison_dataset``, src/utils.py:160-178): stamp the pattern on
    the chosen base-class images and relabel them ``target_class``.  Returns the poisoned indices.  With a ``clean_copy`` list (attack
    schedules), ``(indices, rows, labels)`` of the poisoned samples as they were before stamping are appended to it first."""
    frac = 1 if poison_all else args.poison_frac
    idxs = select_poison_idxs(dataset, args.base_class, frac, data_idxs, rng)
    if not idxs:
        return idxs
    rows, cols, vals, mode = pattern_pixels(args.data, args.pattern_type, agent_idx)
    sel = torch.as_tensor(idxs, dtype=torch.int64, device=dataset.device)
    if clean_copy is not None:
        clean_copy.append((sel, dataset.data[sel], dataset.targets[sel]))
    if rows:
        ops.stamp_pixels(dataset.data, sel, rows, cols, vals, mode)
    dataset.targets[sel] = args.target_class  # label flips even when no pixel changed (src/utils.py:177)
    return idxs


def make_poisoned_val(val_dataset, args):
    """Poisoned validation set (src/federated.py:42-45): every base-class validation image carries the
    *full* pattern (agent_idx=-1) and the target label; "poison accuracy" is accuracy on this set."""
    idxs = (val_dataset.targets == args.base_class).nonzero().flatten()
    sub = val_dataset.subset(idxs)
    poison_dataset(sub, args, None, poison_all=True, agent_idx=-1)
    return sub
