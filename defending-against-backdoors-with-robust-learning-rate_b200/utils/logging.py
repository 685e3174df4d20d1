"""Metrics: TensorBoard scalars with the reference's tag names and run-directory naming
(src/federated.py:27-31, 81-91), the reference's stdout lines (:83-84, 92), plus a JSONL record per round with
device-timed phase durations and the fraction of coordinates whose learning rate was flipped."""
from __future__ import annotations

import json
import os
from time import ctime


def run_name(args) -> str:
    """Same fields as the reference's log directory name (src/federated.py:27-30)."""
    return (f"time:{ctime()}-clip_val:{args.clip}-noise_std:{args.noise}"
            f"-aggr:{args.aggr}-s_lr:{args.server_lr}-num_cor:{args.num_corrupt}"
            f"thrs_robustLR:{args.robustLR_threshold}"
            f"-num_corrupt:{args.num_corrupt}-pttrn:{args.pattern_type}")


class MetricLogger:
    def __init__(self, args, enabled: bool = True):
        self.enabled = enabled
        self.tb = None
        self.jsonl = None
        self.history = []
        if not enabled:
            return
        self.dir = os.path.join(args.log_dir, run_name(args).replace("/", "_"))
        os.makedirs(self.dir, exist_ok=True)
        self.jsonl = open(os.path.join(self.dir, "metrics.jsonl"), "a")
        if not getattr(args, "no_tensorboard", False):
            try:
                from torch.utils.tensorboard import SummaryWriter
                self.tb = SummaryWriter(self.dir)
            except Exception as e:  # noqa: BLE001
                print(f"[log] TensorBoard unavailable ({type(e).__name__}); JSONL only")

    def add_scalar(self, tag, value, step):
        if self.tb is not None:
            self.tb.add_scalar(tag, float(value), step)

    def record(self, rnd: int, **fields):
        rec = {"round": rnd, **{k: (float(v) if hasattr(v, "__float__") and not isinstance(v, bool) else v) for k, v in fields.items()}}
        self.history.append(rec)
        if self.jsonl is not None:
            self.jsonl.write(json.dumps(rec) + "\n")
            self.jsonl.flush()

    def close(self):
        if self.tb is not None:
            self.tb.close()
        if self.jsonl is not None:
            self.jsonl.close()
