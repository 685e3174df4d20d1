"""Checkpoint / resume (absent in the reference, SURVEY.md 5.4): flat global parameters + round + RNG state, plus the server
optimizer's hyper-parameters and full-length state when ``--server_opt`` is not sgd."""
from __future__ import annotations

import os
import random

import numpy as np
import torch


def save_checkpoint(path, w_global, rnd, args, layout, extra=None, server_opt=None):
    """``server_opt``: None (sgd: no key is written) or ``{"server_opt": kind, "beta1", "beta2", "tau", "m", "v"}`` with full-length
    fp32 state vectors."""
    tmp = path + ".tmp"
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    ck = {
        "w_global": w_global.detach().cpu(),
        "round": int(rnd),
        "args": {k: (str(v) if isinstance(v, torch.device) else v) for k, v in vars(args).items()},
        "model": getattr(layout, "name", ""),
        "n_params": layout.n_params, "n_vote": layout.n_vote, "n_total": layout.n_total,
        "rng": {"torch": torch.get_rng_state(), "numpy": np.random.get_state(), "python": random.getstate()},
        "extra": extra or {},
    }
    if server_opt is not None:
        ck["server_opt"] = {k: (v.detach().cpu() if isinstance(v, torch.Tensor) else v) for k, v in server_opt.items()}
    torch.save(ck, tmp)
    os.replace(tmp, path)


def load_checkpoint(path, w_global, layout, restore_rng=True):
    ck = torch.load(path, map_location="cpu", weights_only=False)
    if ck["n_total"] != layout.n_total or ck["n_params"] != layout.n_params:
        raise ValueError(f"checkpoint is for a different model ({ck.get('model')!r}: {ck['n_params']} params)")
    w_global.copy_(ck["w_global"].to(w_global.device))
    if restore_rng:
        torch.set_rng_state(ck["rng"]["torch"])
        np.random.set_state(ck["rng"]["numpy"])
        random.setstate(ck["rng"]["python"])
    return ck


def restore_server_opt(ck, fused):
    """Load a checkpoint's server optimizer state into ``fused`` (a ``parallel.FusedAggregator``; each rank takes its own slice, so
    the checkpoint resumes at any world size).  A missing state, another optimizer or other hyper-parameters are an error."""
    opt = fused.opt
    saved = ck.get("server_opt")
    if saved is None and opt.kind == "sgd":
        return
    if saved is None:
        raise ValueError(f"checkpoint has no server optimizer state, but this run uses --server_opt {opt.kind}")
    diff = [f"{k}: checkpoint {saved.get(k)!r}, run {v!r}" for k, v in opt.hparams.items() if saved.get(k) != v]
    if diff:
        raise ValueError("checkpoint server optimizer does not match this run (" + "; ".join(diff) + ")")
    fused.load_server_opt_state(saved["m"], saved["v"])
