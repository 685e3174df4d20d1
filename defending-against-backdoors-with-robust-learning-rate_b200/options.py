"""Command-line interface.

Same flag names, types and defaults as the reference (src/options.py:4-74) so existing command lines
(src/runner.sh:12-38) keep working, plus engine flags that have no reference counterpart
(``--model --dtype --backend --synthetic --seed --checkpoint ...``).  ``finalize_args`` applies the
reference's post-parse fix-up ``server_lr = server_lr if aggr == 'sign' else 1.0`` (src/federated.py:23) to the plain
sgd server step; with ``--server_opt`` other than sgd, ``--server_lr`` is the optimizer's step size for every aggregator.
"""
from __future__ import annotations

import argparse
import math

import torch

DATASETS = ("fmnist", "fedemnist", "cifar10")
AGGREGATORS = ("avg", "comed", "sign", "fltrust", "rfa", "flame")
ROOT_SIZE = 100                  # FLTrust root set: the paper's 100 clean samples
RFA_ITERS = 3                    # RFA: a few smoothed Weiszfeld passes per round
RFA_NU = 1e-6                    # RFA smoothing: distances below nu count as nu
FLAME_LAMBDA = 1e-3              # FLAME noise factor: the paper's value for image classification
SERVER_OPTS = ("sgd", "momentum", "adagrad", "adam", "yogi")
SELECTIONS = ("none", "krum", "multikrum")
PATTERNS = ("plus", "square", "copyright", "apple")
MODELS = ("auto", "cnn_mnist", "cnn_cifar", "resnet18", "resnet34", "vgg11", "vgg16", "resnet18_gn", "resnet34_gn", "vgg11_gn", "vgg16_gn")


def _default_device():
    return "cuda:0" if torch.cuda.is_available() else "cpu"


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(
        description="Federated learning with the Robust Learning Rate backdoor defense (H100-native engine)")
    # ---- reference flags (names/defaults: src/options.py:7-70) ----
    p.add_argument("--data", type=str, default="fmnist", help="dataset: fmnist | fedemnist | cifar10")
    p.add_argument("--num_agents", type=int, default=10, help="number of agents: K")
    p.add_argument("--agent_frac", type=float, default=1, help="fraction of agents per round: C")
    p.add_argument("--num_corrupt", type=int, default=0, help="number of corrupt agents (ids 0..n-1)")
    p.add_argument("--rounds", type=int, default=200, help="number of communication rounds: R")
    p.add_argument("--aggr", type=str, default="avg",
                   help="aggregation rule: avg | comed | sign | fltrust (trust-weighted mean against a server-trained root update) | "
                        "rfa (smoothed geometric median by Weiszfeld passes, Pillutla et al. 2022) | flame (cosine clustering, "
                        "median-norm clipping and adaptive noise, Nguyen et al. 2022)")
    p.add_argument("--local_ep", type=int, default=2, help="number of local epochs: E")
    p.add_argument("--bs", type=int, default=256, help="local batch size: B")
    p.add_argument("--client_lr", type=float, default=0.1, help="clients' learning rate")
    p.add_argument("--client_moment", type=float, default=0.9, help="clients' momentum")
    p.add_argument("--server_lr", type=float, default=1,
                   help="server learning rate (with --server_opt sgd only honoured for aggr=sign)")
    p.add_argument("--base_class", type=int, default=5, help="base class of the backdoor attack")
    p.add_argument("--target_class", type=int, default=7, help="target class of the backdoor attack")
    p.add_argument("--poison_frac", type=float, default=0.0, help="fraction of base-class samples a corrupt agent poisons")
    p.add_argument("--pattern_type", type=str, default="plus", help="trojan pattern: plus | square | copyright | apple")
    p.add_argument("--robustLR_threshold", type=int, default=0, help="RLR sign-vote threshold theta (0 = defense off)")
    p.add_argument("--clip", type=float, default=0, help="L2 ball radius for client PGD / noise scale (0 = off)")
    p.add_argument("--noise", type=float, default=0, help="server noise multiplier: std = noise*clip (0 = off)")
    p.add_argument("--top_frac", type=int, default=100, help="top-k Fisher coordinates in the sign-agreement diagnostic")
    p.add_argument("--snap", type=int, default=1, help="evaluate every `snap` rounds")
    p.add_argument("--device", default=_default_device(), help="device (single-process mode); ranks use cuda:LOCAL_RANK")
    p.add_argument("--num_workers", type=int, default=0, help="accepted for CLI compatibility; data is device-resident")
    # ---- engine flags (no reference counterpart) ----
    p.add_argument("--model", type=str, default="auto", choices=MODELS,
                   help="auto = reference mapping (fmnist/fedemnist->cnn_mnist, cifar10->cnn_cifar)")
    p.add_argument("--dtype", type=str, default="bf16", choices=("fp32", "bf16"),
                   help="activation/GEMM-operand dtype on GPU (master params, updates, aggregation stay fp32)")
    p.add_argument("--backend", type=str, default="auto", choices=("auto", "fused", "nccl", "gloo", "local"),
                   help="aggregation transport: fused = P2P/multicast sm_90a kernel; nccl/gloo = all_gather + kernel")
    p.add_argument("--agents_in_flight", type=int, default=0,
                   help="agents a GPU trains CONCURRENTLY when it hosts several per round (one trainer + CUDA stream each); helps the "
                        "small launch-bound CNNs, costs one set of activation buffers per extra agent.  0 = auto (2 for models under 4 M "
                        "parameters on a GPU, else 1)")
    p.add_argument("--no_fused_handoff", action="store_true",
                   help="keep the separate round_init pass and the aggregation kernel's barrier-out instead of fusing the parameter "
                        "hand-off of a round with the first local GEMM (native trainer; on by default)")
    p.add_argument("--agg_transport", type=str, default="auto", choices=("auto", "gather", "reduce"),
                   help="nccl/gloo back-ends only: gather = all_gather every participant's parameters (needed for comed); reduce = "
                        "all_reduce per-coordinate vote / weighted-sum partials (avg, sign, RLR: O(N) traffic per rank); "
                        "auto = reduce when the ranks span several hosts")
    p.add_argument("--trainer", type=str, default="auto", choices=("auto", "native", "torch"),
                   help="local-training executor: native = sm_90a kernels, torch = autograd oracle (CPU / baseline)")
    p.add_argument("--class_per_agent", type=int, default=10,
                   help="classes per agent in the partitioner (10 = IID like the reference's calls; fewer = label-skewed non-IID; "
                        "reference distribute_data parameter, src/utils.py:58)")
    p.add_argument("--synthetic", type=int, default=0, help=">0: use a synthetic dataset with this many training samples")
    p.add_argument("--synthetic_val", type=int, default=0, help="synthetic validation-set size (default train/5)")
    p.add_argument("--data_dir", type=str, default="../data", help="dataset root (reference: '../data', src/utils.py:98)")
    p.add_argument("--seed", type=int, default=0, help="seed for init / sampling / shuffling / dropout")
    p.add_argument("--log_dir", type=str, default="logs", help="TensorBoard/JSONL root (reference: 'logs/')")
    p.add_argument("--no_tensorboard", action="store_true", help="JSONL + stdout only")
    p.add_argument("--checkpoint", type=str, default="", help="checkpoint path (written every --ckpt_every rounds)")
    p.add_argument("--ckpt_every", type=int, default=0, help="0 = only at the end (if --checkpoint is set)")
    p.add_argument("--resume", type=str, default="", help="resume from this checkpoint")
    p.add_argument("--diagnostics", action="store_true",
                   help="enable the reference's disabled diagnostics (update norms, Fisher sign agreement)")
    p.add_argument("--server_clip", action="store_true",
                   help="clip each update to L2 norm --clip on the server (reference clip_updates, dead code there)")
    p.add_argument("--no_graphs", action="store_true", help="do not capture the local step in CUDA graphs")
    p.add_argument("--profile_phases", action="store_true", help="print per-phase CUDA-event timings every round")
    p.add_argument("--crop_pad", type=int, default=0,
                   help="training augmentation: pad each image by this many zero pixels and take a random crop of the image size "
                        "(torchvision RandomCrop(padding=P); the CIFAR-10 recipe is 4; 0 = off).  Local training only")
    p.add_argument("--hflip", action="store_true",
                   help="training augmentation: mirror each image left-right with probability 1/2 (local training only)")
    p.add_argument("--server_opt", type=str, default="sgd", choices=SERVER_OPTS,
                   help="server optimizer on the (RLR-signed) aggregate: sgd = w + server_lr * agg (reference); momentum = FedAvgM; "
                        "adagrad / adam / yogi = FedAdagrad / FedAdam / FedYogi (Reddi et al. 2021, no bias correction)")
    p.add_argument("--server_beta1", type=float, default=0.9, help="server optimizer first-moment decay, in [0, 1)")
    p.add_argument("--server_beta2", type=float, default=0.99, help="adam / yogi second-moment decay, in [0, 1)")
    p.add_argument("--server_tau", type=float, default=1e-3, help="adagrad / adam / yogi adaptivity tau > 0 (v starts at tau^2)")
    p.add_argument("--select", type=str, default="none", choices=SELECTIONS,
                   help="participant selection before the --aggr rule (Blanchard et al. 2017): krum admits the participant whose update "
                        "is closest to its K-F-2 nearest neighbours; multikrum the M best such scores.  Rejected participants take no "
                        "part in the round (vote, rule, BatchNorm mean, noise, server optimizer)")
    p.add_argument("--select_f", type=int, default=-1,
                   help="Byzantine participants the selection assumes (-1 = ceil(num_corrupt * K / num_agents), K participants per round)")
    p.add_argument("--select_m", type=int, default=0, help="participants multikrum admits (0 = K - F; krum admits 1)")
    p.add_argument("--root_size", type=int, default=None,
                   help=f"--aggr fltrust: clean training samples the server trains its root update on each round (default {ROOT_SIZE}); "
                        "drawn once from --seed, never a poisoned sample")
    p.add_argument("--rfa_iters", type=int, default=None,
                   help=f"--aggr rfa: smoothed Weiszfeld passes per round (default {RFA_ITERS}; 0 = the avg step).  Each pass reweights "
                        "every participant by its data size over its distance to the current weighted mean; a fixed count keeps the "
                        "cost per round fixed")
    p.add_argument("--rfa_nu", type=float, default=None,
                   help=f"--aggr rfa: smoothing nu > 0 of the Weiszfeld weights alpha_k / max(nu, d_k) (default {RFA_NU})")
    p.add_argument("--flame_lambda", type=float, default=None,
                   help=f"--aggr flame: noise factor lambda >= 0; the round's Gaussian noise has std lambda * S, S the median update norm "
                        f"the admitted updates are clipped to (default {FLAME_LAMBDA})")
    return p


def finalize_args(args: argparse.Namespace) -> argparse.Namespace:
    """Post-parse normalisation shared by the CLI and programmatic users."""
    # reference src/federated.py:23 -- server_lr is forced to 1 unless sign aggregation is used (plain sgd server step only)
    if getattr(args, "server_opt", "sgd") == "sgd":
        args.server_lr = args.server_lr if args.aggr == "sign" else 1.0
    if getattr(args, "server_opt", "sgd") not in SERVER_OPTS:
        raise ValueError(f"unknown --server_opt {args.server_opt!r}; expected one of {SERVER_OPTS}")
    for name in ("server_beta1", "server_beta2"):
        if not 0.0 <= getattr(args, name, 0.0) < 1.0:
            raise ValueError(f"--{name} {getattr(args, name)} must lie in [0, 1)")
    if not getattr(args, "server_tau", 1.0) > 0:
        raise ValueError(f"--server_tau {args.server_tau} must be > 0")
    if args.model == "auto":
        args.model = "cnn_cifar" if args.data == "cifar10" else "cnn_mnist"
    if args.aggr not in AGGREGATORS:
        # the reference silently aggregates to 0 (src/aggregation.py:26); we refuse instead
        raise ValueError(f"unknown --aggr {args.aggr!r}; expected one of {AGGREGATORS}")
    if args.data not in DATASETS:
        raise ValueError(f"unknown --data {args.data!r}; expected one of {DATASETS}")
    from .data.datasets import DATASET_META
    meta = DATASET_META[args.data]
    side = min(meta.height, meta.width)
    if not 0 <= args.crop_pad < side:
        raise ValueError(f"--crop_pad {args.crop_pad} must lie in [0, {side}) for --data {args.data} ({meta.height}x{meta.width} images)")
    _finalize_select(args)
    _finalize_fltrust(args)
    _finalize_rfa(args)
    _finalize_flame(args)
    return args


def _finalize_flame(args) -> None:
    """Validate the FLAME flags and resolve ``flame_lambda`` in place (``FLAME_LAMBDA`` by default under ``--aggr flame``)."""
    lam = getattr(args, "flame_lambda", None)
    if args.aggr != "flame":
        if lam is not None:
            raise ValueError("--flame_lambda needs --aggr flame")
        return
    lam = FLAME_LAMBDA if lam is None else lam
    if not (math.isfinite(lam) and lam >= 0):
        raise ValueError(f"--flame_lambda {lam} must be a finite number >= 0")
    if getattr(args, "server_clip", False):
        raise ValueError("--server_clip does not combine with --aggr flame, which clips every update to the round's median norm")
    if args.noise > 0:
        raise ValueError("--noise does not combine with --aggr flame, which adds noise of std --flame_lambda times the clip bound")
    # FLAME admits at least floor(K'/2) + 1 of the K' candidates whenever their norms are finite: the fewest voters it guarantees
    K = max(1, math.floor(args.num_agents * args.agent_frac))
    cand = args.select_m if getattr(args, "select", "none") != "none" else K
    if args.robustLR_threshold > cand // 2 + 1:
        raise ValueError(f"--robustLR_threshold {args.robustLR_threshold} > {cand // 2 + 1}, the fewest participants --aggr flame admits "
                         f"of {cand}, could flip every coordinate")
    args.flame_lambda = float(lam)


def _finalize_rfa(args) -> None:
    """Validate the RFA flags and resolve their defaults in place (``RFA_ITERS`` / ``RFA_NU`` under ``--aggr rfa``)."""
    iters, nu = getattr(args, "rfa_iters", None), getattr(args, "rfa_nu", None)
    if args.aggr != "rfa":
        if iters is not None or nu is not None:
            raise ValueError("--rfa_iters / --rfa_nu need --aggr rfa")
        return
    iters = RFA_ITERS if iters is None else iters
    nu = RFA_NU if nu is None else nu
    if int(iters) != iters or iters < 0:
        raise ValueError(f"--rfa_iters {iters} must be an integer >= 0")
    if not (nu > 0 and math.isfinite(nu)):
        raise ValueError(f"--rfa_nu {nu} must be a finite number > 0")
    args.rfa_iters, args.rfa_nu = int(iters), float(nu)


def _finalize_fltrust(args) -> None:
    """Validate the FLTrust flags and resolve ``root_size`` in place (``ROOT_SIZE`` by default under ``--aggr fltrust``)."""
    root_size = getattr(args, "root_size", None)
    if args.aggr != "fltrust":
        if root_size is not None:
            raise ValueError("--root_size needs --aggr fltrust")
        return
    if getattr(args, "server_clip", False):
        raise ValueError("--server_clip does not combine with --aggr fltrust, which rescales every update to the root update's norm")
    if root_size is None:
        root_size = ROOT_SIZE
    if root_size < 1:
        raise ValueError(f"--root_size {root_size} must be >= 1")
    args.root_size = int(root_size)


def _finalize_select(args) -> None:
    """Validate ``--select`` and resolve its defaults in place: ``select_f`` = F, ``select_m`` = M (1 for krum)."""
    select = getattr(args, "select", "none")
    if select not in SELECTIONS:
        raise ValueError(f"unknown --select {select!r}; expected one of {SELECTIONS}")
    if select == "none":
        if getattr(args, "select_f", -1) != -1 or getattr(args, "select_m", 0) != 0:
            raise ValueError("--select_f / --select_m need --select krum or multikrum")
        return
    K = max(1, math.floor(args.num_agents * args.agent_frac))
    f = args.select_f
    if f < -1:
        raise ValueError(f"--select_f {f} must be >= 0 (or -1 for the default)")
    if f == -1:
        f = math.ceil(args.num_corrupt * K / args.num_agents)
    if K < 2 * f + 3:
        raise ValueError(f"--select {select} needs K >= 2F + 3 participants per round (K={K}, F={f})")
    m = args.select_m
    if select == "krum":
        if m not in (0, 1):
            raise ValueError(f"--select krum admits one participant; --select_m {m} needs --select multikrum")
        m = 1
    elif m == 0:
        m = K - f
    if not 1 <= m <= K:
        raise ValueError(f"--select_m {m} must lie in [1, K={K}]")
    if args.robustLR_threshold > m:
        raise ValueError(f"--robustLR_threshold {args.robustLR_threshold} > {m} admitted participants would flip every coordinate")
    args.select_f, args.select_m = f, m


def args_parser(argv=None) -> argparse.Namespace:
    """Parse flags the way the reference's ``args_parser`` does (src/options.py:4)."""
    return build_parser().parse_args(argv)


def make_args(**overrides) -> argparse.Namespace:
    """Programmatic construction: defaults + overrides, already finalised."""
    args = build_parser().parse_args([])
    for k, v in overrides.items():
        if not hasattr(args, k):
            raise AttributeError(f"unknown option {k!r}")
        setattr(args, k, v)
    return finalize_args(args)


def print_exp_details(args) -> None:
    """Experiment banner; same 14 fields as reference src/utils.py:287-303 plus engine fields."""
    print("======================================")
    print(f"    Dataset: {args.data}")
    print(f"    Global Rounds: {args.rounds}")
    print(f"    Aggregation Function: {args.aggr}")
    print(f"    Number of agents: {args.num_agents}")
    print(f"    Fraction of agents: {args.agent_frac}")
    print(f"    Batch size: {args.bs}")
    print(f"    Client_LR: {args.client_lr}")
    print(f"    Server_LR: {args.server_lr}")
    print(f"    Client_Momentum: {args.client_moment}")
    print(f"    RobustLR_threshold: {args.robustLR_threshold}")
    print(f"    Noise Ratio: {args.noise}")
    print(f"    Number of corrupt agents: {args.num_corrupt}")
    print(f"    Poison Frac: {args.poison_frac}")
    print(f"    Clip: {args.clip}")
    print(f"    Model / dtype / trainer / backend: {args.model} / {args.dtype} / {args.trainer} / {args.backend}")
    print(f"    Crop pad / hflip: {args.crop_pad} / {args.hflip}")
    if getattr(args, "server_opt", "sgd") != "sgd":
        print(f"    Server optimizer (beta1 / beta2 / tau): {args.server_opt} ({args.server_beta1} / {args.server_beta2} / {args.server_tau})")
    if getattr(args, "select", "none") != "none":
        print(f"    Selection (F / M): {args.select} ({args.select_f} / {args.select_m})")
    if args.aggr == "fltrust":
        print(f"    Root set: {args.root_size}")
    if args.aggr == "rfa":
        print(f"    RFA passes / nu: {args.rfa_iters} / {args.rfa_nu}")
    if args.aggr == "flame":
        print(f"    FLAME lambda: {args.flame_lambda}")
    print("======================================")
