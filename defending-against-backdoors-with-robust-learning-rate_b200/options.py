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
AGGREGATORS = ("avg", "comed", "sign", "fltrust", "rfa", "flame", "foolsgold", "flare", "deepsight")
ROOT_SIZE = 100                  # FLTrust / FLARE root set: the paper's 100 clean samples
FLARE_TAU = 1.0                  # FLARE: temperature of the softmax over the neighbour counts
RFA_ITERS = 3                    # RFA: a few smoothed Weiszfeld passes per round
RFA_NU = 1e-6                    # RFA smoothing: distances below nu count as nu
DEEPSIGHT_SAMPLES = 256          # DeepSight: random inputs per seed (this project's choice; the paper does not fix one)
DEEPSIGHT_TAU = 1.0 / 3.0        # DeepSight: a cluster is accepted when fewer than tau of its members are suspicious
FLAME_LAMBDA = 1e-3              # FLAME noise factor: the paper's value for image classification
LIFESPAN_THRESHOLD = 0.5         # poison accuracy below which the backdoor counts as gone
CERTIFY_N0 = 100                 # CRFL certification: selection draws (this project's choice, in the style of Cohen et al.)
CERTIFY_N = 1000                 # ... estimation draws (likewise)
CERTIFY_ALPHA = 1e-3             # ... failure probability of each input's certificate (likewise)
SERVER_OPTS = ("sgd", "momentum", "adagrad", "adam", "yogi")
SELECTIONS = ("none", "krum", "multikrum", "dnc")
DNC_DIM = 10000                  # DnC: coordinates per subsample b
DNC_ITERS = 1                    # DnC: subsample iterations T
DNC_FRAC = 1.0                   # DnC: filtering fraction c; each iteration removes floor(c F) participants
DETECTORS = ("none", "fldetector")
FLD_WINDOW = 10                  # FLDetector: the L-BFGS memory and the score window N
FLD_START = 0                    # FLDetector: the first round detection may run (it also waits for round 2N + 1)
COLLUDE_MODES = ("none", "alie", "minmax", "minsum")
COLLUDE_DIRS = ("backdoor", "std", "sign", "unit")
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
                        "median-norm clipping and adaptive noise, Nguyen et al. 2022) | foolsgold (a weighted mean that "
                        "down-weights agents whose summed update histories are too similar to another's, Fung et al. 2020) | flare (a "
                        "weighted mean that trusts the models whose penultimate-layer representations of a clean root set lie among the "
                        "others' nearest by MMD, Wang et al. 2022) | deepsight (clusters the models by their output-layer energy, "
                        "update direction and behaviour on random inputs, and drops clusters of models whose output layer was trained "
                        "on few labels, then averages the rest clipped to the median norm, Rieger et al. 2022)")
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
    p.add_argument("--server_topk", type=float, default=0.0,
                   help="SparseFed (Panda et al. 2022): every round the server applies only the k = floor(p * n_params) largest "
                        "coordinates of its accumulated step (after the vote, the rule, noise and --server_opt) and carries the rest over "
                        "as error feedback.  0 <= p <= 1 (0 = off).  The paper's setting adds --server_clip --clip L")
    p.add_argument("--param_clip", type=float, default=0.0,
                   help="CRFL (Xie et al. 2021): after every round's complete server step (vote, rule, noise, --server_opt, --server_topk) "
                        "the global model's real parameters are scaled by min(1, rho / ||w||).  rho > 0 (0 = off)")
    p.add_argument("--param_noise", type=float, default=0.0,
                   help="CRFL: after the clip, every real parameter gets sigma * z, z ~ N(0, 1) keyed by (--seed, round, coordinate), in every "
                        "round including the last.  sigma >= 0 (0 = off)")
    p.add_argument("--certify", action="store_true",
                   help="CRFL: after the last round certify the final global model on the validation and the poisoned validation set by "
                        "parameter smoothing with sigma = --param_noise (needs --param_noise > 0): a prediction per input, or an "
                        "abstention, with an L2 radius in parameter space")
    p.add_argument("--certify_n0", type=int, default=None,
                   help=f"--certify: noisy models that select each input's class, an integer >= 1 (default {CERTIFY_N0})")
    p.add_argument("--certify_n", type=int, default=None,
                   help=f"--certify: noisy models that estimate the selected class's probability, an integer >= 1 (default {CERTIFY_N})")
    p.add_argument("--certify_alpha", type=float, default=None,
                   help=f"--certify: failure probability of each input's certificate, 0 < alpha < 1 (default {CERTIFY_ALPHA})")
    p.add_argument("--select", type=str, default="none", choices=SELECTIONS,
                   help="participant selection before the --aggr rule: krum (Blanchard et al. 2017) admits the participant whose update "
                        "is closest to its K-F-2 nearest neighbours; multikrum the M best such scores; dnc (Shejwalkar and Houmansadr "
                        "2021) removes, on each of --dnc_iters random coordinate subsamples, the floor(c F) participants whose centred "
                        "updates lie furthest along their top principal direction.  Rejected participants take no part in the round "
                        "(vote, rule, BatchNorm mean, noise, server optimizer)")
    p.add_argument("--select_f", type=int, default=-1,
                   help="Byzantine participants the selection assumes (-1 = ceil(num_corrupt * K / num_agents), K participants per round)")
    p.add_argument("--select_m", type=int, default=0, help="participants multikrum admits (0 = K - F; krum admits 1)")
    p.add_argument("--dnc_dim", type=int, default=None,
                   help=f"--select dnc: coordinates b >= 1 of each subsample of the voted coordinates (default {DNC_DIM}; b >= n_vote "
                        "takes every coordinate)")
    p.add_argument("--dnc_iters", type=int, default=None,
                   help=f"--select dnc: subsamples T >= 1 per round; the admitted set is the intersection of their kept sets "
                        f"(default {DNC_ITERS})")
    p.add_argument("--dnc_frac", type=float, default=None,
                   help=f"--select dnc: filtering fraction c >= 0; each subsample removes floor(c F) participants (default {DNC_FRAC})")
    p.add_argument("--root_size", type=int, default=None,
                   help=f"--aggr fltrust / flare: clean training samples the server trains its root update on each round (fltrust) or "
                        f"runs every submitted model on (flare) (default {ROOT_SIZE}); drawn once from --seed, never a poisoned sample")
    p.add_argument("--rfa_iters", type=int, default=None,
                   help=f"--aggr rfa: smoothed Weiszfeld passes per round (default {RFA_ITERS}; 0 = the avg step).  Each pass reweights "
                        "every participant by its data size over its distance to the current weighted mean; a fixed count keeps the "
                        "cost per round fixed")
    p.add_argument("--rfa_nu", type=float, default=None,
                   help=f"--aggr rfa: smoothing nu > 0 of the Weiszfeld weights alpha_k / max(nu, d_k) (default {RFA_NU})")
    p.add_argument("--flame_lambda", type=float, default=None,
                   help=f"--aggr flame: noise factor lambda >= 0; the round's Gaussian noise has std lambda * S, S the median update norm "
                        f"the admitted updates are clipped to (default {FLAME_LAMBDA})")
    p.add_argument("--flare_k", type=int, default=None,
                   help="--aggr flare: neighbours k >= 1 each candidate votes for (default per round floor(|F|/2), F the candidates "
                        "with finite features; capped at |F| - 1)")
    p.add_argument("--flare_tau", type=float, default=None,
                   help=f"--aggr flare: temperature tau > 0 of the softmax that turns neighbour counts into trust (default {FLARE_TAU})")
    p.add_argument("--deepsight_samples", type=int, default=None,
                   help=f"--aggr deepsight: random inputs per seed, an integer >= 1 (default {DEEPSIGHT_SAMPLES}); every submitted model "
                        "and the global model run on 3 seeds of them, drawn once from --seed")
    p.add_argument("--deepsight_tau", type=float, default=None,
                   help="--aggr deepsight: a cluster of models is accepted when the share of suspicious models in it is below tau, "
                        "0 < tau <= 1 (default 1/3).  DeepSight guarantees no number of accepted models: a --robustLR_threshold above "
                        "the accepted count flips every coordinate")
    p.add_argument("--detect", type=str, default="none", choices=DETECTORS,
                   help="detection ahead of the --aggr rule: fldetector (Zhang et al. 2022) predicts every agent's update from its last "
                        "one and an L-BFGS Hessian estimate, scores how far each update lies from its prediction, and once the gap "
                        "statistic finds a minority cluster of high scores stops listening to those agents for the rest of the run.  "
                        "Every agent has to take part in every round")
    p.add_argument("--fld_window", type=int, default=None,
                   help=f"--detect fldetector: the L-BFGS memory and the score window N >= 1 (default {FLD_WINDOW})")
    p.add_argument("--fld_start", type=int, default=None,
                   help=f"--detect fldetector: detection runs only in rounds >= max(R, 2N + 1) (default R = {FLD_START})")
    p.add_argument("--attack_boost", type=float, default=1.0,
                   help="model replacement (Bhagoji et al. 2019, Bagdasaryan et al. 2020): every corrupt agent scales its update by this "
                        "factor gamma > 0 before submitting it, after its --clip projection (1 = off; needs --num_corrupt > 0)")
    p.add_argument("--attack_neurotoxin", type=float, default=0.0,
                   help="Neurotoxin (Zhang et al. 2022): corrupt agents never update the top p fraction of coordinates by magnitude of "
                        "the last global update; their gradient is zeroed there at every local step.  0 <= p < 1 (0 = off; needs "
                        "--num_corrupt > 0)")
    p.add_argument("--attack_constrain", type=float, default=1.0,
                   help="constrain-and-scale (Bagdasaryan et al. 2020): in attack rounds corrupt agents train on alpha CE + (1 - alpha) "
                        "||w - w_g||, which keeps the poisoned model close to the global one; combine with --attack_boost to scale it.  "
                        "0 < alpha <= 1 (1 = off; needs --num_corrupt > 0)")
    p.add_argument("--prox_mu", type=float, default=0.0,
                   help="FedProx (Li et al. 2020): every client, and the FLTrust root job, trains on CE + (mu/2) ||w - w_g||^2, a pull "
                        "toward the round's global parameters w_g.  mu >= 0 (0 = off)")
    p.add_argument("--attack_collude", default="none", choices=COLLUDE_MODES,
                   help="colluding attackers with full knowledge: in attack rounds every corrupt participant submits one update crafted "
                        "from the round's honest updates: alie (A Little Is Enough, Baruch et al. 2019) or the Min-Max / Min-Sum attacks "
                        "(Shejwalkar and Houmansadr 2021).  Needs --num_corrupt > 0 and --attack_boost 1")
    p.add_argument("--collude_dir", default=None, choices=COLLUDE_DIRS,
                   help="--attack_collude: the direction u the crafted update leaves the honest mean along: backdoor (towards the "
                        "corrupt agents' own mean update), std, sign or unit (default backdoor; alie takes backdoor or std)")
    p.add_argument("--alie_z", type=float, default=None,
                   help="--attack_collude alie: the number z >= 0 of honest standard deviations the update may lie from the mean "
                        "(default per round: the inverse normal CDF at (K - s) / K, s = max(1, floor(K/2) + 1 - C), floored at 0)")
    p.add_argument("--attack_start", type=int, default=1, help="attack schedule: the first round the corrupt agents attack (>= 1)")
    p.add_argument("--attack_stop", type=int, default=0,
                   help="attack schedule: the last round that may be an attack round (0 = no end).  In the other rounds a corrupt agent "
                        "trains on its clean samples, unmasked and unboosted, like an honest client")
    p.add_argument("--attack_every", type=int, default=1, help="attack schedule: attack every F-th round from --attack_start (>= 1)")
    p.add_argument("--attack_force", action="store_true",
                   help="attack schedule: every corrupt agent takes part in every attack round; the round's draw keeps its size and "
                        "honest participants give way from the end of the draw")
    p.add_argument("--lifespan_threshold", type=float, default=LIFESPAN_THRESHOLD,
                   help="poison accuracy below which the backdoor counts as gone; the rounds from the last attack round until then are "
                        "logged as the backdoor's lifespan.  In (0, 1]; needs --attack_stop > 0")
    return p


def attack_schedule_set(args) -> bool:
    """True when any attack-schedule flag differs from its default (every round an attack round, no forced participation)."""
    return (getattr(args, "attack_start", 1) != 1 or getattr(args, "attack_stop", 0) != 0 or getattr(args, "attack_every", 1) != 1
            or bool(getattr(args, "attack_force", False)))


def is_attack_round(rnd: int, start: int = 1, stop: int = 0, every: int = 1) -> bool:
    """Round ``rnd`` is an attack round iff ``rnd >= start``, ``stop == 0 or rnd <= stop`` and ``(rnd - start) % every == 0``."""
    return rnd >= start and (stop == 0 or rnd <= stop) and (rnd - start) % every == 0


def last_attack_round(start: int, stop: int, every: int):
    """The last attack round ``L = start + every * floor((stop - start) / every)`` of a schedule with a stop round, else None."""
    return start + every * ((stop - start) // every) if stop > 0 else None


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
    topk = float(getattr(args, "server_topk", 0.0))
    if not (math.isfinite(topk) and 0.0 <= topk <= 1.0):
        raise ValueError(f"--server_topk {topk} must be a finite number in [0, 1]")
    args.server_topk = topk
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
    _finalize_flare(args)
    _finalize_rfa(args)
    _finalize_flame(args)
    _finalize_deepsight(args)
    _finalize_crfl(args)
    _finalize_attack(args)
    _finalize_collude(args)
    _finalize_detect(args)
    return args


def _finalize_collude(args) -> None:
    """Validate the colluding-attacker flags and resolve ``collude_dir`` in place (``backdoor`` under ``--attack_collude``): a mode only
    with corrupt agents and no boost, the direction and z only with a mode, alie only along backdoor or std, and z finite and >= 0."""
    mode = getattr(args, "attack_collude", "none")
    d = getattr(args, "collude_dir", None)
    z = getattr(args, "alie_z", None)
    if mode not in COLLUDE_MODES:
        raise ValueError(f"unknown --attack_collude {mode!r}; expected one of {COLLUDE_MODES}")
    if mode == "none":
        if d is not None or z is not None:
            raise ValueError("--collude_dir / --alie_z need --attack_collude")
        return
    if args.num_corrupt <= 0:
        raise ValueError(f"--attack_collude {mode} needs corrupt agents (--num_corrupt > 0)")
    if float(getattr(args, "attack_boost", 1.0)) != 1.0:
        raise ValueError("--attack_collude chooses the crafted update's size itself: it refuses --attack_boost other than 1")
    d = "backdoor" if d is None else d
    if d not in COLLUDE_DIRS:
        raise ValueError(f"unknown --collude_dir {d!r}; expected one of {COLLUDE_DIRS}")
    if mode == "alie" and d not in ("backdoor", "std"):
        raise ValueError(f"--attack_collude alie takes --collude_dir backdoor or std, not {d}")
    if z is not None:
        if mode != "alie":
            raise ValueError("--alie_z needs --attack_collude alie")
        z = float(z)
        if not (math.isfinite(z) and z >= 0):
            raise ValueError(f"--alie_z {z} must be a finite number >= 0")
    args.collude_dir, args.alie_z = d, z


def _finalize_detect(args) -> None:
    """Validate the detection flags and resolve ``fld_window`` / ``fld_start`` in place (``FLD_WINDOW`` / ``FLD_START`` under
    ``--detect fldetector``): every agent in every round, at least 3 agents, no ``--select``, and an RLR threshold no larger than the
    fewest voters detection leaves (it flags at most ceil(K/2) - 1 of K agents, so floor(K/2) + 1 remain; under FLAME, which admits
    floor(K'/2) + 1 of its K' candidates, floor(K'/2) + 1 of those)."""
    detect = getattr(args, "detect", "none")
    window, start = getattr(args, "fld_window", None), getattr(args, "fld_start", None)
    if detect not in DETECTORS:
        raise ValueError(f"unknown --detect {detect!r}; expected one of {DETECTORS}")
    if detect == "none":
        if window is not None or start is not None:
            raise ValueError("--fld_window / --fld_start need --detect fldetector")
        return
    window = FLD_WINDOW if window is None else window
    start = FLD_START if start is None else start
    if int(window) != window or window < 1:
        raise ValueError(f"--fld_window {window} must be an integer >= 1")
    if int(start) != start or start < 0:
        raise ValueError(f"--fld_start {start} must be an integer >= 0")
    K = math.floor(args.num_agents * args.agent_frac)
    if K != args.num_agents or args.num_agents < 3:
        raise ValueError(f"--detect fldetector needs every agent in every round and at least 3 agents: floor(--num_agents {args.num_agents} "
                         f"x --agent_frac {args.agent_frac}) = {K}")
    if getattr(args, "select", "none") != "none":
        raise ValueError("--detect fldetector does not combine with --select: Krum's K >= 2F + 3 and its M are defined over all participants")
    fewest = K // 2 + 1
    if args.aggr == "flame":
        fewest = fewest // 2 + 1
    if args.robustLR_threshold > fewest:
        raise ValueError(f"--robustLR_threshold {args.robustLR_threshold} > {fewest}, the fewest voters --detect fldetector leaves"
                         f"{' under --aggr flame' if args.aggr == 'flame' else ''} of {K}, could flip every coordinate")
    args.fld_window, args.fld_start = int(window), int(start)


def _finalize_attack(args) -> None:
    """Validate the model-poisoning attack flags in place: ``attack_boost`` finite and > 0, ``attack_neurotoxin`` finite in [0, 1), and
    either attack, when active, only with corrupt agents to run it."""
    gamma = float(getattr(args, "attack_boost", 1.0))
    p = float(getattr(args, "attack_neurotoxin", 0.0))
    if not (math.isfinite(gamma) and gamma > 0):
        raise ValueError(f"--attack_boost {gamma} must be a finite number > 0")
    if not (math.isfinite(p) and 0.0 <= p < 1.0):
        raise ValueError(f"--attack_neurotoxin {p} must be a finite number in [0, 1)")
    if (gamma != 1.0 or p > 0) and args.num_corrupt <= 0:
        raise ValueError("--attack_boost / --attack_neurotoxin need corrupt agents (--num_corrupt > 0)")
    args.attack_boost, args.attack_neurotoxin = gamma, p
    _finalize_objective(args)
    _finalize_schedule(args)


def _finalize_objective(args) -> None:
    """Validate the local-objective flags in place: ``prox_mu`` finite and >= 0, ``attack_constrain`` finite in (0, 1] and, when not 1,
    only with corrupt agents to train on it."""
    mu = float(getattr(args, "prox_mu", 0.0))
    alpha = float(getattr(args, "attack_constrain", 1.0))
    if not (math.isfinite(mu) and mu >= 0.0):
        raise ValueError(f"--prox_mu {mu} must be a finite number >= 0")
    if not (math.isfinite(alpha) and 0.0 < alpha <= 1.0):
        raise ValueError(f"--attack_constrain {alpha} must be a finite number in (0, 1]")
    if alpha != 1.0 and args.num_corrupt <= 0:
        raise ValueError("--attack_constrain needs corrupt agents (--num_corrupt > 0)")
    args.prox_mu, args.attack_constrain = mu, alpha


def local_objective(args, attacking: bool):
    """``(a, b, mu)`` of an agent's local objective ``a CE + b ||w - w_g|| + (mu/2) ||w - w_g||^2`` (``ops.FlatSGD``), or None for plain
    cross-entropy.  ``attacking``: a corrupt agent in an attack round, which trains with ``(a, b) = (alpha, 1 - alpha)``; every other
    agent, the FLTrust root job and a corrupt agent in a quiet round train with ``(1, 0)``.  ``mu = --prox_mu`` for all."""
    mu = float(getattr(args, "prox_mu", 0.0))
    alpha = float(getattr(args, "attack_constrain", 1.0)) if attacking else 1.0
    return None if (alpha == 1.0 and mu == 0.0) else (alpha, 1.0 - alpha, mu)


def _finalize_schedule(args) -> None:
    """Validate the attack-schedule flags: start >= 1, stop 0 or >= start, every >= 1, the lifespan threshold finite in (0, 1] and only
    with a stop round, and any schedule only with corrupt agents to follow it."""
    start, stop, every = (int(getattr(args, k, d)) for k, d in (("attack_start", 1), ("attack_stop", 0), ("attack_every", 1)))
    theta = float(getattr(args, "lifespan_threshold", LIFESPAN_THRESHOLD))
    if start < 1:
        raise ValueError(f"--attack_start {start} must be >= 1")
    if stop != 0 and stop < start:
        raise ValueError(f"--attack_stop {stop} must be 0 (no end) or >= --attack_start {start}")
    if every < 1:
        raise ValueError(f"--attack_every {every} must be >= 1")
    if not (math.isfinite(theta) and 0.0 < theta <= 1.0):
        raise ValueError(f"--lifespan_threshold {theta} must be a finite number in (0, 1]")
    if theta != LIFESPAN_THRESHOLD and stop == 0:
        raise ValueError("--lifespan_threshold needs --attack_stop > 0")
    args.attack_start, args.attack_stop, args.attack_every, args.lifespan_threshold = start, stop, every, theta
    args.attack_force = bool(getattr(args, "attack_force", False))
    if attack_schedule_set(args) and args.num_corrupt <= 0:
        raise ValueError("--attack_start / --attack_stop / --attack_every / --attack_force need corrupt agents (--num_corrupt > 0)")


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
    select = getattr(args, "select", "none")
    cand = dnc_fewest(args) if select == "dnc" else (args.select_m if select != "none" else K)
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
    """Validate the FLTrust flags and resolve ``root_size`` in place (``ROOT_SIZE`` by default under ``--aggr fltrust`` or ``flare``)."""
    root_size = getattr(args, "root_size", None)
    if args.aggr not in ("fltrust", "flare"):
        if root_size is not None:
            raise ValueError("--root_size needs --aggr fltrust or flare")
        return
    if args.aggr == "fltrust" and getattr(args, "server_clip", False):
        raise ValueError("--server_clip does not combine with --aggr fltrust, which rescales every update to the root update's norm")
    if root_size is None:
        root_size = ROOT_SIZE
    if root_size < 1:
        raise ValueError(f"--root_size {root_size} must be >= 1")
    args.root_size = int(root_size)


def _finalize_flare(args) -> None:
    """Validate the FLARE flags and resolve ``flare_tau`` in place (``FLARE_TAU`` by default under ``--aggr flare``); ``flare_k`` stays None
    for the per-round default."""
    k, tau = getattr(args, "flare_k", None), getattr(args, "flare_tau", None)
    if args.aggr != "flare":
        if k is not None or tau is not None:
            raise ValueError("--flare_k / --flare_tau need --aggr flare")
        return
    if k is not None and (int(k) != k or k < 1):
        raise ValueError(f"--flare_k {k} must be an integer >= 1")
    tau = FLARE_TAU if tau is None else tau
    if not (math.isfinite(tau) and tau > 0):
        raise ValueError(f"--flare_tau {tau} must be a finite number > 0")
    args.flare_k = None if k is None else int(k)
    args.flare_tau = float(tau)


def _finalize_deepsight(args) -> None:
    """Validate the DeepSight flags and resolve ``deepsight_samples`` / ``deepsight_tau`` in place (``DEEPSIGHT_SAMPLES`` /
    ``DEEPSIGHT_TAU`` by default under ``--aggr deepsight``).  No ``--server_clip``: DeepSight clips to the median norm itself.  It
    guarantees no number of accepted voters, so, as under FLTrust, the RLR threshold is not checked against one."""
    n, tau = getattr(args, "deepsight_samples", None), getattr(args, "deepsight_tau", None)
    if args.aggr != "deepsight":
        if n is not None or tau is not None:
            raise ValueError("--deepsight_samples / --deepsight_tau need --aggr deepsight")
        return
    n = DEEPSIGHT_SAMPLES if n is None else n
    if int(n) != n or n < 1:
        raise ValueError(f"--deepsight_samples {n} must be an integer >= 1")
    tau = DEEPSIGHT_TAU if tau is None else tau
    if not (math.isfinite(tau) and 0 < tau <= 1):
        raise ValueError(f"--deepsight_tau {tau} must be a finite number in (0, 1]")
    if getattr(args, "server_clip", False):
        raise ValueError("--server_clip does not combine with --aggr deepsight, which clips every update to the round's median norm")
    args.deepsight_samples, args.deepsight_tau = int(n), float(tau)


def dnc_fewest(args) -> int:
    """The fewest participants ``--select dnc`` can admit: ``K - T floor(c F)``, every iteration removing others."""
    K = max(1, math.floor(args.num_agents * args.agent_frac))
    return K - args.dnc_iters * math.floor(args.dnc_frac * args.select_f)


def _finalize_dnc(args) -> None:
    """Validate the DnC flags and resolve their defaults in place (``DNC_DIM`` / ``DNC_ITERS`` / ``DNC_FRAC`` under ``--select dnc``)."""
    dim, iters, frac = (getattr(args, k, None) for k in ("dnc_dim", "dnc_iters", "dnc_frac"))
    if getattr(args, "select", "none") != "dnc":
        if dim is not None or iters is not None or frac is not None:
            raise ValueError("--dnc_dim / --dnc_iters / --dnc_frac need --select dnc")
        return
    dim = DNC_DIM if dim is None else dim
    iters = DNC_ITERS if iters is None else iters
    frac = DNC_FRAC if frac is None else frac
    if int(dim) != dim or dim < 1:
        raise ValueError(f"--dnc_dim {dim} must be an integer >= 1")
    if int(iters) != iters or iters < 1:
        raise ValueError(f"--dnc_iters {iters} must be an integer >= 1")
    if not (math.isfinite(frac) and frac >= 0):
        raise ValueError(f"--dnc_frac {frac} must be a finite number >= 0")
    args.dnc_dim, args.dnc_iters, args.dnc_frac = int(dim), int(iters), float(frac)


def _finalize_select(args) -> None:
    """Validate ``--select`` and resolve its defaults in place: ``select_f`` = F, ``select_m`` = M (1 for krum; unused by dnc) and,
    under dnc, its flags (``_finalize_dnc``)."""
    select = getattr(args, "select", "none")
    if select not in SELECTIONS:
        raise ValueError(f"unknown --select {select!r}; expected one of {SELECTIONS}")
    _finalize_dnc(args)
    if select == "none":
        if getattr(args, "select_f", -1) != -1 or getattr(args, "select_m", 0) != 0:
            raise ValueError("--select_f / --select_m need --select krum or multikrum (--select_f also dnc)")
        return
    K = max(1, math.floor(args.num_agents * args.agent_frac))
    f = args.select_f
    if f < -1:
        raise ValueError(f"--select_f {f} must be >= 0 (or -1 for the default)")
    if f == -1:
        f = math.ceil(args.num_corrupt * K / args.num_agents)
    if select == "dnc":
        if getattr(args, "select_m", 0) != 0:
            raise ValueError(f"--select_m {args.select_m} needs --select multikrum; dnc admits what its iterations keep")
        args.select_f = f
        fewest = dnc_fewest(args)
        if fewest < 1:
            raise ValueError(f"--select dnc could admit nobody: K - T floor(c F) = {K} - {args.dnc_iters} x floor({args.dnc_frac} x {f}) "
                             f"= {fewest} < 1")
        if args.robustLR_threshold > fewest:
            raise ValueError(f"--robustLR_threshold {args.robustLR_threshold} > {fewest}, the fewest participants --select dnc admits, "
                             "could flip every coordinate")
        return
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


def _finalize_crfl(args) -> None:
    """Validate the CRFL flags and resolve ``certify_n0`` / ``certify_n`` / ``certify_alpha`` in place (defaults under ``--certify``)."""
    rho, sigma = float(getattr(args, "param_clip", 0.0)), float(getattr(args, "param_noise", 0.0))
    if not (math.isfinite(rho) and rho >= 0.0):
        raise ValueError(f"--param_clip {rho} must be a finite number > 0 (0 = off)")
    if not (math.isfinite(sigma) and sigma >= 0.0):
        raise ValueError(f"--param_noise {sigma} must be a finite number >= 0 (0 = off)")
    args.param_clip, args.param_noise = rho, sigma
    certify = bool(getattr(args, "certify", False))
    n0, n, alpha = (getattr(args, k, None) for k in ("certify_n0", "certify_n", "certify_alpha"))
    if not certify:
        if n0 is not None or n is not None or alpha is not None:
            raise ValueError("--certify_n0 / --certify_n / --certify_alpha need --certify")
        return
    if sigma <= 0.0:
        raise ValueError("--certify smooths with the training noise sigma and needs --param_noise > 0")
    n0 = CERTIFY_N0 if n0 is None else n0
    n = CERTIFY_N if n is None else n
    alpha = CERTIFY_ALPHA if alpha is None else float(alpha)
    if int(n0) != n0 or n0 < 1:
        raise ValueError(f"--certify_n0 {n0} must be an integer >= 1")
    if int(n) != n or n < 1:
        raise ValueError(f"--certify_n {n} must be an integer >= 1")
    if not 0.0 < alpha < 1.0:
        raise ValueError(f"--certify_alpha {alpha} must lie strictly between 0 and 1")
    args.certify, args.certify_n0, args.certify_n, args.certify_alpha = True, int(n0), int(n), alpha


def print_exp_details(args, n_params: int | None = None) -> None:
    """Experiment banner; same 14 fields as reference src/utils.py:287-303 plus engine fields.  ``n_params``: the model's parameter count,
    which sizes SparseFed's k (shown as ``-`` when not given)."""
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
    if getattr(args, "server_topk", 0.0) > 0:
        k = math.floor(args.server_topk * n_params) if n_params is not None else "-"
        print(f"    Server top-k (SparseFed): {args.server_topk} / {k}")
    if getattr(args, "param_clip", 0.0) > 0 or getattr(args, "param_noise", 0.0) > 0:
        print(f"    CRFL (param clip rho / noise sigma): {args.param_clip} / {args.param_noise}")
    if getattr(args, "certify", False):
        print(f"    Certify (n0 / n / alpha): {args.certify_n0} / {args.certify_n} / {args.certify_alpha}")
    if getattr(args, "select", "none") in ("krum", "multikrum"):
        print(f"    Selection (F / M): {args.select} ({args.select_f} / {args.select_m})")
    if getattr(args, "select", "none") == "dnc":
        print(f"    Selection DnC (F / c / b / T): {args.select_f} / {args.dnc_frac} / {args.dnc_dim} / {args.dnc_iters}")
    if args.aggr == "fltrust":
        print(f"    Root set: {args.root_size}")
    if args.aggr == "flare":
        print(f"    FLARE (root / k / tau): {args.root_size} / {'floor(|F|/2)' if args.flare_k is None else args.flare_k} / {args.flare_tau}")
    if args.aggr == "deepsight":
        print(f"    DeepSight (seeds x samples / tau): 3 x {args.deepsight_samples} / {args.deepsight_tau:.4g}")
    if args.aggr == "rfa":
        print(f"    RFA passes / nu: {args.rfa_iters} / {args.rfa_nu}")
    if args.aggr == "flame":
        print(f"    FLAME lambda: {args.flame_lambda}")
    if getattr(args, "attack_boost", 1.0) != 1.0 or getattr(args, "attack_neurotoxin", 0.0) > 0:
        print(f"    Attack (boost / neurotoxin): {args.attack_boost} / {args.attack_neurotoxin}")
    if getattr(args, "prox_mu", 0.0) != 0.0 or getattr(args, "attack_constrain", 1.0) != 1.0:
        print(f"    Local objective (prox mu / constrain alpha): {args.prox_mu} / {args.attack_constrain}")
    if getattr(args, "attack_collude", "none") != "none":
        z = "per round" if args.alie_z is None else args.alie_z
        print(f"    Attack (collude / dir / z): {args.attack_collude} / {args.collude_dir} / {z if args.attack_collude == 'alie' else '-'}")
    if getattr(args, "detect", "none") != "none":
        print(f"    Detection (window / start): {args.detect} ({args.fld_window} / {args.fld_start})")
    if attack_schedule_set(args):
        print(f"    Attack schedule (start / stop / every / force): {args.attack_start} / {args.attack_stop} / {args.attack_every} / "
              f"{args.attack_force}")
    print("======================================")
