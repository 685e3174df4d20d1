"""Round engine: the reference's driver loop (src/federated.py:21-95) re-designed as one process per GPU.

Reference                                   | here
------------------------------------------- | --------------------------------------------------------------------
agents trained sequentially on 1 device     | participant j of a round trains on rank ``j % world`` (all ranks hold
(src/federated.py:68-72)                    | the device-resident dataset, so any rank can host any agent)
``agent_updates_dict`` of fp64 updates      | each agent's parameters land in a symmetric-memory slot; updates are
(src/federated.py:67,70)                    | formed inside the aggregation kernel
``vector_to_parameters(deepcopy(global))``  | the aggregation kernel multicasts the new global params (fp32 + bf16)
(src/federated.py:72)                       | into every rank's ``w_global``; trainers start each round from it
``aggregator.aggregate_updates``            | ``FusedAggregator.aggregate`` -- one kernel, P2P reads + NVLS stores
evaluation every ``snap`` rounds            | same metrics, device-side confusion matrix, batches strided over ranks

Timed region of the headline metric "FL rounds/sec" = ``run_round`` (local training of all sampled agents +
aggregation + parameter hand-off), evaluation excluded -- BASELINE.md section 2.
"""
from __future__ import annotations

import contextlib
import math
import random

import numpy as np
import torch

from . import ops
from .agent import Agent
from .aggregation import Aggregation, server_opt_spec
from .data import distribute_data, get_datasets, make_poisoned_val
from .data.datasets import DeviceDataset, h5_to_device_dataset, load_fedemnist_client
from .models import get_layout
from .models.graph import feature_dim, head_slices
from .options import (CERTIFY_ALPHA, CERTIFY_N, CERTIFY_N0, attack_schedule_set, is_attack_round, last_attack_round,
                      print_exp_details)
from .parallel import FusedAggregator, init_distributed
from .trainers import make_trainer
from .utils import (MetricLogger, PhaseTimer, backdoor_lifespan, get_loss_n_accuracy, load_checkpoint, restore_server_opt,
                    save_checkpoint)


_ROOT_SET_TAG = 0x464C5472           # "FLTr": keeps the root-set draw apart from every other stream seeded by --seed


def draw_root_set(n_train: int, excluded, size: int, seed: int):
    """FLTrust's root set: ``size`` distinct training-sample indices drawn uniformly without replacement from ``[0, n_train)`` minus
    ``excluded`` (the poisoned samples), seeded by ``seed`` alone -- every rank, and a resumed run, draws the same set.  Ascending
    int64 array; raises ValueError when fewer than ``size`` samples are eligible."""
    keep = np.ones(int(n_train), dtype=bool)
    keep[np.asarray(list(excluded), dtype=np.int64)] = False
    pool = np.flatnonzero(keep)
    if not 1 <= size <= pool.size:
        raise ValueError(f"--root_size {size}: only {pool.size} of {n_train} training samples are unpoisoned")
    return np.sort(np.random.default_rng([int(seed), _ROOT_SET_TAG]).choice(pool, int(size), replace=False)).astype(np.int64)


def force_participants(drawn, num_corrupt: int):
    """Forced participation in an attack round: the corrupt ids (``< num_corrupt``) missing from ``drawn``, in ascending order, take
    the places of the honest ids from the last position of the draw toward the first, until no corrupt id is missing or no honest id
    is left.  A draw that already holds every corrupt id comes back unchanged."""
    out = list(drawn)
    missing = [a for a in range(num_corrupt) if a not in set(out)]
    for pos in range(len(out) - 1, -1, -1):
        if not missing:
            break
        if out[pos] >= num_corrupt:
            out[pos] = missing.pop(0)
    return out


class FLEngine:
    def __init__(self, args, ctx=None, datasets=None, verbose=True):
        self.args = args
        self.ctx = ctx if ctx is not None else init_distributed(args.device, args.backend if args.backend in ("nccl", "gloo") else None)
        ctx = self.ctx
        args.device = ctx.device
        dev = ctx.device
        self.verbose = verbose and ctx.is_main
        torch.manual_seed(args.seed); np.random.seed(args.seed); random.seed(args.seed)
        if self.verbose:
            print_exp_details(args, get_layout(args.model).n_params)

        # ---- data (device resident), partition, poisoned validation set (src/federated.py:34-45) ------------
        if datasets is None:
            datasets = get_datasets(args.data, args.data_dir, args.synthetic, args.synthetic_val, args.seed, dev)
        self.train_dataset, self.val_dataset = datasets
        self.train_dataset.to(dev); self.val_dataset.to(dev)
        self.poisoned_val = make_poisoned_val(self.val_dataset, args)
        self.layout = get_layout(args.model)
        self.n_classes = self.train_dataset.meta.n_classes

        # ---- agents (src/federated.py:49-56) --------------------------------------------------------------------
        self.agents, self.agent_data_sizes = [], {}
        if args.data == "fedemnist" and not args.synthetic:
            # One pre-partitioned file per client (src/agent.py:16-20).  The shards are concatenated into ONE device-resident
            # dataset and every agent gets its index range, so all clients share the trainer's CUDA graphs (keyed by dataset).
            shards = [h5_to_device_dataset(load_fedemnist_client(args.data_dir, _id), "cpu") for _id in range(args.num_agents)]
            self.train_dataset = DeviceDataset("fedemnist", torch.cat([s.data for s in shards]).to(dev),
                                               torch.cat([s.targets for s in shards]).to(dev))
            off = 0
            for _id, s in enumerate(shards):
                self.agents.append(Agent(_id, args, self.train_dataset, range(off, off + len(s)), seed=args.seed))
                off += len(s)
            del shards
        else:
            groups = distribute_data(self.train_dataset, args, n_classes=self.n_classes,
                                     class_per_agent=getattr(args, "class_per_agent", 10))
            for _id in range(args.num_agents):
                self.agents.append(Agent(_id, args, self.train_dataset, groups[_id], seed=args.seed))
        for a in self.agents:
            self.agent_data_sizes[a.id] = a.n_data
        # ---- attack schedule (DESIGN.md section 3): one side copy per poisoned dataset, swapped in for quiet rounds --------------------
        self.schedule = attack_schedule_set(args)
        self._swaps = self._build_swaps() if self.schedule else []
        self._data_poisoned = True                                      # the datasets as the agents left them
        self.last_attack_active = None
        self.last_attack = last_attack_round(args.attack_start, args.attack_stop, args.attack_every)
        self.backdoor_lifespan = None
        # ---- FLTrust: the server's root job, an agent (id num_agents, never corrupt) on a clean sample of the training set -----------
        self.root_agent = None
        if args.aggr == "fltrust":
            poisoned = [i for a in self.agents for i in a.poisoned_idxs]      # poisoning is in place on the shared dataset
            root = draw_root_set(len(self.train_dataset), poisoned, args.root_size, args.seed)
            self.root_agent = Agent(args.num_agents, args, self.train_dataset, root.tolist(), seed=args.seed)
        self.n_part = max(1, math.floor(args.num_agents * args.agent_frac))
        self.detect = getattr(args, "detect", "none") == "fldetector"
        n_jobs = self.n_part + (1 if self.root_agent is not None else 0)   # the root job is position n_part of every round
        max_slots = (n_jobs + ctx.world - 1) // ctx.world
        max_shard = max(a.n_data for a in self._jobs())

        # ---- parameters: flat, symmetric ---------------------------------------------------------------------
        backend = args.backend
        if backend in ("nccl", "gloo") and not ctx.is_dist:
            backend = "local"
        if backend == "auto" and ctx.is_dist and ctx.backend == "gloo":
            backend = "gloo"
        # SparseFed (--server_topk; DESIGN.md section 3): k of the top-k server step, its error vector and scratch live in the aggregator
        p = float(getattr(args, "server_topk", 0.0))
        self.topk_k = ops.sparsefed_k(p, self.layout.n_params) if p > 0 else 0
        self.last_sparse = None
        # CRFL (--param_clip / --param_noise; DESIGN.md section 3): the clip-and-perturb pass after the server step, keyed by (seed, round)
        self.crfl = getattr(args, "param_clip", 0.0) > 0 or getattr(args, "param_noise", 0.0) > 0
        self.last_crfl = None
        self.last_certify = None
        self.fused = FusedAggregator(ctx, self.layout.n_total, self.layout.n_vote, max_slots, backend,
                                     transport=getattr(args, "agg_transport", "auto"), server_opt=server_opt_spec(args),
                                     n_part=self.n_part, history_agents=args.num_agents if args.aggr == "foolsgold" else 0,
                                     fld_agents=args.num_agents if self.detect else 0, fld_window=args.fld_window if self.detect else 0,
                                     topk_k=self.topk_k,
                                     crfl=(args.param_clip, args.param_noise, ops.real_mask(self.layout)) if self.crfl else None)
        init = torch.zeros(self.layout.n_total, dtype=torch.float32)
        self.layout.init_(init, args.seed)
        self.fused.w_global.copy_(init.to(dev))
        if self.fused.w_bf16 is not None:
            self.fused.w_bf16.copy_(self.fused.w_global.to(torch.bfloat16))
        self.w_global = self.fused.w_global
        # ---- FLARE: the clean root set every submitted model runs on, assembled once (eval normalisation, no augmentation), and this
        # rank's [max_slots][|R|][d] block of its participants' penultimate-layer features.  Nothing is trained on R.
        self.flare_x = self.flare_local = None
        if args.aggr == "flare":
            poisoned = [i for a in self.agents for i in a.poisoned_idxs]
            root = draw_root_set(len(self.train_dataset), poisoned, args.root_size, args.seed)
            self.flare_x, _ = self.train_dataset.batch(torch.as_tensor(root, device=dev))
            self.flare_local = torch.zeros((max_slots, len(root), feature_dim(self.layout)), dtype=torch.float32, device=dev)
        # ---- DeepSight: its random inputs (S seeds of --deepsight_samples images, drawn once from --seed) and this rank's
        # [max_slots][(S + 2) P] block of its participants' statistics.  A head without a bias is refused here.
        self.ds_x = self.ds_local = None
        if args.aggr == "deepsight":
            self.ds_head = head_slices(self.layout)
            self.ds_x = ops.deepsight_inputs(self.train_dataset.meta, args.seed, args.deepsight_samples, dev)
            self.ds_local = torch.zeros((max_slots, (ops.DEEPSIGHT_SEEDS + 2) * self.ds_head[2]), dtype=torch.float64, device=dev)

        self.trainer = make_trainer(args.trainer, self.layout, args, dev, max_shard)
        # Several agents per GPU and round can be trained concurrently: trainer i (own parameters, activations, CUDA graphs) runs
        # on stream i.  The small reference CNNs are launch-latency bound at batch 256, so two to four agents in flight fill the GPU.
        n_flight = int(getattr(args, "agents_in_flight", 0))
        if n_flight <= 0:
            # auto: two agents in flight whenever this rank hosts more than one (native trainer on CUDA).  The small reference CNNs are
            # launch / latency bound at batch 256; the large models run one-wave kernels in lock step whose ragged tails a second
            # agent's kernels fill.  One agent per rank (the multi-GPU headline): nothing to overlap.
            # Native trainer only: the autograd trainer drives cuDNN from PyTorch's backward threads (see below).
            n_flight = 2 if (dev.type == "cuda" and self.trainer.name == "native") else 1
        if n_flight > 1 and dev.type == "cuda" and self.trainer.name != "native":
            # two autograd trainers replaying cuDNN / cuBLAS graphs on two streams dead-lock
            # the device within a few rounds (library kernels whose CTAs wait for each other while the other graph holds the SMs)
            if ctx.is_main:
                print(f"[engine] --agents_in_flight {n_flight} needs the native trainer; the {self.trainer.name} trainer trains one agent at a time")
            n_flight = 1
        n_flight = min(max(1, n_flight), max_slots)
        self.trainers = [self.trainer] + [make_trainer(args.trainer, self.layout, args, dev, max_shard) for _ in range(n_flight - 1)]
        # (on CPU the extra trainers are still used round-robin -- same bookkeeping, no overlap)
        self.streams = [torch.cuda.Stream(dev) for _ in range(n_flight)] if (n_flight > 1 and dev.type == "cuda") else None
        # Round hand-off fused with the first local GEMM (native trainer only): no round_init pass, no barrier-out in the aggregation
        # kernel -- the first step of every agent reads the broadcast buffer behind per-slice ready flags (parallel/fused_agg.py).
        self.handoff = False
        if not getattr(args, "no_fused_handoff", False) and all(hasattr(t, "attach_broadcast") for t in self.trainers):
            if all([t.attach_broadcast(self.fused) for t in self.trainers]):
                self.handoff = self.fused.enable_handoff()
        self._loss_parts = [torch.zeros(1, dtype=torch.float32, device=dev) for _ in range(n_flight)]
        self.logger = MetricLogger(args, enabled=ctx.is_main and bool(args.log_dir))
        self.aggregator = Aggregation(self.agent_data_sizes, self.layout.n_params, self.poisoned_val, args,
                                      self.logger, self.layout, self.fused)
        self.timer = PhaseTimer(dev)
        self.round_loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self.cum_poison_acc_mean = 0.0
        self.start_round = 1
        self._stream_src = None
        # ---- model-poisoning attackers (DESIGN.md section 3): boost factor, and Neurotoxin's state -------------------------
        # w_prev = the global parameters at the start of the previous round; the mask words and |M| are rewritten in place every round,
        # so the corrupt agents' captured graphs stay valid
        self.attack_boost = float(getattr(args, "attack_boost", 1.0))
        p = float(getattr(args, "attack_neurotoxin", 0.0))
        self.neurotoxin_k = math.floor(p * self.layout.n_params) if p > 0 else None
        self.last_masked_coords = None
        # colluding attackers (DESIGN.md section 3): stateless, so nothing is allocated and checkpoints are unchanged
        self.collude = getattr(args, "attack_collude", "none")
        self.last_collude = None
        if self.neurotoxin_k is not None:
            nv = self.layout.n_vote
            self.w_prev = torch.zeros(nv, dtype=torch.float32, device=dev)
            self.attack_mask = torch.zeros(ops.mask_words(nv), dtype=torch.int32, device=dev)
            self.masked_coords = torch.zeros(1, dtype=torch.int64, device=dev)
            self._have_prev = False
        if args.resume:
            ck = load_checkpoint(args.resume, self.w_global, self.layout)
            if self.fused.w_bf16 is not None:
                self.fused.w_bf16.copy_(self.w_global.to(torch.bfloat16))   # the hand-off's first step reads the shadow
            restore_server_opt(ck, self.fused)
            self.start_round = ck["round"] + 1
            self.cum_poison_acc_mean = ck["extra"].get("cum_poison_acc_mean", 0.0)
            if self.neurotoxin_k is not None:
                w_prev = ck["extra"].get("neurotoxin_w_prev")
                if w_prev is None:
                    raise ValueError("checkpoint has no Neurotoxin state (w_prev), but this run uses --attack_neurotoxin")
                self.w_prev.copy_(w_prev.to(dev))
                self._have_prev = True
            if self.last_attack is not None:
                if "backdoor_lifespan" not in ck["extra"]:
                    raise ValueError("checkpoint has no backdoor lifespan, but this run uses --attack_stop")
                self.backdoor_lifespan = ck["extra"]["backdoor_lifespan"]
            if self.fused.history is not None:
                hist = ck["extra"].get("foolsgold_history")
                if hist is None:
                    raise ValueError("checkpoint has no FoolsGold history, but this run uses --aggr foolsgold")
                self.fused.load_foolsgold_history(hist)
            if self.detect:
                fld = ck["extra"].get("fldetector")
                if fld is None:
                    raise ValueError("checkpoint has no FLDetector state, but this run uses --detect fldetector")
                self.fused.load_fld_tables(fld["table"], fld["ring"], fld["w_prev"])
                self.aggregator.load_fld_state(fld)
            if self.topk_k:
                e = ck["extra"].get("sparsefed_error")
                if e is None:
                    raise ValueError("checkpoint has no SparseFed state (error vector), but this run uses --server_topk")
                self.fused.load_sparsefed_error(e)
        ctx.barrier()

    def _build_swaps(self):
        """The corrupt agents' side copies, concatenated per poisoned dataset: ``[(dataset, idx, rows, labels)]``.  The indices of one
        dataset are checked distinct here, once, so a swap needs no host sync."""
        by_ds = {}
        for a in self.agents:
            for sel, x, y in a.clean_copy or ():
                by_ds.setdefault(id(a.dataset), (a.dataset, []))[1].append((sel, x, y))
        swaps = []
        for ds, parts in by_ds.values():
            idx = torch.cat([p[0] for p in parts])
            if torch.unique(idx).numel() != idx.numel():
                raise ValueError("attack schedule: two corrupt agents poisoned the same training sample")
            swaps.append((ds, idx, torch.cat([p[1] for p in parts]), torch.cat([p[2] for p in parts])))
        return swaps

    def attack_active(self, rnd: int) -> bool:
        """Whether round ``rnd`` is an attack round of ``--attack_start / --attack_stop / --attack_every``."""
        a = self.args
        return is_attack_round(rnd, a.attack_start, a.attack_stop, a.attack_every)

    def _set_poisoned(self, poisoned: bool):
        """Bring every poisoned dataset to the wanted state: one swap launch per dataset on the current stream when it differs."""
        if poisoned != self._data_poisoned:
            for ds, idx, x, y in self._swaps:
                ops.swap_samples(ds.data, ds.targets, idx, x, y)
            self._data_poisoned = poisoned

    def _jobs(self):
        """Every agent this engine may train: the clients, then the FLTrust root job."""
        return self.agents + ([self.root_agent] if self.root_agent is not None else [])

    # ---- sampling (src/federated.py:68; seeded here) ---------------------------------------------------------
    def sample_agents(self, rnd: int):
        rs = np.random.RandomState((self.args.seed * 1_000_003 + rnd) % (2 ** 31))
        return [int(a) for a in rs.choice(self.args.num_agents, self.n_part, replace=False)]

    def place_participants(self, chosen):
        """Order the round's participants so that the static participant -> (rank, slot) map (j % world, j // world) balances the
        local-training time of the ranks.  With equal shards (the FMNIST / CIFAR-10 partitions) the sampled order is kept; with
        skewed shards (Fed-EMNIST clients differ ~10x) the participants are sorted by their number of local steps and dealt to the
        ranks in serpentine order, which keeps equal slot counts per rank and evens out the step sums.  Deterministic, identical
        on every rank; aggregation is order-independent, so only the floating-point summation order changes."""
        world = self.ctx.world
        if world <= 1 or len(chosen) <= world:
            return list(chosen)
        bs, ep = self.args.bs, self.args.local_ep
        cost = {a: ep * ((self.agents[a].n_data + bs - 1) // bs) for a in chosen}
        if max(cost.values()) == min(cost.values()):
            return list(chosen)
        by_cost = sorted(chosen, key=lambda a: (-cost[a], a))
        out = []
        for row in range(0, len(by_cost), world):
            chunk = by_cost[row:row + world]
            out.extend(chunk if (row // world) % 2 == 0 else chunk[::-1])
        return out

    # ---- end-to-end input streaming (bench "e2e"): shards come from pinned host memory every round ----------
    def enable_input_streaming(self):
        """End-to-end mode: every agent's shard is kept in pinned host memory and ``run_round(stream_inputs=True)`` uploads the
        shard of each agent this rank is about to train (one contiguous H2D copy, no scatter, no allocation) into ONE per-rank
        device staging dataset -- what a deployment that receives fresh client data every round does.  A single staging buffer
        keeps the device addresses (and therefore the captured CUDA graphs) identical no matter which agent a rank hosts in a
        round.  Returns the total bytes of all shards."""
        from .data import DeviceDataset
        if self.schedule:
            raise ValueError("input streaming keeps one fixed copy of every shard and cannot follow an attack schedule")
        self._stream_src = {}
        dev = self.ctx.device
        pin = (lambda t: t.cpu().pin_memory()) if dev.type == "cuda" else (lambda t: t.cpu().clone())
        total, n_max = 0, max(a.n_data for a in self._jobs())
        ref = self.agents[0].dataset
        # one staging dataset per in-flight trainer: trainer i always trains out of buffer i, so its CUDA graphs keep their addresses
        self._stream_bufs = [DeviceDataset(ref.name, torch.zeros((n_max, *ref.data.shape[1:]), dtype=ref.data.dtype, device=dev),
                                           torch.zeros(n_max, dtype=torch.int64, device=dev)) for _ in self.trainers]
        for a in self._jobs():
            x, y = a.dataset.data[a.idxs].contiguous(), a.dataset.targets[a.idxs].contiguous()
            self._stream_src[a.id] = (pin(x), pin(y))
            a.dataset = self._stream_bufs[0]                         # re-pointed to its trainer's buffer right before training
            a.idxs = torch.arange(a.n_data, device=dev)              # ... with local indices
            total += x.numel() * x.element_size() + y.numel() * y.element_size()
        self._stream_buf = self._stream_bufs[0]
        return total

    def _upload_shard(self, agent, buf=None):
        """Host->device copy of one agent's shard (pinned source, current stream) into a staging dataset; the agent then trains out of it."""
        buf = buf if buf is not None else self._stream_buf
        x, y = self._stream_src[agent.id]
        n = agent.n_data
        buf.data[:n].copy_(x, non_blocking=True)
        buf.targets[:n].copy_(y, non_blocking=True)
        agent.dataset = buf
        return x.numel() * x.element_size() + y.numel() * y.element_size()

    # ---- one federated round (src/federated.py:66-74) --------------------------------------------------------
    def run_round(self, rnd: int, stream_inputs: bool = False):
        attack = self.attack_active(rnd)
        drawn = self.sample_agents(rnd)
        if attack and self.args.attack_force:
            drawn = force_participants(drawn, self.args.num_corrupt)
        chosen = self.place_participants(drawn)
        ctx, fused = self.ctx, self.fused
        self.last_attack_active = attack
        self.round_loss.zero_()
        steps = 0
        h2d = 0
        self.timer.start("local_train")
        self._set_poisoned(attack)                                       # queued ahead of every trainer stream
        mask = self._neurotoxin_mask(attack) if self.neurotoxin_k is not None else None
        for t in self.trainers:
            t.attack_mask = mask
            t.attack_round = attack                                      # --attack_constrain's objective for corrupt agents
        concurrent = len(self.trainers) > 1
        if concurrent:
            for part in self._loss_parts:
                part.zero_()
            if self.streams is not None:
                cur = torch.cuda.current_stream(ctx.device)
                for st_ in self.streams:
                    st_.wait_stream(cur)                                 # w_global of this round is ready
        jobs = [self.agents[aid] for aid in chosen]
        if self.root_agent is not None:
            jobs.append(self.root_agent)                                 # position len(chosen): trained like any agent
        k = 0
        for j, agent in enumerate(jobs):
            r, s = fused.slot_owner(j)
            if r != ctx.rank:
                continue
            client = agent is not self.root_agent                        # the loss and step count describe the clients
            if concurrent:
                i = k % len(self.trainers)
                with (torch.cuda.stream(self.streams[i]) if self.streams is not None else contextlib.nullcontext()):
                    if stream_inputs:
                        h2d += self._upload_shard(agent, self._stream_bufs[i])     # on stream i: ordered after trainer i's previous agent
                    st = agent.local_train(self.trainers[i], self.w_global, fused.slots[s], rnd)
                    self._boost(agent, fused.slots[s], attack)
                    if client:
                        self._loss_parts[i] += st["loss_sum"]
            else:
                if stream_inputs:
                    h2d += self._upload_shard(agent)
                st = agent.local_train(self.trainer, self.w_global, fused.slots[s], rnd)
                self._boost(agent, fused.slots[s], attack)
                if client:
                    self.round_loss += st["loss_sum"]
            if client:
                steps += st["steps"]
            k += 1
        if concurrent:
            if self.streams is not None:
                for st_ in self.streams:
                    cur.wait_stream(st_)                                 # every slot is final before the aggregation kernel
            for part in self._loss_parts:
                self.round_loss += part
        self.timer.stop("local_train")
        self.timer.start("aggregate")
        self.last_collude = self._collude(chosen, rnd) if (attack and self.collude != "none") else None
        if self.flare_x is not None:
            self.aggregator.aggregate_slots(chosen, rnd, flare_local=self._flare_features(chosen))
        elif self.ds_x is not None:
            self.aggregator.aggregate_slots(chosen, rnd, deepsight_local=self._deepsight_stats(chosen))
        else:
            self.aggregator.aggregate_slots(chosen, rnd)
        self.timer.stop("aggregate")
        return {"chosen": chosen, "steps": steps, "h2d_bytes": h2d}

    def _flare_features(self, chosen):
        """FLARE: the root-set features of the participants this rank owns (``slot_owner``), from their final slots (after boosting and
        collusion), into ``flare_local``; on the main stream, after the trainer streams have joined."""
        fused = self.fused
        for j in range(len(chosen)):
            r, s = fused.slot_owner(j)
            if r == self.ctx.rank:
                self.flare_local[s].copy_(self.trainer.root_features(fused.slots[s], self.flare_x))
        return self.flare_local

    def _deepsight_stats(self, chosen):
        """DeepSight: the statistics of the participants this rank owns (``slot_owner``), from their final slots (after boosting and
        collusion) and the global model's logits on the random inputs, into ``ds_local``; on the main stream, after the trainer streams
        have joined.  One statistics pass covers every owned slot."""
        fused = self.fused
        owned = [s for r, s in map(fused.slot_owner, range(len(chosen))) if r == self.ctx.rank]
        if owned:
            zg = self.trainer.root_features(self.w_global, self.ds_x, tap=False)
            z = torch.stack([self.trainer.root_features(fused.slots[s], self.ds_x, tap=False) for s in owned])
            st = ops.deepsight_stats(z, zg, [fused.slots[s] for s in owned], self.w_global, self.ds_head)
            self.ds_local[torch.as_tensor(owned, dtype=torch.int64, device=self.ds_local.device)] = st.to(self.ds_local.device)
        return self.ds_local

    def _neurotoxin_mask(self, attack: bool = True):
        """Start of a round with Neurotoxin on: the mask of the last global update ``w_global - w_prev`` (the top-k coordinates by
        magnitude) and ``w_prev <- w_global``, queued on the current stream ahead of the trainers.  Returns the mask words, or None
        when the mask is empty (the first round a run executes, or k = 0) and in a quiet round, which only refreshes ``w_prev``."""
        nv = self.layout.n_vote
        self.fused.acquire()                                             # the pass reads w_global
        if not self._have_prev or not attack:
            self.w_prev.copy_(self.w_global[:nv])
            self.masked_coords.zero_()
            self._have_prev = True
            return None
        ops.neurotoxin_mask(self.w_global, self.w_prev, nv, self.neurotoxin_k, self.attack_mask, self.masked_coords)
        return self.attack_mask if self.neurotoxin_k > 0 else None

    def _boost(self, agent, slot, attack: bool = True):
        """Model replacement: a corrupt agent's update in its slot scaled by ``--attack_boost`` in an attack round, on the agent's
        stream."""
        if self.attack_boost != 1.0 and agent.is_corrupt and attack:
            ops.boost_update(slot, self.w_global, self.attack_boost, self.layout.n_vote)

    def _collude(self, chosen, rnd: int):
        """Colluding attackers in an attack round: every corrupt participant's slot gets the update crafted from the honest participants'
        ones (``FusedAggregator.collude``).  Returns the round's log fields, or None when no corrupt agent takes part (nothing is launched).
        With no honest participant there is nothing to craft from: the corrupt updates stay as trained, and the round logs H = 0."""
        corrupt = [j for j, a in enumerate(chosen) if self.agents[a].is_corrupt]
        if not corrupt:
            return None
        honest = [j for j, a in enumerate(chosen) if not self.agents[a].is_corrupt]
        if not honest:
            if self.verbose:
                print(f"| Collude: no honest participant in round {rnd}; the corrupt updates are left as trained |")
            return {"collude_honest": 0}
        alie = self.collude == "alie"
        z = (self.args.alie_z if self.args.alie_z is not None else ops.collude_z(len(honest), len(corrupt))) if alie else None
        info = self.fused.collude(len(chosen), honest, corrupt, self.collude, self.args.collude_dir, z)
        rec = {"collude_honest": len(honest), "collude_deviation": info["deviation"]}
        if alie:
            rec["collude_z"] = z
        return rec

    def round_result(self):
        """Device->host read of the round's result: (summed local training loss on this rank, number of REAL coordinates whose
        learning rate was flipped this round).  On the fused multi-GPU back-end every rank counts only its own coordinate slice, so
        the count is all-reduced; the always-zero alignment padding below ``n_vote`` (vote 0 < theta) is taken out, so the count is
        over ``layout.n_params`` coordinates whatever the transport."""
        flipped = self.fused.flipped.double()
        if self.fused.flipped_is_partial:
            flipped = self.ctx.all_reduce_sum(flipped.clone())
        parts = [self.round_loss.double(), flipped]
        if self.neurotoxin_k is not None:
            parts.append(self.masked_coords.double())                   # |M| of the round, read with the same copy
        if self.topk_k:
            parts.append(self.fused.sparse_stats)                       # SparseFed's |M|, tau and ||e||, likewise
        if self.crfl:
            parts.append(self.fused.crfl_stats)                         # CRFL's pre-clip norm and scale, likewise
        vals = torch.cat(parts).cpu()
        if self.neurotoxin_k is not None:
            self.last_masked_coords = int(vals[2])
        if self.crfl:
            s = vals[-2:].tolist()
            self.last_crfl = {"param_norm": s[0], "param_scale": s[1]}
            vals = vals[:-2]
        if self.topk_k:
            s = vals[-3:].tolist()
            self.last_sparse = {"sparse_applied": int(s[0]), "sparse_threshold": s[1], "sparse_error_norm": s[2]}
        n_flip = int(vals[1])
        if self.args.robustLR_threshold > 0:
            n_flip = max(0, n_flip - (self.layout.n_vote - self.layout.n_params))
        return float(vals[0]), n_flip

    # ---- evaluation (src/federated.py:78-92) ---------------------------------------------------------------
    def global_params(self):
        """The current global parameter vector, complete on this rank (acquires the broadcast slices when the hand-off is fused)."""
        self.fused.acquire()
        return self.w_global

    def evaluate(self, rnd: int):
        args = self.args
        fwd = self.trainer.eval_forward(self.global_params())
        kw = dict(bs=args.bs, num_classes=self.n_classes, ctx=self.ctx)
        val_loss, (val_acc, per_class) = get_loss_n_accuracy(fwd, self.val_dataset, **kw)
        poison_loss, (poison_acc, _) = get_loss_n_accuracy(fwd, self.poisoned_val, **kw)
        self.cum_poison_acc_mean += poison_acc
        out = {"val_loss": val_loss, "val_acc": val_acc, "per_class_acc": per_class,
               "poison_loss": poison_loss, "poison_acc": poison_acc,
               "base_class_acc": float(per_class[args.base_class]),
               # reference divides by rnd, not by the number of evaluations (src/federated.py:91; quirk 6 kept)
               "cum_poison_acc_mean": self.cum_poison_acc_mean / rnd}
        lg = self.logger
        lg.add_scalar("Validation/Loss", val_loss, rnd)
        lg.add_scalar("Validation/Accuracy", val_acc, rnd)
        lg.add_scalar("Poison/Base_Class_Accuracy", out["base_class_acc"], rnd)
        lg.add_scalar("Poison/Poison_Accuracy", poison_acc, rnd)
        lg.add_scalar("Poison/Poison_Loss", poison_loss, rnd)
        lg.add_scalar("Poison/Cumulative_Poison_Accuracy_Mean", out["cum_poison_acc_mean"], rnd)
        if self.verbose:
            print(f"| Val_Loss/Val_Acc: {val_loss:.3f} / {val_acc:.3f} |")
            print(f"| Val_Per_Class_Acc: {per_class} ")
            print(f"| Poison Loss/Poison Acc: {poison_loss:.3f} / {poison_acc:.3f} |")
        if self.last_attack is not None and self.backdoor_lifespan is None:
            span = backdoor_lifespan([(rnd, poison_acc)], self.last_attack, args.lifespan_threshold)
            if span is not None:                                         # logged once, in the round the backdoor is gone
                self.backdoor_lifespan = out["backdoor_lifespan"] = span
                lg.add_scalar("Poison/Lifespan", span, rnd)
                if self.verbose:
                    print(f"| Backdoor lifespan: {span} rounds |")
        return out

    # ---- CRFL certification (DESIGN.md section 3) ----------------------------------------------------------
    @torch.no_grad()
    def certify(self):
        """Certify the current global model w on the validation and the poisoned validation set by parameter smoothing (Cohen et al.'s
        CERTIFY in parameter space, sigma = ``--param_noise``).  Draw m < n0 + n writes w + sigma z_m into the trainer's certification
        executor (``ops.crfl_smooth``, stream ``ops.crfl_stream(m, certify=True)``) and sweeps both datasets, whose batches are assembled
        and normalised once; every row's vote lands in int32 counts (``ops.vote_count``): selection counts for m < n0, estimation counts
        after.  With several ranks draw m runs on rank m % world and the counts are all-reduced, so the result does not depend on the
        world size.  Returns ``{"val": ..., "poison": ...}``, each a dict of the per-input ``pred`` (-1 = abstain), ``radius`` (L2 in
        parameter space), ``p_a``, ``labels`` and the ``selection`` / ``estimation`` counts, plus ``acc``, ``abstain`` and ``certified``
        (the certified accuracy at R / sigma in ``ops.CERTIFY_RATIOS``)."""
        args, ctx = self.args, self.ctx
        sigma = float(getattr(args, "param_noise", 0.0))
        if not sigma > 0:
            raise ValueError("certification smooths with the training noise and needs --param_noise > 0")
        n0 = int(getattr(args, "certify_n0", None) or CERTIFY_N0)
        n = int(getattr(args, "certify_n", None) or CERTIFY_N)
        alpha = float(getattr(args, "certify_alpha", None) or CERTIFY_ALPHA)
        w = self.global_params()
        cw, cwb, prepare, forward = self.trainer.certify_executor()
        mask = self.fused.crfl_mask if self.fused.crfl_mask is not None else ops.real_mask(self.layout).to(w.device)
        sets = []
        for name, ds in (("val", self.val_dataset), ("poison", self.poisoned_val)):
            N = len(ds)
            idx = torch.arange(N, device=ds.device)
            batches, labels = [], []
            for s in range(0, N, args.bs):
                x, y = ds.batch(idx[s:s + args.bs])
                batches.append((s, prepare(x)))
                labels.append(y)
            y = torch.cat(labels) if labels else torch.zeros(0, dtype=torch.int64)
            sets.append((name, batches, y, torch.zeros((2, N, self.n_classes), dtype=torch.int32, device=w.device)))
        for m in range(ctx.rank, n0 + n, ctx.world):
            ops.crfl_smooth(w, mask, self.layout.n_vote, sigma, args.seed, m, cw, cwb)
            for _, batches, _, counts in sets:
                c = counts[0 if m < n0 else 1]
                for s, xb in batches:
                    ops.vote_count(forward(xb), c, s)
        out = {}
        for name, _, y, counts in sets:
            if ctx.is_dist:
                ctx.all_reduce_sum(counts)
            cnt = counts.cpu().numpy()
            labels = y.cpu().numpy()
            pred, radius, pa = ops.certify_decision(cnt[0], cnt[1], n, alpha, sigma)
            total = max(1, labels.size)
            out[name] = {"pred": pred, "radius": radius, "p_a": pa, "labels": labels, "selection": cnt[0], "estimation": cnt[1],
                         "acc": float(np.sum(pred == labels)) / total, "abstain": float(np.sum(pred < 0)) / total,
                         "certified": ops.certified_accuracy(pred, radius, labels, sigma)}
        self.last_certify = out
        return out

    def _certify_record(self, rnd: int):
        """Run ``certify()`` and report it: the stdout line, the Certify/* TensorBoard tags and the ``certify_*`` record fields."""
        args = self.args
        res = self.certify()
        rec = {}
        for name, tag in (("val", "Val"), ("poison", "Poison")):
            r = res[name]
            rec[f"certify_{name}_acc"], rec[f"certify_{name}_abstain"] = r["acc"], r["abstain"]
            rec[f"certify_{name}_certified"] = r["certified"]
            self.logger.add_scalar(f"Certify/{tag}_Accuracy", r["acc"], rnd)
            self.logger.add_scalar(f"Certify/{tag}_Abstain", r["abstain"], rnd)
        if self.verbose:
            print(f"| Certified (sigma {args.param_noise}, n0/n {args.certify_n0}/{args.certify_n}, alpha {args.certify_alpha}): "
                  f"val acc {res['val']['acc']:.3f} / abstain {res['val']['abstain']:.3f} | "
                  f"poison acc {res['poison']['acc']:.3f} / abstain {res['poison']['abstain']:.3f} |")
        return rec

    # ---- the training loop --------------------------------------------------------------------------------
    def fit(self, rounds: int | None = None):
        args = self.args
        rounds = rounds if rounds is not None else args.rounds
        history = []
        it = range(self.start_round, rounds + 1)
        if self.verbose:
            try:
                from tqdm import tqdm
                it = tqdm(it)
            except Exception:  # noqa: BLE001
                pass
        for rnd in it:
            info = self.run_round(rnd)
            rec = {"steps": info["steps"]}
            if rnd % args.snap == 0:
                ev = self.evaluate(rnd)
                rec.update({k: v for k, v in ev.items() if k != "per_class_acc"})
            loss, flipped = self.round_result()
            rec["train_loss"] = loss / max(1, info["steps"])
            rec["frac_flipped"] = flipped / max(1, self.layout.n_params)
            if self.last_masked_coords is not None:
                rec["attack_masked_coords"] = self.last_masked_coords
                self.logger.add_scalar("Attack/Masked_Coords", self.last_masked_coords, rnd)
            if self.last_sparse is not None:
                rec.update(self.last_sparse)
                for key, tag in (("sparse_applied", "Applied"), ("sparse_threshold", "Threshold"), ("sparse_error_norm", "Error_Norm")):
                    self.logger.add_scalar(f"SparseFed/{tag}", self.last_sparse[key], rnd)
            if self.last_crfl is not None:
                rec.update(self.last_crfl)
                self.logger.add_scalar("ParamClip/Norm", self.last_crfl["param_norm"], rnd)
                self.logger.add_scalar("ParamClip/Scale", self.last_crfl["param_scale"], rnd)
            if self.last_collude is not None:
                rec.update(self.last_collude)
                for key, tag in (("collude_honest", "Honest"), ("collude_deviation", "Deviation"), ("collude_z", "Z")):
                    if key in self.last_collude:
                        self.logger.add_scalar(f"Attack/Collude_{tag}", self.last_collude[key], rnd)
            if self.schedule:
                rec["attack_active"] = self.last_attack_active
                self.logger.add_scalar("Attack/Active", int(self.last_attack_active), rnd)
            if rnd == rounds and self.last_attack is not None and self.backdoor_lifespan is None and rnd >= self.last_attack:
                rec["backdoor_lifespan_at_least"] = rnd - self.last_attack
            if self.aggregator.last_select is not None:
                rec["select_corrupt_participants"] = self.aggregator.last_select["Select/Corrupt_Participants"]
                rec["select_corrupt_admitted"] = self.aggregator.last_select["Select/Corrupt_Admitted"]
            if self.aggregator.last_trust is not None:
                rec["trust_avg_honest"] = self.aggregator.last_trust["Trust/Avg_Honest"]
                rec["trust_avg_corrupt"] = self.aggregator.last_trust["Trust/Avg_Corrupt"]
                rec["trust_admitted"] = self.aggregator.last_trust["Trust/Admitted"]
            if self.aggregator.last_rfa is not None:
                rec["rfa_corrupt_weight"] = self.aggregator.last_rfa["RFA/Corrupt_Weight"]
                rec["rfa_passes"] = self.aggregator.last_rfa["RFA/Passes"]
            if self.aggregator.last_flame is not None:
                rec["flame_admitted"] = self.aggregator.last_flame["FLAME/Admitted"]
                rec["flame_corrupt_admitted"] = self.aggregator.last_flame["FLAME/Corrupt_Admitted"]
                rec["flame_clip_bound"] = self.aggregator.last_flame["FLAME/Clip_Bound"]
                rec["flame_noise_std"] = self.aggregator.last_flame["FLAME/Noise_Std"]
            if self.aggregator.last_flare is not None:
                for key, tag in (("flare_avg_honest", "Avg_Honest_Trust"), ("flare_avg_corrupt", "Avg_Corrupt_Trust"),
                                 ("flare_corrupt_weight", "Corrupt_Weight"), ("flare_bandwidth", "Bandwidth")):
                    rec[key] = self.aggregator.last_flare[f"FLARE/{tag}"]
            if self.aggregator.last_deepsight is not None:
                for key in ("accepted", "corrupt_accepted", "suspicious", "corrupt_suspicious", "clusters", "clip_bound"):
                    tag = "_".join(w.capitalize() for w in key.split("_"))
                    rec[f"deepsight_{key}"] = self.aggregator.last_deepsight[f"DeepSight/{tag}"]
            if self.aggregator.last_foolsgold is not None:
                rec["foolsgold_avg_honest"] = self.aggregator.last_foolsgold["FoolsGold/Avg_Honest_Weight"]
                rec["foolsgold_avg_corrupt"] = self.aggregator.last_foolsgold["FoolsGold/Avg_Corrupt_Weight"]
                rec["foolsgold_admitted"] = self.aggregator.last_foolsgold["FoolsGold/Admitted"]
            if self.detect and self.aggregator.last_fld is not None:
                rec.update(self.aggregator.last_fld)
                if "fld_flagged" in rec and self.verbose:
                    print(f"| FLDetector: flagged {rec['fld_flagged']} in round {rnd} ({rec['fld_corrupt_flagged']} corrupt) |")
            if rnd == rounds and getattr(args, "certify", False):
                rec.update(self._certify_record(rnd))
            rec.update({f"ms_{k}": v for k, v in self.timer.elapsed().items()})
            if args.profile_phases and self.verbose:
                print({k: round(v, 3) for k, v in rec.items() if k.startswith("ms_")})
            self.logger.record(rnd, **rec)
            history.append({"round": rnd, **rec})
            if args.checkpoint and ((args.ckpt_every and rnd % args.ckpt_every == 0) or rnd == rounds):
                state = self.fused.server_opt_state()      # every rank takes part: each holds one slice on the fused multi-GPU path
                hist = self.fused.foolsgold_history() if self.fused.history is not None else None      # collective, likewise
                fld = self.fused.fld_tables() if self.detect else None                                    # collective, likewise
                if self.ctx.is_main:
                    so = None if state is None else {**self.fused.opt.hparams, "m": state[0], "v": state[1]}
                    extra = {"cum_poison_acc_mean": self.cum_poison_acc_mean}
                    if self.neurotoxin_k is not None:
                        extra["neurotoxin_w_prev"] = self.w_prev.cpu()
                    if self.topk_k:
                        extra["sparsefed_error"] = self.fused.sparsefed_error()     # replicated on every rank: no collective
                    if hist is not None:
                        extra["foolsgold_history"] = hist
                    if fld is not None:
                        extra["fldetector"] = {"table": fld[0], "ring": fld[1], "w_prev": fld[2], **self.aggregator.fld_state()}
                    if self.last_attack is not None:
                        extra["backdoor_lifespan"] = self.backdoor_lifespan
                    save_checkpoint(args.checkpoint, self.global_params(), rnd, args, self.layout, extra, so)
        if self.verbose:
            if history and "backdoor_lifespan_at_least" in history[-1]:
                print(f"| Backdoor lifespan: > {history[-1]['backdoor_lifespan_at_least']} rounds |")
            print("Training has finished!")
        return history

    def close(self):
        self.logger.close()
        self.fused.close()
