"""Fused aggregate + server-step + broadcast across GPUs (the product path of SURVEY.md 5.8).

Per-rank symmetric slab layout (byte offsets identical on every rank):

    [ flags: uint32[3*world] (+pad to 4 KiB) | w_global fp32[n] | w_global bf16[n] | slot_0 fp32[n] | slot_1 ... ]

Flag words of a rank: [0, world) barrier-in arrivals, [world, 2 world) barrier-out arrivals, [2 world, 3 world) broadcast-ready
words ("slice r of the new global parameters has landed here", written by rank r).

``w_global`` is what every local trainer reads at the start of a round; ``slot_j`` receives the parameters of the
j-th agent this rank trained.  One launch of ``fused_aggregate_kernel`` per rank then (i) waits until every rank has
signalled "slots ready", (ii) reads the owned coordinate slice of every participant's slot straight from the owning
GPU's HBM over NVLink, (iii) computes sign vote / aggregator / RLR flip / server step, (iv) stores the new global
slice into EVERY rank's ``w_global`` (+bf16 shadow) with NVLS multicast stores (or per-peer P2P stores), and (v)
signals/awaits "slice landed".  No NCCL call, no host synchronisation, no materialised update vectors.

Reference counterpart: the Python dict ``agent_updates_dict[agent_id] = update`` (src/federated.py:67-70), the ~30 elementwise
fp64 passes of ``Aggregation.aggregate_updates`` (src/aggregation.py:19-75) and the per-agent
``vector_to_parameters(copy.deepcopy(rnd_global_params), ...)`` "broadcast" (src/federated.py:72).

Hand-off fused with the next round's first GEMM (``enable_handoff``; SURVEY.md A9 / 5.8): the kernel then has NO barrier-out.  Rank r
publishes its slice in every peer's ready word and exits; the consumer of the broadcast is the first local step of the next round
(``models.native.NativeTrainer``): the producer warp of the stem convolution's wgmma GEMM acquires the ready word(s) of the slice(s)
that hold its filter -- it reads that filter straight out of the multicast bf16 shadow -- and a one-warp ``acquire_slices`` kernel
queued right behind it waits for the remaining slices, so the first-layer GEMM overlaps the rest of the broadcast.  The separate
``round_init`` pass (w <- w_global, bf16 shadow, momentum <- 0) does not exist on that path: the first optimizer step reads
``w_global`` directly with zero momentum.  Host-side readers of ``w_global`` (evaluation, checkpoints, tests) call ``acquire()`` first.

With ``backend in {nccl, gloo}`` (the baseline transport) the slots are all-gathered and the same kernel runs on the
gathered copies locally; on CPU it runs the fp64 oracle.

Server optimizer state (``--server_opt`` other than sgd; ``ops.ServerOptState``) lives in ordinary device memory, allocated once:
on the fused multi-GPU path rank r keeps only the state of its slice [begin, end) -- it is the only rank that ever steps those
coordinates -- and with every other transport each rank keeps the full vector (identical on all ranks).
"""
from __future__ import annotations

from functools import partial

import torch

from .. import ops
from .symm import SymmetricBuffer

FLAG_BYTES = 4096


class FusedAggregator:
    def __init__(self, ctx, n_total: int, n_vote: int, max_slots: int, backend: str = "auto", with_bf16: bool = True,
                 transport: str = "auto", server_opt=None, n_part: int | None = None):
        """``server_opt``: optional ``dict(kind=..., beta1=..., beta2=..., tau=...)``; ``n_part``: participants per round (default
        every slot), which fixes whether the fused multi-GPU kernel or the gather fallback runs, and so the state layout."""
        self.ctx = ctx
        # nccl / gloo back-ends: "gather" all-gathers every participant's parameters and runs the kernel on the copies (any
        # aggregator); "reduce" all-reduces per-coordinate partial sums (vote, weighted update sum) -- O(N) instead of O(K N)
        # traffic per rank, avg / sign / RLR only (coordinate median falls back to gather).  auto = reduce across hosts.
        self.transport = transport if transport in ("gather", "reduce") else ("gather" if getattr(ctx, "single_node", True) else "reduce")
        self.n, self.n_vote, self.max_slots = int(n_total), int(n_vote), int(max_slots)
        dev = ctx.device
        if backend == "auto":
            backend = "fused" if (dev.type == "cuda") else ("gloo" if ctx.is_dist else "local")
            if backend == "fused" and ctx.is_dist and not getattr(ctx, "single_node", True):
                backend = "nccl"       # ranks on several hosts: no common peer-memory domain -> all-gather transport + local kernel
                if ctx.is_main:
                    print("[parallel] ranks span several hosts: aggregation uses the NCCL all-gather transport")
        if backend == "fused" and ctx.is_dist and not getattr(ctx, "single_node", True):
            raise ValueError("backend=fused needs all ranks on one host (peer-mapped memory); use --backend nccl across hosts")
        if backend == "fused" and dev.type != "cuda":
            raise ValueError("backend=fused needs CUDA devices")
        self.backend = backend
        self.with_bf16 = with_bf16 and dev.type == "cuda"
        n = self.n
        self.off_flags = 0
        self.off_wg = FLAG_BYTES
        self.off_wb = self.off_wg + 4 * n
        self.off_slots = self.off_wb + 2 * n
        nbytes = self.off_slots + 4 * n * self.max_slots
        use_symm = backend == "fused" and ctx.is_dist
        self.buf = SymmetricBuffer(ctx, nbytes) if use_symm else SymmetricBuffer(_Solo(ctx), nbytes)
        self.w_global = self.buf.tensor(self.off_wg, n, torch.float32)
        self.w_bf16 = self.buf.tensor(self.off_wb, n, torch.bfloat16) if self.with_bf16 else None
        self.slots = [self.buf.tensor(self.off_slots + 4 * n * j, n, torch.float32) for j in range(self.max_slots)]
        self.flipped = torch.zeros(1, dtype=torch.int64, device=dev)
        self.flipped_is_partial = False   # True after a launch in which every rank counted only its own coordinate slice
        self.epoch = 0
        self._tables = {}
        # hand-off state: the epoch consumers of the broadcast wait for (device word read by captured kernels), ready-word address
        self.handoff = False
        self.epoch_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        self.ready_ptr = 0
        self.n_slices = 0
        self.per = n
        if use_symm:
            world = ctx.world
            self.local_sync = torch.zeros(2, dtype=torch.int32, device=dev)
            self.flag_ptrs = ops.PtrTable([self.buf.peer_ptr(r, self.off_flags) for r in range(world)], dev)
            mc = self.buf.mc_ptr(self.off_wg)
            self.use_multimem = bool(mc)
            if self.use_multimem:
                self.out_ptrs = ops.PtrTable([mc], dev)
                self.out_bf16_ptrs = ops.PtrTable([self.buf.mc_ptr(self.off_wb)], dev) if self.with_bf16 else None
            else:
                self.out_ptrs = ops.PtrTable([self.buf.peer_ptr(r, self.off_wg) for r in range(world)], dev)
                self.out_bf16_ptrs = (ops.PtrTable([self.buf.peer_ptr(r, self.off_wb) for r in range(world)], dev)
                                      if self.with_bf16 else None)
            # coordinate slices: multiples of 4, cover [0, n)
            per = (n // 4 + world - 1) // world * 4
            self.per = per
            self.begin = min(n, ctx.rank * per)
            self.end = min(n, self.begin + per)
        n_part = self.max_slots * ctx.world if n_part is None else int(n_part)
        self.sharded = use_symm and n_part <= ops.MAX_FUSED_AGENTS
        so = dict(server_opt or {})
        kind = so.pop("kind", "sgd")
        if self.sharded:
            self.opt = ops.ServerOptState(kind, self.end - self.begin, device=dev, base=self.begin, **so)
        else:
            self.opt = ops.ServerOptState(kind, n, device=dev, **so)

    # ---- hand-off fused with the next round's first GEMM -------------------------------------------------------------------
    def enable_handoff(self):
        """Replace the kernel's barrier-out by per-slice ready words that the consumers acquire (see the module docstring).  With
        one process (no peers) there is nothing to wait for: consumers get ``ready_ptr = 0`` and only the round_init-free first step
        remains.  Returns True."""
        self.handoff = True
        if self.backend == "fused" and self.ctx.is_dist:
            world = self.ctx.world
            self.ready_ptr = self.buf.peer_ptr(self.ctx.rank, self.off_flags) + 4 * 2 * world
            self.n_slices = world
        return True

    def slices_of(self, lo: int, hi: int):
        """Indices (first, last) of the broadcast slices that hold coordinates [lo, hi)."""
        if not self.n_slices:
            return 0, 0
        return min(self.n_slices - 1, lo // self.per), min(self.n_slices - 1, max(lo, hi - 1) // self.per)

    def acquire(self):
        """Make every slice of the current global parameters visible to work queued afterwards on the current stream (needed
        before reading ``w_global`` outside the trainers when the hand-off is fused; a no-op otherwise)."""
        if self.handoff and self.ready_ptr:
            ops.ext().acquire_slices(self.ready_ptr, 0, self.n_slices - 1, self.epoch_dev, None, None)

    # ---------------------------------------------------------------------------------------------------------
    def slot_owner(self, j: int):
        """(rank, local slot) of the j-th participant of a round."""
        return j % self.ctx.world, j // self.ctx.world

    def _agent_table(self, n_part: int):
        if n_part not in self._tables:
            ptrs = []
            for j in range(n_part):
                r, s = self.slot_owner(j)
                ptrs.append(self.buf.peer_ptr(r, self.off_slots + 4 * self.n * s))
            self._tables[n_part] = ops.PtrTable(ptrs, self.ctx.device)
        return self._tables[n_part]

    def _member_table(self, idx):
        """Pointer table of the slots of the participants at positions ``idx`` (the admitted ones)."""
        return ops.PtrTable([self.buf.peer_ptr(r, self.off_slots + 4 * self.n * s) for r, s in map(self.slot_owner, idx)], self.ctx.device)

    def gathers(self, n_part: int) -> bool:
        """True when a round of ``n_part`` participants runs on all-gathered copies of the participants (the nccl / gloo transports,
        and more participants than the fused kernel's tables hold).  Selection then gathers once (``gather_participants``) and hands the
        copies to both ``pairwise_sqdist`` and ``aggregate``."""
        return self.ctx.is_dist and not self._p2p(n_part)

    def _p2p(self, n_part: int) -> bool:
        """True when a round of ``n_part`` participants runs on the fused multi-GPU path (peer-mapped slots, in-kernel barriers)."""
        return self.backend == "fused" and self.ctx.is_dist and n_part <= ops.MAX_FUSED_AGENTS

    def _fused_pass(self, shape, launch):
        """A participant pass on the fused multi-GPU path: ``launch(begin, end, out, flag_ptrs, local_sync, rank, world, epoch)`` over
        this rank's slice of ``[0, n_vote)`` into a float64 ``out`` of ``shape``, behind the aggregation kernel's barrier-in at an epoch
        of its own; the ranks all_gather their partials and add them in rank order, so the result is identical on every rank."""
        ctx = self.ctx
        self.epoch += 1
        part = torch.empty(shape, dtype=torch.float64, device=ctx.device)
        launch(self.begin, max(self.begin, min(self.end, self.n_vote)), part, self.flag_ptrs.tensor, self.local_sync, ctx.rank, ctx.world,
               self.epoch)
        parts = ctx.all_gather(part)                                     # [world, *shape]
        out = parts[0].clone()
        for r in range(1, ctx.world):
            out += parts[r]
        return out

    def pairwise_sqdist(self, n_part: int, scales=None, participants=None):
        """K x K float64 squared distances between the round's ``n_part`` participants' updates over ``[0, n_vote)`` (Krum / Multi-Krum
        selection), identical on every rank.  Call it after the slots are final and before ``aggregate`` of the same round.

        Fused multi-GPU path: each rank runs ``pairwise_sqdist_kernel`` over its coordinate slice of the peer-mapped participant slots,
        behind the aggregation kernel's barrier-in (an epoch of its own), and the ranks all_gather their partial matrices and add them in
        rank order.  Gather transport and single process: the same kernel over ``participants`` (every participant's parameters on
        this rank, as ``gather_participants`` returns them; gathered here when not given).  The reduce transport never holds cross-rank
        pairs, so selection always takes the gather transport, as the coordinate median does."""
        if self._p2p(n_part):
            if scales is not None:
                self.acquire()                       # the clipped distances read this rank's w_global
            sc = torch.as_tensor(scales, dtype=torch.float32).to(self.ctx.device) if scales is not None else None
            return self._fused_pass((n_part, n_part), partial(ops.ext().pairwise_sqdist, self._agent_table(n_part).tensor,
                                                              self.w_global.data_ptr() if sc is not None else 0, sc))
        agents = self._participants(n_part, participants)
        return ops.pairwise_sqdist(agents, self.n_vote, self.w_global if scales is not None else None, scales)

    def trust_stats(self, n_part: int, ref: int, participants=None):
        """FLTrust statistics (``ops.trust_statement``'s float64 ``[2 n_part + 1]`` layout) of the round's ``n_part`` participants against
        the root job at position ``ref`` (its parameters live in ``slot_owner(ref)``) over ``[0, n_vote)``, identical on every rank.
        Call it after the slots are final and before ``aggregate`` of the same round.

        Fused multi-GPU path: each rank runs ``trust_stats_kernel`` over its coordinate slice of the peer-mapped slots, behind the
        aggregation kernel's barrier-in (an epoch of its own), and the ranks all_gather their partials and add them in rank order.  The
        pass reads ``w_global``, so it first acquires the broadcast slices of a fused hand-off.  Gather transport and single process:
        the same kernel over ``participants`` (``gather_participants(max(n_part, ref + 1))``'s copies, indexed by position; gathered
        here when not given).  The reduce transport never holds a participant and the root on one rank, so the trust pass always takes
        the gather transport; the step that follows then gathers too whenever it leaves a participant out (``members``), and forms the
        same weighted mean from all-reduced partials when every participant is trusted or none is."""
        if self._p2p(n_part):
            self.acquire()
            owner, slot = self.slot_owner(ref)
            return self._fused_pass((2 * n_part + 1,), partial(ops.ext().trust_stats, self._agent_table(n_part).tensor,
                                                               self.buf.peer_ptr(owner, self.off_slots + 4 * self.n * slot),
                                                               self.w_global.data_ptr()))
        copies = participants if participants is not None else self.gather_participants(max(n_part, ref + 1))
        if len(copies) <= max(n_part - 1, ref):
            raise ValueError(f"{len(copies)} participant copies for {n_part} participants and the root job at position {ref}")
        return ops.trust_stats(list(copies[:n_part]), copies[ref], self.w_global, self.n_vote)

    def rfa_sqdist(self, n_part: int, b, scales=None, members=None, participants=None):
        """RFA distance pass (``ops.rfa_statement``): the float64 squared distances of the updates of the participants at positions
        ``members`` (ascending; every one of the round's ``n_part`` when None) to their ``b``-weighted mean over ``[0, n_vote)``, identical
        on every rank.  ``b`` is per member and sums to 1; ``scales`` (server clipping) is per participant.  Call it after the slots are
        final and before ``aggregate`` of the same round.

        Fused multi-GPU path: each rank runs ``rfa_sqdist_kernel`` over its coordinate slice of the peer-mapped slots of the members (the
        pointer table ``aggregate(members=)`` uses), behind the aggregation kernel's barrier-in (an epoch of its own), and the ranks
        all_gather their partials and add them in rank order.  With clipping the pass reads ``w_global``, so it first acquires the
        broadcast slices of a fused hand-off.  Gather transport and single process: the same kernel over ``participants``
        (``gather_participants``' copies; gathered here when not given).  The reduce transport never holds every participant on one rank,
        so the passes take the gather transport, as the coordinate median does; the step that follows keeps every member and may still
        all-reduce."""
        idx = list(range(n_part)) if members is None else [int(j) for j in members]
        if scales is not None:
            scales = scales[torch.as_tensor(idx, device=scales.device)] if torch.is_tensor(scales) else [scales[j] for j in idx]
        if self._p2p(n_part):
            if scales is not None:
                self.acquire()
            dev = self.ctx.device
            table = self._agent_table(n_part) if idx == list(range(n_part)) else self._member_table(idx)
            bt = torch.as_tensor(b, dtype=torch.float64).to(dev)
            sc = torch.as_tensor(scales, dtype=torch.float32).to(dev) if scales is not None else None
            return self._fused_pass((len(idx),), partial(ops.ext().rfa_sqdist, table.tensor, bt,
                                                         self.w_global.data_ptr() if sc is not None else 0, sc))
        agents = self._participants(n_part, participants)
        return ops.rfa_sqdist([agents[j] for j in idx], b, self.n_vote, self.w_global if scales is not None else None, scales)

    def pairwise_gram(self, n_part: int, members=None, participants=None):
        """FLAME Gram pass (``ops.gram_statement``): the float64 Gram matrix of the updates ``w_j - w_global`` of the participants at
        positions ``members`` (ascending; every one of the round's ``n_part`` when None) over ``[0, n_vote)``, identical on every rank.
        Call it after the slots are final and before ``aggregate`` of the same round.

        Fused multi-GPU path: each rank runs ``pairwise_sqdist_kernel<true>`` over its coordinate slice of the peer-mapped slots of the
        members, behind the aggregation kernel's barrier-in (an epoch of its own), and the ranks all_gather their partial matrices and add
        them in rank order.  The pass reads ``w_global``, so it first acquires the broadcast slices of a fused hand-off.  Gather transport
        and single process: the same kernel over ``participants`` (``gather_participants``' copies; gathered here when not given).  The
        reduce transport never holds cross-rank pairs, so the pass takes the gather transport, as Krum's does; the step that follows
        forms the mean from all-reduced partials when everyone is admitted."""
        idx = list(range(n_part)) if members is None else [int(j) for j in members]
        if self._p2p(n_part):
            self.acquire()
            table = self._agent_table(n_part) if idx == list(range(n_part)) else self._member_table(idx)
            return self._fused_pass((len(idx), len(idx)), partial(ops.ext().pairwise_gram, table.tensor, self.w_global.data_ptr()))
        agents = self._participants(n_part, participants)
        return ops.pairwise_gram([agents[j] for j in idx], self.w_global, self.n_vote)

    def aggregate(self, weights, mode, theta, server_lr, noise_std=0.0, seed=0, rnd=0, scales=None, members=None, participants=None,
                  total_weight=None):
        """Aggregate the round's ``len(weights)`` participants (participant j lives in ``slot_owner(j)``; ``weights`` and ``scales`` are
        per participant) and update ``w_global`` on every rank.  ``members``: positions of the participants admitted by selection
        (ascending); only they enter the vote, the rule, the BatchNorm mean and the server step.  ``participants``: copies from
        ``gather_participants`` for the gather transport (gathered here when not given).  ``total_weight``: the weighted mean's
        denominator (default: the members' summed weights).  Returns nothing; ``self.flipped`` accumulates the flipped-coordinate
        count."""
        n_part = len(weights)
        ctx, dev = self.ctx, self.ctx.device
        if members is not None and [int(j) for j in members] == list(range(n_part)):
            members = None                           # everyone admitted: exactly the unselected launch
        if members is not None:
            idx = [int(j) for j in members]
            weights = [weights[j] for j in idx]
            if scales is not None:
                scales = scales[torch.as_tensor(idx, device=scales.device)] if torch.is_tensor(scales) else [scales[j] for j in idx]
        total = float(sum(float(x) for x in weights)) if total_weight is None else float(total_weight)
        self.flipped.zero_()
        self.flipped_is_partial = False
        fused_p2p = self._p2p(n_part)
        if self.opt.kind != "sgd" and fused_p2p != self.sharded:
            raise ValueError(f"{n_part} participants: the server optimizer state was laid out for the "
                             f"{'fused multi-GPU' if self.sharded else 'gather'} path")
        if fused_p2p:
            self.flipped_is_partial = True
            self.epoch += 1
            wt = torch.as_tensor(weights, dtype=torch.float64).to(dev)
            sc = torch.as_tensor(scales, dtype=torch.float32).to(dev) if scales is not None else None
            table = self._agent_table(n_part) if members is None else self._member_table(idx)
            ops.ext().fused_aggregate(
                table.tensor, wt, sc, total, self.w_global.data_ptr(),
                self.out_ptrs.tensor, self.out_bf16_ptrs.tensor if self.out_bf16_ptrs else None, self.use_multimem,
                self.begin, self.end, self.n_vote, ops.MODE_IDS[mode], int(theta), float(server_lr), float(noise_std),
                int(seed), int(rnd), self.flipped, self.flag_ptrs.tensor, self.local_sync, ctx.rank, ctx.world, self.epoch,
                bool(self.handoff), *ops.opt_launch_args(self.opt))
            if self.handoff:
                self.epoch_dev.fill_(self.epoch)      # what the next round's consumers wait for (stream-ordered before their graphs)
            return
        # ---- baseline transports / single process ------------------------------------------------------------------
        if ctx.is_dist and self.transport == "reduce" and mode in ("avg", "sign") and members is None:
            self._aggregate_reduce(weights, mode, theta, server_lr, noise_std, seed, rnd, scales, total)
            return
        # gather participant params, run the kernel locally
        agents = self._participants(n_part, participants)
        if members is not None:
            agents = [agents[j] for j in idx]
        ops.fused_aggregate(self.w_global, agents, weights, mode, theta, server_lr, noise_std, seed, rnd, self.n_vote,
                            scales, out=self.w_global, out_bf16=self.w_bf16, flipped=self.flipped, opt=self.opt, total_weight=total)

    def _aggregate_reduce(self, weights, mode, theta, server_lr, noise_std, seed, rnd, scales, total_weight):
        """All-reduce transport: every rank folds its local participants into (vote, weighted sum), two all_reduce calls make them
        global, and every rank finishes the identical server step locally (ops.aggregate_from_partials).  The noise vector is
        drawn from a torch generator seeded like the CPU oracle on every rank (same stream everywhere; it is NOT the Philox
        stream of the fused kernel)."""
        ctx, n_part = self.ctx, len(weights)
        mine = [j for j in range(n_part) if self.slot_owner(j)[0] == ctx.rank]
        vote, wsum = ops.aggregate_partials(self.w_global, [self.slots[self.slot_owner(j)[1]] for j in mine], [weights[j] for j in mine],
                                            self.n_vote, [scales[j] for j in mine] if scales is not None else None)
        ctx.all_reduce_sum(vote)
        ctx.all_reduce_sum(wsum)
        noise = None
        if noise_std > 0:
            gen = torch.Generator().manual_seed(int(seed) * 1000003 + int(rnd))
            noise = (torch.randn(self.n, generator=gen, dtype=torch.float64) * noise_std).to(self.w_global.device)
            noise[self.n_vote:] = 0
        new, nflip = ops.aggregate_from_partials(self.w_global, vote, wsum, total_weight, mode, theta, server_lr,
                                                 noise, self.n_vote, self.opt)
        self.w_global.copy_(new)
        if self.w_bf16 is not None:
            self.w_bf16.copy_(new.to(torch.bfloat16))
        self.flipped += nflip

    def server_opt_state(self):
        """Full-length fp32 copies ``(m, v)`` of the server optimizer state on every rank (``v`` is None for momentum), or None for
        sgd.  Collective on the fused multi-GPU path, where each rank contributes its slice."""
        opt = self.opt
        if opt.kind == "sgd":
            return None
        full = []
        for t in (opt.m, opt.v):
            if t is None:
                full.append(None)
            elif not self.sharded:
                full.append(t.clone())
            else:
                part = torch.zeros(self.per, dtype=t.dtype, device=t.device)
                part[: t.numel()] = t
                full.append(self.ctx.all_gather(part).view(-1)[: self.n].clone())
        return tuple(full)

    def load_server_opt_state(self, m, v):
        """Set the state from full-length vectors (this rank's slice of them on the fused multi-GPU path)."""
        lo, hi = (self.begin, self.end) if self.sharded else (0, self.n)
        for dst, src in ((self.opt.m, m), (self.opt.v, v)):
            if dst is not None:
                dst.copy_(src[lo:hi].to(dst.device))

    def gather_participants(self, n_part: int):
        """Every participant's flat parameter vector on THIS rank (list of ``n_part`` tensors; remote slots are copied through an
        all_gather).  The gather transport's input, and the copies the ``--diagnostics`` analyses and bench.py's post-run aggregation
        check read."""
        ctx = self.ctx
        if not ctx.is_dist:
            return [self.slots[j] for j in range(n_part)]
        allp = ctx.all_gather(torch.stack(self.slots, 0))            # [world, max_slots, n]
        return [allp[j % ctx.world, j // ctx.world] for j in range(n_part)]

    def _participants(self, n_part: int, participants):
        if participants is None:
            return self.gather_participants(n_part)
        if len(participants) != n_part:
            raise ValueError(f"{len(participants)} participant copies for {n_part} participants")
        return list(participants)

    def update_norms(self, n_part: int):
        """||w_j - w_global|| for every participant (float64 [n_part]), computed where the slot lives."""
        ctx = self.ctx
        mine = [j for j in range(n_part) if self.slot_owner(j)[0] == ctx.rank]
        local = torch.zeros(n_part, dtype=torch.float64, device=ctx.device)
        if mine:
            norms = ops.update_norms(self.w_global, [self.slots[self.slot_owner(j)[1]] for j in mine], self.n_vote)
            local[torch.as_tensor(mine, device=ctx.device)] = norms ** 2
        ctx.all_reduce_sum(local)
        return local.sqrt()

    def close(self):
        self.buf.close()


class _Solo:
    """Context stand-in that makes SymmetricBuffer allocate plain local memory."""

    def __init__(self, ctx):
        self.device, self.world, self.rank, self.is_dist, self.is_main = ctx.device, 1, 0, False, True
