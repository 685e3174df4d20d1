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
coordinates -- and with every other transport each rank keeps the full vector (identical on all ranks).  FoolsGold's per-agent update
histories (``--aggr foolsgold``) are laid out the same way: ``[num_agents][slice ∩ [0, n_vote)]`` on the fused multi-GPU path, the full
``[num_agents][n_vote]`` table on every rank otherwise.  FLDetector's state (``--detect fldetector``: the per-agent last-update table,
the ring of the last N + 1 global updates and the previous global parameters) uses the same column layout.
"""
from __future__ import annotations

import math
from functools import partial

import numpy as np
import torch

from .. import ops
from .symm import SymmetricBuffer

FLAG_BYTES = 4096


class FusedAggregator:
    def __init__(self, ctx, n_total: int, n_vote: int, max_slots: int, backend: str = "auto", with_bf16: bool = True,
                 transport: str = "auto", server_opt=None, n_part: int | None = None, history_agents: int = 0, fld_agents: int = 0,
                 fld_window: int = 0):
        """``server_opt``: optional ``dict(kind=..., beta1=..., beta2=..., tau=...)``; ``n_part``: participants per round (default
        every slot), which fixes whether the fused multi-GPU kernel or the gather fallback runs, and so the state layout;
        ``history_agents``: agents whose FoolsGold update history this aggregator keeps (``--aggr foolsgold``: ``--num_agents``; 0 = none);
        ``fld_agents`` / ``fld_window``: agents and window N of the FLDetector state (``--detect fldetector``; 0 = none)."""
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
        # FoolsGold's update histories (history_agents > 0): [history_agents][hist_hi - hist_lo] fp32, zero at the start.  On the fused
        # multi-GPU path rank r keeps the columns of its slice that lie below n_vote (the only rank that ever reads or writes them);
        # with every other transport each rank keeps the full [0, n_vote) table, identical on all ranks.
        # FLDetector (fld_window > 0): the last-update table [fld_agents][width], the ring [fld_window + 1][width] and w_prev [width], in
        # the same columns as the history.
        self.history = None
        self.fld_table = self.fld_ring = self.fld_w_prev = None
        if history_agents or fld_window:
            self._alloc_history(int(history_agents or fld_agents), int(fld_window), foolsgold=bool(history_agents))

    def _alloc_history(self, agents: int, fld_window: int = 0, foolsgold: bool = True):
        """Allocate the zero FoolsGold history (``foolsgold``) and / or the zero FLDetector state (``fld_window`` > 0) of ``agents`` rows over
        ``[hist_lo, hist_hi)``: this rank's slice below n_vote on the fused multi-GPU path (empty when the slice lies past n_vote), all of
        ``[0, n_vote)`` otherwise.  Refuses tables that together do not fit in the free device memory."""
        self.hist_lo, self.hist_hi = (self.begin, max(self.begin, min(self.end, self.n_vote))) if self.sharded else (0, self.n_vote)
        width = self.hist_hi - self.hist_lo
        dev = self.ctx.device
        if dev.type == "cuda":
            check_history_memory(agents, width, torch.cuda.mem_get_info(dev)[0], fld_window, foolsgold)
        if foolsgold:
            self.history = torch.zeros((agents, width), dtype=torch.float32, device=dev)
        if fld_window:
            self.fld_table = torch.zeros((agents, width), dtype=torch.float32, device=dev)
            self.fld_ring = torch.zeros((fld_window + 1, width), dtype=torch.float32, device=dev)
            self.fld_w_prev = torch.zeros(width, dtype=torch.float32, device=dev)

    def _col_ptr(self, t, row: int = 0):
        """Address of row ``row`` of a column-sliced table, offset by ``hist_lo`` so that absolute coordinates index it."""
        return t.data_ptr() + 4 * (t.shape[-1] * int(row) - self.hist_lo)

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

    def dnc_grams(self, n_part: int, samples, scales=None, members=None, participants=None):
        """DnC pass (``ops.dnc_gram_statement``): the float64 ``[T][K][K]`` Gram matrices of the centred updates of the participants at
        positions ``members`` (ascending; every one of the round's ``n_part`` when None) at the sorted coordinate samples ``samples``
        (``[T][S]``, ``ops.dnc_sample``'s rows), identical on every rank.  ``scales`` (server clipping) is per participant.  Call it after
        the slots are final and before ``aggregate`` of the same round.

        Fused multi-GPU path: one ``_fused_pass``.  Each rank takes the sample positions whose coordinates lie in its slice of
        ``[0, n_vote)`` (``searchsorted`` on the sorted rows; centring works one coordinate at a time, so the split is exact), runs
        ``dnc_gather_kernel`` over the peer-mapped slots behind the aggregation kernel's barrier-in (an epoch of its own) and the Gram
        kernel over its rows; the ranks all_gather their partial matrices and add them in rank order.  The gather reads ``w_global``,
        so it first acquires the broadcast slices of a fused hand-off.  Gather transport and single process: the same kernels over
        ``participants`` (``gather_participants``' copies; gathered here when not given).  The reduce transport never holds every
        participant on one rank, so the pass takes the gather transport, as Krum's does."""
        idx = list(range(n_part)) if members is None else [int(j) for j in members]
        if scales is not None:
            scales = scales[torch.as_tensor(idx, device=scales.device)] if torch.is_tensor(scales) else [scales[j] for j in idx]
        samples = np.asarray(samples, dtype=np.int64).reshape(len(samples), -1)
        if self._p2p(n_part):
            if self.n_vote >= 1 << 31:
                raise ValueError(f"DnC samples int32 coordinates: n_vote {self.n_vote} >= 2^31")
            self.acquire()
            dev = self.ctx.device
            table = self._agent_table(n_part) if idx == list(range(n_part)) else self._member_table(idx)
            K = len(idx)
            return self._fused_pass((samples.shape[0], K, K), lambda begin, end, out, *gate: ops.dnc_launch(
                table.tensor, K, self.w_global.data_ptr(), samples, scales, out, dev, begin, end, gate))
        agents = self._participants(n_part, participants)
        return ops.dnc_grams([agents[j] for j in idx], self.w_global, samples, self.n_vote, scales)

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

    def collude(self, n_part: int, honest, corrupt, mode: str, direction: str, z=None):
        """Colluding attackers (``ops.collude_statement``): overwrite the voted coordinates of the slots of the round's corrupt participants
        (positions ``corrupt``) with one update crafted from the honest ones (positions ``honest``, at least one), identically on every rank.
        ``z``: alie's z (required for alie).  Call it after the slots are final and before any selection, detection or aggregation pass
        of the same round.  Returns ``{"gamma": gamma* or None, "deviation": ||m - mu||}``.

        Fused multi-GPU path: for minmax / minsum the honest distances (``pairwise_sqdist_kernel`` over the honest members) and the
        statistics pass each run as a ``_fused_pass`` behind the aggregation kernel's barrier-in, so gamma* is the same on every rank; then
        each rank writes its coordinate slice of every corrupt slot through the peer pointers (alie needs only this pass).  Every later
        slice pass reads slice r on rank r, on the stream that wrote it.  The all_gather of the write pass's partials orders every rank's
        writes before anything a rank queues afterwards, so readers of whole slots (``update_norms``, ``gather_participants``) see the
        crafted update.  The passes read ``w_global``, so they first acquire the broadcast slices of a fused hand-off.  Gather and reduce
        transports and single process: the same kernels over ``gather_participants``' copies, identical on every rank, and each rank
        writes the corrupt slots it owns, whole."""
        honest, corrupt = [int(j) for j in honest], [int(j) for j in corrupt]
        H = len(honest)
        if H < 1:
            raise ValueError("collude: the craft needs at least one honest participant")
        dirn, mid = ops.COLLUDE_DIR_IDS[direction], 0 if mode == "alie" else 1
        gamma = None
        if self._p2p(n_part):
            self.acquire()
            table = self._member_table(honest + corrupt)
            outs = self._member_table(corrupt)
            wg = self.w_global.data_ptr()
            if mode != "alie":
                D = torch.zeros((1, 1), dtype=torch.float64)
                if H > 1:
                    D = self._fused_pass((H, H), partial(ops.ext().pairwise_sqdist, self._member_table(honest).tensor, 0, None))
                st = self._fused_pass((2 * H + 1,), partial(ops.ext().collude_stats, table.tensor, H, wg, dirn))
                gamma = ops.collude_gamma(mode, st[:H], st[H:2 * H], st[2 * H], D)
            dev2 = self._fused_pass((1,), partial(ops.ext().collude_write, table.tensor, H, outs.tensor, wg, mid, dirn, float(z or 0.0),
                                                  float(gamma or 0.0)))
        else:
            copies = self.gather_participants(n_part)
            hon, cor = [copies[j] for j in honest], [copies[j] for j in corrupt]
            outs = [self.slots[s] for r, s in map(self.slot_owner, corrupt) if r == self.ctx.rank]
            if mode != "alie":
                D = ops.pairwise_sqdist(hon, self.n_vote) if H > 1 else torch.zeros((1, 1), dtype=torch.float64)
                st = ops.collude_stats(hon, cor, self.w_global, self.n_vote, direction)
                gamma = ops.collude_gamma(mode, st[:H], st[H:2 * H], st[2 * H], D)
            dev2 = ops.collude_write(hon, cor, outs, self.w_global, self.n_vote, mode, direction, z, gamma)
        return {"gamma": gamma, "deviation": math.sqrt(max(0.0, float(dev2.reshape(-1)[0])))}

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

    def foolsgold_gram(self, n_part: int, agent_ids, members=None, participants=None):
        """FoolsGold history pass: fold the updates ``w_j - w_global`` of the participants at positions ``members`` (ascending; every one of
        the round's ``n_part`` when None) into the history rows of their agents ``agent_ids[j]`` over ``[0, n_vote)``, then return the
        float64 Gram matrix of those rows (``ops.history_gram_statement``), identical on every rank.  Call it after the slots are final
        and before ``aggregate`` of the same round.

        Fused multi-GPU path: one ``_fused_pass``.  Each rank runs ``history_accumulate_kernel`` over its coordinate slice of the
        peer-mapped slots behind the aggregation kernel's barrier-in (an epoch of its own) into its own columns of the history, then the
        Gram kernel over those columns; the ranks all_gather their partial matrices and add them in rank order.  The pass reads
        ``w_global``, so it first acquires the broadcast slices of a fused hand-off.  Gather transport and single process: the same
        kernels over ``participants`` (``gather_participants``' copies; gathered here when not given) and the full table every rank
        keeps.  The reduce transport never holds every participant on one rank, so the pass takes the gather transport, as FLAME's does."""
        if self.history is None:
            raise ValueError("this aggregator keeps no FoolsGold history (history_agents = 0)")
        if self._p2p(n_part) != self.sharded:
            raise ValueError(f"{n_part} participants: the FoolsGold history was laid out for the "
                             f"{'fused multi-GPU' if self.sharded else 'gather'} path")
        idx = list(range(n_part)) if members is None else [int(j) for j in members]
        if self._p2p(n_part):
            self.acquire()
            dev = self.ctx.device
            table = self._agent_table(n_part) if idx == list(range(n_part)) else self._member_table(idx)
            width = self.hist_hi - self.hist_lo
            # row pointers offset by hist_lo so that absolute coordinates index them (only [hist_lo, hist_hi) is ever touched)
            base = self.history.data_ptr() - 4 * self.hist_lo
            tab = ops.PtrTable([base + 4 * width * int(agent_ids[j]) for j in idx], dev)

            def launch(begin, end, out, flag_ptrs, local_sync, rank, world, epoch):
                ops.ext().history_accumulate(table.tensor, tab.tensor, self.w_global.data_ptr(), begin, end, flag_ptrs, local_sync, rank,
                                             world, epoch)
                ops.ext().history_gram(tab.tensor, begin, end, out)
            return self._fused_pass((len(idx), len(idx)), launch)
        agents = self._participants(n_part, participants)
        rows = [self.history[int(agent_ids[j])] for j in idx]
        ops.history_accumulate(rows, [agents[j] for j in idx], self.w_global, 0, self.n_vote)
        return ops.history_gram(rows, self.n_vote)

    def foolsgold_history(self, chunk_bytes: int = 256 << 20):
        """The full ``[history_agents, n_vote]`` fp32 FoolsGold history on the host of the main rank (what a checkpoint saves); None on the
        other ranks.  Collective on the fused multi-GPU path, where each rank contributes its columns: the rows are all-gathered in chunks
        of about ``chunk_bytes`` of gathered data, so no rank holds more than one chunk of extra device memory, and only the main rank
        copies them to the host."""
        return self._gather_columns(self.history, chunk_bytes)

    def _gather_columns(self, table, chunk_bytes: int = 256 << 20):
        """The full ``[rows, n_vote]`` fp32 form of a column-sliced ``table`` on the host of the main rank; None on the other ranks.
        Collective on the fused multi-GPU path, where each rank contributes its columns: the rows are all-gathered in chunks of about
        ``chunk_bytes`` of gathered data, so no rank holds more than one chunk of extra device memory, and only the main rank copies them
        to the host."""
        main = self.ctx.is_main
        if not self.sharded:
            if not main:
                return None
            return table.cpu() if table.is_cuda else table.clone()
        A = table.shape[0]
        world, per = self.ctx.world, self.per
        full = torch.empty((A, self.n_vote), dtype=torch.float32) if main else None
        rows = max(1, int(chunk_bytes) // (4 * per * world))
        width = self.hist_hi - self.hist_lo
        for a0 in range(0, A, rows):
            a1 = min(A, a0 + rows)
            part = torch.zeros((a1 - a0, per), dtype=torch.float32, device=table.device)
            part[:, :width] = table[a0:a1]
            allp = self.ctx.all_gather(part)                                 # [world, rows, per]: rank r holds columns [r per, r per + per)
            if main:
                full[a0:a1] = allp.permute(1, 0, 2).reshape(a1 - a0, world * per)[:, : self.n_vote].cpu()
            del part, allp
        return full

    def load_foolsgold_history(self, full):
        """Set the history from a full ``[history_agents, n_vote]`` table (this rank's columns of it on the fused multi-GPU path)."""
        if self.history is None:
            raise ValueError("this aggregator keeps no FoolsGold history (history_agents = 0)")
        if tuple(full.shape) != (self.history.shape[0], self.n_vote):
            raise ValueError(f"FoolsGold history of shape {tuple(full.shape)}; this run keeps {self.history.shape[0]} agents x "
                             f"{self.n_vote} voted coordinates")
        self.history.copy_(full[:, self.hist_lo:self.hist_hi])

    # ---- FLDetector ----------------------------------------------------------------------------------------------
    def _fld_check(self, n_part: int):
        if self.fld_table is None:
            raise ValueError("this aggregator keeps no FLDetector state (fld_window = 0)")
        if self._p2p(n_part) != self.sharded:
            raise ValueError(f"{n_part} participants: the FLDetector state was laid out for the "
                             f"{'fused multi-GPU' if self.sharded else 'gather'} path")

    def fld_ring_update(self, row=None):
        """The ring pass on this rank's columns: ring row ``row`` <- ``fp32(w_global - w_prev)`` (skipped when None), then ``w_prev <-
        w_global``.  Purely local; it reads ``w_global``, so it first acquires the broadcast slices of a fused hand-off."""
        if self.fld_table is None:
            raise ValueError("this aggregator keeps no FLDetector state (fld_window = 0)")
        self.acquire()
        if self.sharded:
            ops.ext().fld_ring(self.w_global.data_ptr(), self._col_ptr(self.fld_w_prev), 0 if row is None else self._col_ptr(self.fld_ring, row),
                               self.hist_lo, self.hist_hi)
        else:
            ops.fld_ring(self.w_global, self.fld_w_prev, None if row is None else self.fld_ring[int(row)], 0, self.n_vote)

    def fld_gram(self, order):
        """The float64 Gram matrix of the ring rows ``order`` (chronological) over ``[0, n_vote)``, identical on every rank: one
        ``_fused_pass`` of ``pairwise_sqdist_kernel<true, true>`` over this rank's columns on the fused multi-GPU path, the same kernel over
        the full ring otherwise."""
        if self.fld_table is None:
            raise ValueError("this aggregator keeps no FLDetector state (fld_window = 0)")
        order = [int(i) for i in order]
        if self.sharded:
            tab = ops.PtrTable([self._col_ptr(self.fld_ring, i) for i in order], self.ctx.device)
            return self._fused_pass((len(order), len(order)), lambda begin, end, out, *gate: ops.ext().history_gram(tab.tensor, begin, end, out))
        return ops.history_gram([self.fld_ring[i] for i in order], self.n_vote)

    def fld_predict(self, n_part: int, agent_ids, order=None, coef=None, participants=None):
        """FLDetector's prediction pass over the round's ``n_part`` participants, whose agents are ``agent_ids``: with ``coef``
        (``ops.fld_hvp_coefficients`` of the ring rows ``order``) the float64 squared distances ``d^2 [n_part]`` of every update to its
        prediction, identical on every rank; then every participant's update is recorded in its agent's row of the last-update table.
        Without ``coef`` it only records and returns None.  Call it after the slots are final and before ``aggregate`` of the same round.

        Fused multi-GPU path: one ``_fused_pass``.  Each rank forms ``Hv`` over its columns of the ring (``fld_hvp_kernel``) and runs
        ``fld_predict_kernel`` over its coordinate slice of the peer-mapped slots behind the aggregation kernel's barrier-in (an epoch of its
        own); the ranks all_gather their partials and add them in rank order.  Gather transport and single process: the same kernels over
        ``participants`` (``gather_participants``' copies; gathered here when not given) and the full tables every rank keeps."""
        self._fld_check(n_part)
        ids = [int(a) for a in agent_ids]
        if self._p2p(n_part):
            self.acquire()
            dev = self.ctx.device
            table = self._agent_table(n_part)
            rows = ops.PtrTable([self._col_ptr(self.fld_table, a) for a in ids], dev)
            if coef is not None:
                ring = ops.PtrTable([self._col_ptr(self.fld_ring, i) for i in order], dev)
                ct = torch.as_tensor(coef, dtype=torch.float64).to(dev)
                hv = torch.empty(max(4, self.hist_hi - self.hist_lo), dtype=torch.float32, device=dev)

            def launch(begin, end, out, flag_ptrs, local_sync, rank, world, epoch):
                hv_ptr = 0
                if coef is not None:
                    hv_ptr = hv.data_ptr() - 4 * begin
                    ops.ext().fld_hvp(ring.tensor, ct, hv_ptr, begin, end)
                else:
                    out.zero_()
                ops.ext().fld_predict(table.tensor, rows.tensor, self.w_global.data_ptr(), hv_ptr, begin, end, out, flag_ptrs, local_sync,
                                      rank, world, epoch)
            d2 = self._fused_pass((n_part,), launch)
            return d2 if coef is not None else None
        agents = self._participants(n_part, participants)
        hv = ops.fld_hvp([self.fld_ring[int(i)] for i in order], coef, 0, self.n_vote) if coef is not None else None
        return ops.fld_predict([self.fld_table[a] for a in ids], agents, self.w_global, hv, 0, self.n_vote)

    def fld_tables(self):
        """``(table, ring, w_prev)``: the full fp32 ``[agents, n_vote]``, ``[N + 1, n_vote]`` and ``[n_vote]`` FLDetector state on the host of
        the main rank (what a checkpoint saves); None on the other ranks.  Collective on the fused multi-GPU path."""
        table, ring = self._gather_columns(self.fld_table), self._gather_columns(self.fld_ring)
        w_prev = self._gather_columns(self.fld_w_prev[None])
        return None if table is None else (table, ring, w_prev[0])

    def load_fld_tables(self, table, ring, w_prev):
        """Set the FLDetector state from its full tables (this rank's columns of them on the fused multi-GPU path)."""
        if self.fld_table is None:
            raise ValueError("this aggregator keeps no FLDetector state (fld_window = 0)")
        for name, dst, src in (("table", self.fld_table, table), ("ring", self.fld_ring, ring), ("w_prev", self.fld_w_prev[None], w_prev[None])):
            if tuple(src.shape) != (dst.shape[0], self.n_vote):
                raise ValueError(f"FLDetector {name} of shape {tuple(src.shape)}; this run keeps {dst.shape[0]} x {self.n_vote}")
            dst.copy_(src[:, self.hist_lo:self.hist_hi])

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


def check_history_memory(num_agents: int, width: int, free_bytes: int, fld_window: int = 0, foolsgold: bool = True):
    """Refuse per-agent state of ``width`` fp32 columns that does not fit in ``free_bytes`` of device memory: FoolsGold's history
    (``foolsgold``: ``4 num_agents width`` bytes) plus FLDetector's state (``fld_window`` = N > 0: the last-update table, the ring of N + 1
    global updates and w_prev, ``4 num_agents width + 4 (N + 2) width`` bytes).  Returns the bytes."""
    A, W, N = int(num_agents), int(width), int(fld_window)
    nbytes = (4 * A * W if foolsgold else 0) + ((4 * A * W + 4 * (N + 2) * W) if N else 0)
    if nbytes > int(free_bytes):
        what = " and ".join(x for x in (("--aggr foolsgold" if foolsgold else ""), (f"--detect fldetector (--fld_window {N})" if N else "")) if x)
        raise ValueError(f"{what} keep fp32 per-agent state: {nbytes} bytes on this GPU for --num_agents {num_agents} x {width} voted "
                         f"coordinates, but only {int(free_bytes)} bytes are free.  Use fewer agents, a smaller --fld_window or more GPUs "
                         "(the fused multi-GPU path shards this state over the ranks)")
    return nbytes


class _Solo:
    """Context stand-in that makes SymmetricBuffer allocate plain local memory."""

    def __init__(self, ctx):
        self.device, self.world, self.rank, self.is_dist, self.is_main = ctx.device, 1, 0, False, True
