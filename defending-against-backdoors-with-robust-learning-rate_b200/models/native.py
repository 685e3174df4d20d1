"""Native (no-autograd) executor of the model IR and the trainer built on it.

``NativeNet`` compiles an IR program (models/graph.py) into a static plan of fused forward ops and their hand-derived
backward ops over pre-allocated NHWC bf16 activation buffers, with parameters read from the flat fp32 buffer ``w``
(bf16 operand shadow ``wb``) and gradients written straight into the flat fp32 buffer ``g`` -- no autograd graph, no
per-tensor optimizer state, no zero_grad (every gradient is overwritten).  The plan fuses

    conv(+bias)(+ReLU)            conv -> per-channel sum / sum^2 (BatchNorm statistics) in the GEMM epilogue
    BN(batch stats) + residual add + ReLU in one pass; BN backward in two (reduce, apply) passes
    avg-pool + flatten + linear head + softmax cross-entropy

Each primitive has two back-ends selected per op in ``self.impl``: ``"sm100"`` -- the hand-written wgmma/TMA
kernels of ops/csrc (gemm.cu / conv.cu / norm.cu) -- and ``"aten"`` -- the same math through library calls on the
same buffers, used as the in-place numerical oracle for the kernels (tests/test_gpu_native.py) and for shapes a
kernel does not cover yet.  ``NativeTrainer`` captures the whole step (gather -> forward -> loss -> backward -> fused
clip+SGD) in CUDA graphs, like ``TorchTrainer``.

Reference call sites replaced: src/models.py:22-31,47-58 (forward), src/agent.py:46-51 (loss/backward/clip/step).
"""
from __future__ import annotations

import math
import os

import torch
import torch.nn.functional as F

from .. import ops
from .graph import FlatLayout

ACT = torch.bfloat16   # default activation / GEMM-operand dtype on GPU (tests may run the plan in fp32 on CPU)
# Weight gradients are off the critical path of the backward pass (nothing but the optimizer reads them): every conv weight-gradient
# kernel is queued on a side stream (forked / joined with events, so it becomes a parallel branch of the captured step graph) while the
# data-gradient / BatchNorm chain continues on the main stream.  RLR_WGRAD_OVERLAP=0 serialises them again.
# partial-sum slots of the per-channel reductions: with N > 1 the CTAs of channel_reduce_kernel spread their atomics over N buffers
# (consumers sum them) and the reductions run four / three CTAs per SM instead of two; default 1 (the two-CTA grid).
# Dropout after a max-pool or a Linear+ReLU is fused into that producer (SURVEY.md K5): the pooling kernel / the GEMM epilogue applies the
# Philox keep-mask, the backward recomputes it (pool) or reads it off the output together with the ReLU mask (linear).  RLR_FUSE_DROPOUT=0
# restores the stand-alone dropout kernels.
FUSE_DROPOUT = bool(int(os.environ.get("RLR_FUSE_DROPOUT", "1")))
# ReLU of a conv whose only consumer is a max-pool: back-propagated inside the pooling backward kernel (no relu_bwd pass over the un-pooled tensor)
FUSE_RELU_POOL = bool(int(os.environ.get("RLR_FUSE_RELU_POOL", "1")))
# BatchNorm statistics from the conv epilogue where they are free (generic kernel, TMA-store epilogue: sums taken while the store drains)
EPILOGUE_BN_STATS = bool(int(os.environ.get("RLR_EPILOGUE_BN_STATS", "0")))
# projection shortcuts (1x1 conv + BatchNorm) of residual blocks on a second stream during the forward pass
FWD_BRANCH = bool(int(os.environ.get("RLR_FWD_BRANCH", "1")))
BWD_BRANCH = bool(int(os.environ.get("RLR_BWD_BRANCH", "1")))     # ... and their backward (needs RLR_FWD_BRANCH)
EPI_STAT_SLOTS = min(16, max(1, int(os.environ.get("RLR_EPI_STAT_SLOTS", "2"))))
FWD_SLOTS = BWD_SLOTS = max(1, int(os.environ.get("RLR_BN_SLOTS", "1")))
WGRAD_OVERLAP = bool(int(os.environ.get("RLR_WGRAD_OVERLAP", "1")))


def dropout_stream_base(seed: int, agent_id: int, rnd: int) -> int:
    """First Philox step-counter value of (agent, round): a splitmix64 hash kept below 2^62 so that the per-step increments of
    one local training run (< 2^20) can neither overflow nor realistically meet another agent's range."""
    z = (int(seed) * 0x9E3779B97F4A7C15 + (int(agent_id) + 1) * 0xBF58476D1CE4E5B9 + (int(rnd) + 1) * 0x94D049BB133111EB) & (2 ** 64 - 1)
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & (2 ** 64 - 1)
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & (2 ** 64 - 1)
    return (z ^ (z >> 31)) & (2 ** 62 - 1)


def native_supported(layout: FlatLayout) -> bool:
    return all(nd.op in ("conv", "bn", "relu", "maxpool", "avgpool", "flatten", "dropout", "linear", "save", "add")
               for nd in layout.nodes)


class _Op:
    """One fused plan entry."""
    __slots__ = ("kind", "node", "name", "attrs", "x", "y", "res", "relu", "saved", "acc_dx", "need_dx", "in_shape", "out_shape")

    def __init__(self, kind, **kw):
        self.kind = kind
        self.node = self.name = self.x = self.y = self.res = None
        self.attrs, self.relu, self.saved, self.acc_dx, self.need_dx = {}, False, {}, False, True
        self.in_shape = self.out_shape = None
        for k, v in kw.items():
            setattr(self, k, v)


class NativeNet:
    def __init__(self, layout: FlatLayout, device, max_batch: int, impl: str | dict = "auto", seed: int = 0, act_dtype=None):
        self.layout, self.device, self.max_batch = layout, torch.device(device), int(max_batch)
        self.act_dtype = act_dtype or ACT
        default = ("sm100" if self.device.type == "cuda" else "aten") if impl == "auto" else impl
        self.impl = dict(conv_fwd=default, conv_dgrad=default, conv_wgrad=default, bn=default, pool=default,
                         linear=default, dropout=default) if not isinstance(impl, dict) else dict(impl)
        self.seed = seed
        self.fuse_bn_stats = False
        self.first_wait = None        # (ready_ptr, lo, hi, epoch tensor): flag wait handed to the first layer's GEMM (round hand-off)
        self.after_first_op = None    # callable run right after the first plan op of a forward pass
        self.step_counter = torch.zeros(1, dtype=torch.int64, device=device)  # Philox offset for dropout
        self._build_plan()
        self._alloc()

    # ------------------------------------------------------------------------------------------------------------
    # planning: shape inference + fusion
    # ------------------------------------------------------------------------------------------------------------
    def _build_plan(self):
        nodes = self.layout.nodes
        C, H, W = self.layout.in_shape
        shape = {"x": (H, W, C)}          # per-slot current (H,W,C) or (F,) after flatten
        ver = {"x": 0}                    # per-slot version counter -> tensor ids "slot@v"
        tid = lambda s: f"{s}@{ver[s]}"
        self.tshape = {tid("x"): shape["x"]}
        plan, consumed = [], set()
        pending_bn = {}
        alias = {}

        def new_out(slot, shp):
            ver[slot] = ver.get(slot, -1) + 1
            shape[slot] = shp
            self.tshape[tid(slot)] = shp
            return tid(slot)

        def next_same_slot(i, slot):
            for j in range(i + 1, len(nodes)):
                if j in consumed:
                    continue
                nd = nodes[j]
                if nd.op == "save":
                    if nd.inp == slot:
                        return None, None  # value is captured: do not fuse across
                    continue
                if nd.inp == slot or nd.out == slot:
                    return j, nd
            return None, None

        for i, nd in enumerate(nodes):
            if i in consumed:
                continue
            a = nd.attrs
            if nd.op == "save":
                ver[nd.out] = ver.get(nd.out, -1) + 1
                alias[f"{nd.out}@{ver[nd.out]}"] = tid(nd.inp)
                shape[nd.out] = shape[nd.inp]
                self.tshape[f"{nd.out}@{ver[nd.out]}"] = shape[nd.inp]
                continue
            src = alias.get(tid(nd.inp), tid(nd.inp))
            if nd.op == "conv":
                h, w, c = shape[nd.inp]
                k, s, p = a["k"], a.get("stride", 1), a.get("pad", 0)
                ho, wo = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
                op = _Op("conv", node=i, name=nd.name, attrs=a, x=src, in_shape=(h, w, c), out_shape=(ho, wo, a["cout"]))
                j, nx = next_same_slot(i, nd.out)
                want_stats = nx is not None and nx.op == "bn"
                if nx is not None and nx.op == "relu":
                    op.relu = True
                    consumed.add(j)
                op.saved["want_stats"] = want_stats
                op.y = new_out(nd.out, op.out_shape)
                plan.append(op)
            elif nd.op == "bn":
                shp = shape[nd.inp]
                op = _Op("bn", node=i, name=nd.name, attrs=a, x=src, in_shape=shp, out_shape=shp)
                j, nx = next_same_slot(i, nd.out)
                if nx is not None and nx.op == "relu":
                    op.relu = True
                    consumed.add(j)
                    op.y = new_out(nd.out, shp)
                    plan.append(op)
                elif nx is not None and nx.op == "add":
                    pending_bn[j] = op   # emitted when the add node is reached (its other operand is ready then)
                else:
                    op.y = new_out(nd.out, shp)
                    plan.append(op)
            elif nd.op == "add":
                other = alias.get(tid(a["other"]), tid(a["other"]))
                op = pending_bn.pop(i, None)
                if op is None:
                    raise NotImplementedError("add without a preceding BatchNorm is not used by any model in the zoo")
                op.res = other
                j, nx = next_same_slot(i, nd.out)
                if nx is not None and nx.op == "relu":
                    op.relu = True
                    consumed.add(j)
                op.y = new_out(nd.out, op.out_shape)
                plan.append(op)
            elif nd.op == "relu":
                raise NotImplementedError("stand-alone ReLU (every ReLU in the zoo follows conv/bn/linear)")
            elif nd.op == "maxpool":
                h, w, c = shape[nd.inp]
                op = _Op("maxpool", node=i, x=src, in_shape=(h, w, c), out_shape=(h // 2, w // 2, c))
                op.y = new_out(nd.out, op.out_shape)
                plan.append(op)
            elif nd.op == "avgpool":
                h, w, c = shape[nd.inp]
                op = _Op("avgpool", node=i, x=src, in_shape=(h, w, c), out_shape=(1, 1, c))
                op.y = new_out(nd.out, op.out_shape)
                plan.append(op)
            elif nd.op == "flatten":
                shp = shape[nd.inp]
                ver[nd.out] += 1
                alias[tid(nd.out)] = src
                shape[nd.out] = (int(math.prod(shp)),)
                self.tshape[tid(nd.out)] = shape[nd.out]
            elif nd.op == "dropout":
                shp = shape[nd.inp]
                prod = next((q for q in reversed(plan) if q.y == src), None)
                fusable = (prod is not None and a.get("p", 0.0) > 0 and "drop" not in prod.saved and
                           (prod.kind == "maxpool" or
                            (prod.kind == "linear" and prod.relu and ops.linear_fused_dropout_ok(prod.attrs["cout"], prod.attrs["cin"]))))
                if fusable and FUSE_DROPOUT:
                    # dropout fused into the producer (pooling kernel / GEMM epilogue): no op, no mask tensor, the output IS the dropped tensor
                    prod.saved["drop"] = (float(a["p"]), i)
                    ver[nd.out] += 1
                    alias[tid(nd.out)] = src
                    shape[nd.out] = shp
                    self.tshape[tid(nd.out)] = shp
                else:
                    op = _Op("dropout", node=i, attrs=a, x=src, in_shape=shp, out_shape=shp)
                    op.y = new_out(nd.out, shp)
                    plan.append(op)
            elif nd.op == "linear":
                op = _Op("linear", node=i, name=nd.name, attrs=a, x=src, in_shape=shape[nd.inp], out_shape=(a["cout"],))
                j, nx = next_same_slot(i, nd.out)
                if nx is not None and nx.op == "relu":
                    op.relu = True
                    consumed.add(j)
                op.y = new_out(nd.out, op.out_shape)
                plan.append(op)
            else:
                raise NotImplementedError(nd.op)
        # ReLU fused into a conv's epilogue and consumed ONLY by a max-pool: its backward rides on the pooling backward (the arg-max
        # is positive iff the pooled value is) instead of a relu_bwd pass over the un-pooled tensor
        for op in plan:
            if op.kind != "maxpool":
                continue
            prod = next((q for q in plan if q.y == op.x), None)
            users = [q for q in plan if q.x == op.x or q.res == op.x]
            if prod is not None and prod.kind == "conv" and prod.relu and len(users) == 1 and FUSE_RELU_POOL:
                op.saved["relu_bwd_here"] = True
                prod.saved["relu_bwd_fused"] = True
        self.plan = plan
        self.alias = alias
        self.out_tid = alias.get(tid("x"), tid("x"))
        self.in_tid = "x@0"
        # static gradient-flow analysis: which tensors need grads, and which dgrad writes accumulate
        written = set()
        for op in reversed(plan):
            op.need_dx = op.x != self.in_tid
            if op.res is not None:
                written.add(op.res)        # fused bn+add writes the residual gradient first (plain store)
            if op.need_dx:
                op.acc_dx = op.x in written
                written.add(op.x)

    def _numel(self, shp):
        return int(math.prod(shp))

    def _alloc(self):
        B, dev = self.max_batch, self.device
        self.act, self.grad = {}, {}
        for op in self.plan:
            self.act[op.y] = torch.empty((B, *op.out_shape), dtype=self.act_dtype, device=dev)
        for op in self.plan:
            for t in (op.x, op.res):
                if t is not None and t != self.in_tid and t not in self.grad:
                    self.grad[t] = torch.empty((B, *self.tshape[t]), dtype=self.act_dtype, device=dev)
        self.grad[self.out_tid] = torch.empty((B, *self.tshape[self.out_tid]), dtype=self.act_dtype, device=dev)
        self.logits = torch.empty((B, self.tshape[self.out_tid][-1]), dtype=torch.float32, device=dev)
        # all per-channel accumulators live in two arenas so one memset per pass re-arms every layer's atomics
        need = [op for op in self.plan if op.kind == "bn" or (op.kind == "conv" and op.saved.get("want_stats"))]
        S = ops.STAT_SLOTS
        tot = sum(2 * op.out_shape[-1] for op in need)
        self.stats_arena = torch.zeros(max(1, tot * S), dtype=torch.float32, device=dev)   # forward: [slots][sum, sum^2][C] per op
        D = BWD_SLOTS
        self.dsum_arena = torch.zeros(max(1, tot * D), dtype=torch.float32, device=dev)    # backward: [slots][sum dy, sum dy*xhat][C] per op
        off = 0
        for op in need:
            c = op.out_shape[-1]
            op.saved["stats"] = self.stats_arena[off * S:(off + 2 * c) * S].view(S, 2, c)
            op.saved["dsum"] = self.dsum_arena[off * D:(off + 2 * c) * D].view(D, 2, c)
            op.saved["mean_rstd"] = torch.zeros(2, c, dtype=torch.float32, device=dev)
            off += 2 * c
        for op in self.plan:
            if op.kind == "maxpool":
                op.saved["idx"] = torch.empty((B, *op.out_shape), dtype=torch.uint8, device=dev)
                if "drop" in op.saved and self.impl["pool"] != "sm100":
                    op.saved["dmask"] = torch.ones((B, *op.out_shape), dtype=torch.uint8, device=dev)   # aten back-end only
            if op.kind == "dropout":
                op.saved["mask"] = torch.empty((B, *op.out_shape), dtype=torch.uint8, device=dev)
        self._bn_src = {}
        # Side branch of a residual block with a projection shortcut (1x1 conv + BatchNorm on the block input): independent of the main
        # path until the fused bn2 + add, so in the forward pass it runs on a second stream forked where the block input is ready --
        # in the captured step graph a parallel branch whose small kernels fill the tails of the main path's conv waves.
        for i, op in enumerate(self.plan):
            if not (FWD_BRANCH and op.kind == "conv" and ".downsample." in (op.name or "")):
                continue
            nxt = self.plan[i + 1] if i + 1 < len(self.plan) else None
            first = next((q for q in self.plan[:i] if q.x == op.x and q is not op), None)            # the block's conv1 reads the same input
            join = next((q for q in self.plan[i + 1:] if nxt is not None and q.res == nxt.y), None)  # the fused bn2 + add
            if nxt is None or nxt.kind != "bn" or nxt.x != op.y or first is None or join is None:
                continue
            first.saved["fork_before"] = True
            op.saved["side_branch"] = nxt.saved["side_branch"] = True
            join.saved["join_before"] = True
        for i, op in enumerate(self.plan):   # a BN op reads the statistics its producer conv accumulated
            if op.kind == "bn":
                prod = next((q for q in self.plan[:i] if q.y == op.x and q.kind == "conv"), None)
                op.saved["producer"] = prod

    # ------------------------------------------------------------------------------------------------------------
    # parameter views
    # ------------------------------------------------------------------------------------------------------------
    def bind(self, w, wb, g, w_buffers=None):
        """Point the net at flat fp32 params ``w``, their bf16 shadow ``wb`` and the flat fp32 gradient ``g``.  ``w_buffers``: flat
        vector that holds the BatchNorm running statistics (default ``w``) -- the first step of a round reads its PARAMETERS from the
        broadcast buffer but must update the running statistics in the trainer's own vector."""
        self.w, self.wb, self.g = w, wb, g
        lay = self.layout
        self.pw = {p.name: lay.view(w, p) for p in lay.params}
        self.pw.update({b.name: lay.view(w if w_buffers is None else w_buffers, b) for b in lay.buffers})
        self.pwb = {p.name: lay.view(wb, p) for p in lay.params} if wb is not None else {}
        self.pg = {p.name: lay.view(g, p) for p in lay.params} if g is not None else {}

    def T(self, t, B):
        return self.act[t][:B] if t != self.in_tid else self._x      # the input is handed in already sized for the batch

    def stem_geometry(self):
        """(k, pad, Ho, Wo) when the first layer takes the im2col stem path on this back-end (the trainer then lets the batch-assembly
        kernel write the im2col matrix directly and passes it as the network input), else None."""
        op = self.plan[0]
        if op.kind != "conv" or op.x != self.in_tid or self.impl["conv_fwd"] != "sm100" or self.impl["conv_wgrad"] != "sm100":
            return None
        return ops.stem_geometry(op.in_shape, op.attrs)

    def G(self, t, B):
        return self.grad[t][:B]

    # ------------------------------------------------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------------------------------------------------
    def forward(self, x_nhwc, train: bool):
        """``x_nhwc``: [B,H,W,C] bf16 (channels of the first conv, un-padded).  Returns fp32 logits [B,classes]."""
        out = self.forward_raw(x_nhwc, train)
        B = out.shape[0]
        self.logits[:B].copy_(out)
        return self.logits[:B]

    def forward_raw(self, x_nhwc, train: bool):
        """Forward pass; returns the head's output [B,classes] in the activation dtype, in place in its activation buffer (the
        training step hands it straight to the loss kernel -- no fp32 staging copy).  ``x_nhwc``: [B,H,W,C], or the first layer's
        im2col matrix [B*Ho*Wo, 64] when ``stem_geometry()`` is not None (batch = rows / (Ho*Wo))."""
        B = x_nhwc.shape[0] if x_nhwc.dim() == 4 else x_nhwc.shape[0] // (self.plan[0].out_shape[0] * self.plan[0].out_shape[1])
        self._x, self._B, self._train = x_nhwc, B, train
        self._epoch = getattr(self, "_epoch", 0) + 1     # forward-pass id: lets stride-2 convs share their parity-split input copy
        if train:
            ops.zero_(self.stats_arena)
        branch = FWD_BRANCH and self.device.type == "cuda" and ops.nn.USE_STRIDED_TMA and self.impl["conv_fwd"] == "sm100"
        if branch and getattr(self, "_branch_stream", None) is None:
            self._branch_stream = torch.cuda.Stream(self.device)
        for i, op in enumerate(self.plan):
            if branch and op.saved.get("fork_before"):
                self._branch_stream.wait_stream(torch.cuda.current_stream(self.device))      # the block input is final
            if branch and op.saved.get("join_before"):
                torch.cuda.current_stream(self.device).wait_stream(self._branch_stream)      # shortcut output ready for bn2 + add
            if branch and op.saved.get("side_branch"):
                with torch.cuda.stream(self._branch_stream):
                    getattr(self, "_fwd_" + op.kind)(op, B, train)
            else:
                getattr(self, "_fwd_" + op.kind)(op, B, train)
            if i == 0 and self.after_first_op is not None:
                self.after_first_op()        # hand-off: acquire the rest of the broadcast once the first-layer GEMM is queued
        return self.T(self.out_tid, B).reshape(B, -1)

    def dlogits_buffer(self, B):
        """Gradient buffer of the head's output ([B,classes], activation dtype): the loss kernel writes into it directly."""
        return self.G(self.out_tid, B).reshape(B, -1)

    def backward(self, dlogits):
        """``dlogits`` [B,classes] (already scaled by 1/B).  Fills the flat gradient buffer."""
        B = dlogits.shape[0]
        gout = self.G(self.out_tid, B)
        if dlogits.data_ptr() != gout.data_ptr():
            gout.copy_(dlogits.reshape(gout.shape))
        ops.zero_(self.g)        # wgmma weight gradients are added into the flat buffer
        ops.zero_(self.dsum_arena)
        self._side = None
        if WGRAD_OVERLAP and self.device.type == "cuda":
            if getattr(self, "_side_stream", None) is None:
                self._side_stream = torch.cuda.Stream(self.device)
            self._side = self._side_stream
            self._side.wait_stream(torch.cuda.current_stream(self.device))       # the flat gradient is zeroed
        branch = (BWD_BRANCH and FWD_BRANCH and self.device.type == "cuda" and ops.nn.USE_STRIDED_TMA and self.impl["conv_fwd"] == "sm100"
                  and getattr(self, "_branch_stream", None) is not None)
        cur = torch.cuda.current_stream(self.device) if branch else None
        for op in reversed(self.plan):
            # projection shortcut (see _alloc): its backward -- BatchNorm backward, 1x1 weight and data gradients -- only needs the
            # residual gradient that the fused bn2 + add backward just wrote, and must be complete before conv1's data gradient
            # ACCUMULATES into the block-input gradient the shortcut's data gradient stored first
            if branch and op.saved.get("fork_before"):
                cur.wait_stream(self._branch_stream)
            if branch and op.saved.get("side_branch"):
                if op.kind == "bn":
                    self._branch_stream.wait_stream(cur)
                with torch.cuda.stream(self._branch_stream):
                    getattr(self, "_bwd_" + op.kind)(op, B)
            else:
                getattr(self, "_bwd_" + op.kind)(op, B)
        if self._side is not None:
            torch.cuda.current_stream(self.device).wait_stream(self._side)       # every weight gradient has landed before the optimizer
            self._side = None

    # ---- conv ---------------------------------------------------------------------------------------------------
    def _epilogue_stats_free(self, op):
        """BatchNorm statistics in the conv epilogue cost nothing where the conv runs the generic kernel's TMA-store epilogue: the
        column sums are taken from the staged tile while the TMA unit drains it (gemm.cu).  That is every stride-1 conv on whole
        64-channel groups except the 64-channel 3x3 layers (halo kernel) -- ResNet-18: 9 of 20 BatchNorm inputs; the others keep the
        streaming statistics pass."""
        if not EPILOGUE_BN_STATS or self.impl["conv_fwd"] != "sm100":
            return False
        a = op.attrs
        return a.get("stride", 1) == 1 and a["cin"] % 64 == 0 and a["cout"] % 64 == 0 and not (a["k"] == 3 and a["cin"] == 64)

    def _fwd_conv(self, op, B, train):
        a = op.attrs
        x, y = self.T(op.x, B), self.T(op.y, B)
        bias = self.pw.get(op.name + ".bias")
        # BatchNorm statistics: fused into the conv epilogue (FUSE_BN_STATS) or taken by one streaming pass over the conv output
        # while it is still L2-resident (default: cheaper than the in-epilogue reduction)
        stats = op.saved.get("stats") if (train and op.saved.get("want_stats") and (self.fuse_bn_stats or self._epilogue_stats_free(op))) else None
        op.saved["stats_done"] = stats is not None
        if self.impl["conv_fwd"] == "sm100" and ops.conv_supported(op.in_shape, a, "fwd"):
            ops.conv2d_fwd_sm100(x, self.pwb[op.name + ".weight"], bias, y, a.get("stride", 1), a.get("pad", 0), op.relu, stats, tag=(id(self), op.name),
                                 zero_stats=False, s2d_epoch=self._epoch, wait=self.first_wait if (op is self.plan[0] and x.dim() == 2) else None)
            return
        if self.impl["conv_fwd"] == "sm100":
            ops.note_fallback("conv_fwd", f"{op.name} in={op.in_shape} {a}")
        wt = self.pwb[op.name + ".weight"].permute(0, 3, 1, 2)
        out = F.conv2d(x.permute(0, 3, 1, 2), wt, bias.to(self.act_dtype) if bias is not None else None, a.get("stride", 1), a.get("pad", 0))
        if op.relu:
            out = F.relu(out)
        y.copy_(out.permute(0, 2, 3, 1))
        if stats is not None:
            yf = y.float().reshape(-1, y.shape[-1])
            stats[0, 0].copy_(yf.sum(0)); stats[0, 1].copy_((yf * yf).sum(0))   # slot 0; the others stay zero

    def _bwd_conv(self, op, B):
        a = op.attrs
        x, y, dy = self.T(op.x, B), self.T(op.y, B), self.G(op.y, B)
        if op.relu and not op.saved.get("relu_bwd_fused"):  # dy <- dy * (y > 0), in place (y is the post-ReLU output)
            ops.relu_bwd_(dy, y, self.impl["bn"])
        name = op.name + ".weight"
        gw, gb = self.pg[name], self.pg.get(op.name + ".bias")
        s, p = a.get("stride", 1), a.get("pad", 0)
        if self.impl["conv_wgrad"] == "sm100" and ops.conv_supported(op.in_shape, a, "wgrad"):
            if getattr(self, "_side", None) is not None:
                self._side.wait_stream(torch.cuda.current_stream(self.device))   # dy (and its ReLU mask) is final
                with torch.cuda.stream(self._side):
                    ops.conv2d_wgrad_sm100(x, dy, gw, gb, s, p, tag=(id(self), op.name), zero=False)
            else:
                ops.conv2d_wgrad_sm100(x, dy, gw, gb, s, p, tag=(id(self), op.name), zero=False)
        else:
            if self.impl["conv_wgrad"] == "sm100":
                ops.note_fallback("conv_wgrad", f"{op.name} in={op.in_shape} {a}")
            _, dw, db = torch.ops.aten.convolution_backward(
                dy.permute(0, 3, 1, 2), x.permute(0, 3, 1, 2), self.pwb[name].permute(0, 3, 1, 2),
                [a["cout"]] if gb is not None else None, [s, s], [p, p], [1, 1], False, [0, 0], 1, [False, True, gb is not None])
            gw.copy_(dw.permute(0, 2, 3, 1))
            if gb is not None:
                gb.copy_(db)
        if not op.need_dx:
            return
        dx = self.G(op.x, B)
        if self.impl["conv_dgrad"] == "sm100" and ops.conv_supported(op.in_shape, a, "dgrad"):
            ops.conv2d_dgrad_sm100(dy, self.pwb[name], dx, s, p, op.acc_dx)
            return
        if self.impl["conv_dgrad"] == "sm100":
            ops.note_fallback("conv_dgrad", f"{op.name} in={op.in_shape} {a}")
        di, _, _ = torch.ops.aten.convolution_backward(
            dy.permute(0, 3, 1, 2), x.permute(0, 3, 1, 2), self.pwb[name].permute(0, 3, 1, 2), None, [s, s], [p, p], [1, 1],
            False, [0, 0], 1, [True, False, False])
        di = di.permute(0, 2, 3, 1)
        if op.acc_dx:
            dx.add_(di)
        else:
            dx.copy_(di)

    # ---- batch norm (+ residual + relu) ------------------------------------------------------------------------------
    def _fwd_bn(self, op, B, train):
        a = op.attrs
        x, y = self.T(op.x, B), self.T(op.y, B)
        res = self.T(op.res, B) if op.res is not None else None
        gamma, beta = self.pw[op.name + ".weight"], self.pw[op.name + ".bias"]
        rm, rv = self.pw[op.name + ".running_mean"], self.pw[op.name + ".running_var"]
        prod = op.saved["producer"]
        stats = prod.saved["stats"] if (train and prod is not None and prod.saved.get("stats_done")) else None
        if stats is not None and not self.fuse_bn_stats:
            stats = stats[0:EPI_STAT_SLOTS]     # the TMA-store epilogue spreads its atomics over this prefix only (gemm.cu, same variable)
        count = x.numel() // x.shape[-1]
        ops.bn_fwd(x, y, res, gamma, beta, rm, rv, stats, op.saved["mean_rstd"], count, a.get("eps", 1e-5),
                   a.get("momentum", 0.1), train, op.relu, self.impl["bn"],
                   stats_buf=op.saved["stats"][0:FWD_SLOTS] if train else None)   # first slots of the (pre-zeroed) statistics arena

    def _bwd_bn(self, op, B):
        x, y, dy = self.T(op.x, B), self.T(op.y, B), self.G(op.y, B)
        dres = self.G(op.res, B) if op.res is not None else None
        dx = self.G(op.x, B)
        gamma = self.pw[op.name + ".weight"]
        ops.bn_bwd(dy, y, x, gamma, op.saved["mean_rstd"], op.saved["dsum"], dx, dres,
                   self.pg[op.name + ".weight"], self.pg[op.name + ".bias"], op.relu, self.impl["bn"], zero_dsum=False,
                   beta=self.pw[op.name + ".bias"])

    # ---- pooling ---------------------------------------------------------------------------------------------------
    def _drop(self, op, train=True):
        """(p, seed, step counter, node id) of the dropout fused into ``op`` (None in evaluation mode / when nothing is fused)."""
        d = op.saved.get("drop")
        return (d[0], self.seed, self.step_counter, d[1]) if (d is not None and train) else None

    def _fwd_maxpool(self, op, B, train):
        drop = self._drop(op, train)
        op.saved["drop_on"] = drop is not None
        mask = op.saved["dmask"][:B] if (drop is not None and "dmask" in op.saved) else None
        ops.maxpool2_fwd(self.T(op.x, B), self.T(op.y, B), op.saved["idx"][:B], self.impl["pool"], drop, mask)

    def _bwd_maxpool(self, op, B):
        drop = self._drop(op, op.saved.get("drop_on", False))
        mask = op.saved["dmask"][:B] if (drop is not None and "dmask" in op.saved) else None
        ops.maxpool2_bwd(self.G(op.y, B), op.saved["idx"][:B], self.G(op.x, B), self.impl["pool"], drop, mask,
                         relu_out=self.T(op.y, B) if op.saved.get("relu_bwd_here") else None)

    def _fwd_avgpool(self, op, B, train):
        ops.avgpool_fwd(self.T(op.x, B), self.T(op.y, B), self.impl["pool"])

    def _bwd_avgpool(self, op, B):
        ops.avgpool_bwd(self.G(op.y, B), self.G(op.x, B), self.impl["pool"])

    # ---- dropout ---------------------------------------------------------------------------------------------------
    def _fwd_dropout(self, op, B, train):
        x, y = self.T(op.x, B), self.T(op.y, B)
        if not train:
            y.copy_(x.reshape(y.shape))
            return
        ops.dropout_fwd(x.reshape(B, -1), y.reshape(B, -1), op.saved["mask"][:B].reshape(B, -1), op.attrs["p"], self.seed,
                        self.step_counter, op.node, self.impl["dropout"])

    def _bwd_dropout(self, op, B):
        ops.dropout_bwd(self.G(op.y, B).reshape(B, -1), op.saved["mask"][:B].reshape(B, -1), self.G(op.x, B).reshape(B, -1),
                        op.attrs["p"], self.impl["dropout"])

    # ---- linear -----------------------------------------------------------------------------------------------------
    def _fwd_linear(self, op, B, train):
        x, y = self.T(op.x, B).reshape(B, -1), self.T(op.y, B)
        drop = self._drop(op, train)
        op.saved["drop_on"] = drop is not None
        ops.linear_fwd(x, self.pwb[op.name + ".weight"], self.pw.get(op.name + ".bias"), y, op.relu, self.impl["linear"], drop)

    def _bwd_linear(self, op, B):
        x, y, dy = self.T(op.x, B).reshape(B, -1), self.T(op.y, B), self.G(op.y, B)
        if op.relu:
            # fused dropout: y = relu(z) * keep / (1-p) -> (y > 0) is the ReLU mask AND the keep mask; the gradient carries 1/(1-p)
            scale = 1.0 / (1.0 - op.saved["drop"][0]) if op.saved.get("drop_on", False) else 1.0
            ops.relu_bwd_(dy, y, self.impl["bn"], scale)
        dx = self.G(op.x, B).reshape(B, -1) if op.need_dx else None
        ops.linear_bwd(x, dy, self.pwb[op.name + ".weight"], dx, self.pg[op.name + ".weight"], self.pg.get(op.name + ".bias"),
                       op.acc_dx, self.impl["linear"], zero=False)


class NativeTrainer:
    """Trainer with the TorchTrainer interface whose forward/backward is ``NativeNet``."""
    name = "native"

    def __init__(self, layout, args, device, max_shard: int, impl="auto"):
        self.layout, self.args = layout, args
        self.device = torch.device(device)
        assert self.device.type == "cuda", "the native trainer runs on sm_90a devices only"
        n = layout.n_total
        self.w = torch.zeros(n, dtype=torch.float32, device=device)
        self.wb = torch.zeros(n, dtype=torch.bfloat16, device=device)
        self.g = torch.zeros(n, dtype=torch.float32, device=device)
        self.m = torch.zeros(n, dtype=torch.float32, device=device)
        self.bs = args.bs
        self.net = NativeNet(layout, device, self.bs, impl, seed=args.seed)
        self.net.bind(self.w, self.wb, self.g)
        self.opt = ops.FlatSGD(n, device, args.client_lr, args.client_moment, 10.0, args.clip, n_pgd=layout.n_vote)
        self.loss_sum = torch.zeros(1, dtype=torch.float32, device=device)
        self.use_graphs = not args.no_graphs
        self.max_shard = max_shard
        self.perm = torch.zeros(max(1, max_shard), dtype=torch.int64, device=device)
        self.cursor = torch.zeros(1, dtype=torch.int32, device=device)
        self.y = torch.zeros(self.bs, dtype=torch.int64, device=device)
        C, H, W = layout.in_shape
        self.x = torch.zeros(self.bs, H, W, C, dtype=ACT, device=device)
        # tiny-K first layer: the batch-assembly kernel writes the stem convolution's im2col matrix directly (gather_im2col)
        self.stem = self.net.stem_geometry()
        self.xA = torch.zeros(self.bs * self.stem[2] * self.stem[3], 64, dtype=ACT, device=device) if self.stem else None
        self._graphs = {}
        self._eval_nets = {}
        self.bcast = None             # round hand-off source (parallel.FusedAggregator) once attach_broadcast() was called

    # ---- round hand-off fused with the first local step ---------------------------------------------------------------------
    def attach_broadcast(self, fused):
        """Fuse the parameter hand-off of a round with the first local step (SURVEY.md A9 / 5.8 "broadcast fused with the first GEMM").
        Instead of a ``round_init`` pass (w <- w_global, bf16 shadow, m <- 0), the FIRST step of every agent reads its parameters
        straight from the broadcast buffer of the aggregator -- fp32 ``w_global`` and the bf16 operand shadow that the aggregation
        kernels of all GPUs multicast into every rank -- and its optimizer kernel starts from zero momentum.  The step's first kernel
        that needs parameters is the stem convolution's GEMM: its producer warp acquires the ready word(s) of the slice(s) holding the
        stem filter (in-kernel ``ld.acquire.sys`` spin) and starts while the remaining slices are still landing; a one-warp
        ``acquire_slices`` kernel queued behind it waits for the rest and seeds the BatchNorm running statistics.  Needs the im2col
        stem (every zoo model has one) and the bf16 shadow."""
        if self.stem is None or fused.w_bf16 is None:
            return False
        self.bcast = fused
        return True

    def _bind_first(self, w0):
        f = self.bcast
        self.net.bind(f.w_global, f.w_bf16, self.g, w_buffers=self.w)
        lay = self.layout
        first_w = lay.by_name[self.net.plan[0].name + ".weight"]
        lo, hi = f.slices_of(first_w.offset, first_w.offset + first_w.numel)
        self.net.first_wait = (f.ready_ptr, lo, hi, f.epoch_dev) if f.ready_ptr else None
        tail_src, tail_dst = f.w_global[lay.n_vote:], self.w[lay.n_vote:]
        self.net.after_first_op = lambda: ops.ext().acquire_slices(f.ready_ptr, 0, max(0, f.n_slices - 1), f.epoch_dev, tail_src, tail_dst)

    def _bind_normal(self):
        self.net.bind(self.w, self.wb, self.g)
        self.net.first_wait = None
        self.net.after_first_op = None

    def _step(self, dataset, B, w0, first=False):
        if first:
            self._bind_first(w0)
        meta = dataset.meta
        if self.stem is not None:
            k, pad, Ho, Wo = self.stem
            xin = self.xA[:B * Ho * Wo]
            ops.gather_im2col(dataset.data, self.perm, meta.mean, meta.std, k, pad, xin, cursor=self.cursor, targets=dataset.targets,
                              out_labels=self.y, batch=B)
        else:
            xin = self.x[:B]
            ops.gather_normalize(dataset.data, self.perm, meta.mean, meta.std, out=xin, nhwc=True, cursor=self.cursor,
                                 targets=dataset.targets, out_labels=self.y, batch=B)
        logits = self.net.forward_raw(xin, True)                              # bf16 [B,classes], in the head's activation buffer
        _, dl = ops.softmax_xent(logits, self.y[:B], True, self.loss_sum, dlogits=self.net.dlogits_buffer(B))
        self.net.backward(dl)
        self.opt.step(self.w, self.g, self.m, w0=w0, w_bf16=self.wb, w_in=self.bcast.w_global if first else None)
        ops.ext().advance_cursor(self.cursor, B, self.net.step_counter)       # next batch; next Philox step for the dropout masks
        if first:
            self._bind_normal()

    def _get_graph(self, dataset, B, w0, first=False):
        key = (B, dataset.data.data_ptr(), w0.data_ptr(), bool(first))
        if key in self._graphs:
            return self._graphs[key]
        keep = (self.w.clone(), self.wb.clone(), self.m.clone(), self.cursor.clone(), self.loss_sum.clone(),
                self.net.step_counter.clone())
        self.perm.zero_()   # warm-up / capture must only touch valid sample indices (perm may hold another dataset's indices)
        s = torch.cuda.Stream(self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(3):
                self.cursor.zero_()
                c0 = ops.launch_calls()
                self._step(dataset, B, w0, first)
                self._launches = ops.launch_calls() - c0
        torch.cuda.current_stream(self.device).wait_stream(s)
        self.cursor.zero_()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, capture_error_mode="thread_local"):
            self._step(dataset, B, w0, first)
        self.w.copy_(keep[0]); self.wb.copy_(keep[1]); self.m.copy_(keep[2]); self.cursor.copy_(keep[3])
        self.loss_sum.copy_(keep[4]); self.net.step_counter.copy_(keep[5])
        self._graphs[key] = graph
        return graph

    def train_agent(self, agent, w_global, out, rnd: int = 0):
        args, bs = self.args, self.bs
        dataset, n = agent.dataset, agent.n_data
        self.loss_sum.zero_()
        graphs = self.use_graphs and n <= self.max_shard
        fused = self.bcast is not None and w_global.data_ptr() == self.bcast.w_global.data_ptr()
        if graphs:
            full = self._get_graph(dataset, bs, w_global) if n >= bs else None
            tail = self._get_graph(dataset, n % bs, w_global) if n % bs else None
            if fused:     # first step of the round: parameters from the broadcast buffer, zero momentum (no round_init pass)
                first_g = self._get_graph(dataset, bs if n >= bs else n % bs, w_global, first=True)
        if not fused:
            ops.round_init(w_global, self.w, self.wb, self.m)
        # dropout Philox stream = (seed, step counter, node): start every (agent, round) at its own counter so agents trained in
        # the same round -- on different GPUs or one after another -- draw independent masks, as the reference's agents do from
        # one sequential RNG (src/federated.py:68-72); the captured graphs increment the device counter once per step
        self.net.step_counter.fill_(dropout_stream_base(args.seed, agent.id, rnd))
        steps = 0
        for ep in range(args.local_ep):
            idx = agent.epoch_indices(args.seed, rnd, ep)
            self.perm[:n].copy_(idx)
            self.cursor.zero_()
            for b in range(n // bs):
                is_first = fused and ep == 0 and b == 0
                if graphs:
                    (first_g if is_first else full).replay()
                else:
                    self._step(dataset, bs, w_global, first=is_first)
            if n % bs:
                is_first = fused and ep == 0 and n < bs
                if graphs:
                    (first_g if is_first else tail).replay()
                else:
                    self._step(dataset, n % bs, w_global, first=is_first)
            steps += (n + bs - 1) // bs
        if out.data_ptr() != self.w.data_ptr():
            out.copy_(self.w)
        return {"loss_sum": self.loss_sum, "steps": steps}

    def launches_per_step(self):
        """Calls into our extension per local step (every call launches at least one of our kernels), measured during
        the eager warm-up step that precedes graph capture."""
        return getattr(self, "_launches", 0)

    @torch.no_grad()
    def eval_forward(self, w):
        """Eval-mode forward of parameters ``w`` through the native executor (running BN statistics, no dropout)."""
        key = w.data_ptr()
        if key not in self._eval_nets:
            net = NativeNet(self.layout, self.device, self.bs, self.net.impl, seed=self.args.seed)
            self._eval_nets = {key: (net, torch.zeros(self.layout.n_total, dtype=ACT, device=self.device))}
        net, wb = self._eval_nets[key]
        wb.copy_(w)
        net.bind(w, wb, None)

        def fwd(x_nchw):
            x = x_nchw.permute(0, 2, 3, 1).to(ACT).contiguous()
            return net.forward(x, False).clone()
        return fwd
