"""Local-training executors.

``TorchTrainer`` runs the IR with PyTorch autograd (cuDNN/cuBLAS on GPU): it is the CPU path, the numerical oracle
for the native kernels, and the "ours-in-torch" baseline of BASELINE.md.  Everything around the forward/backward is
already the engine's own: device-resident data + gather kernel, flat buffers, fused clip+SGD(+PGD) kernel, CUDA-graph
capture of the whole step.  ``models.native.NativeTrainer`` replaces forward/backward with sm_90a kernels behind the
same interface.

One local step (reference src/agent.py:41-60): zero grads -> forward -> CE loss -> backward -> clip_grad_norm_(10) ->
SGD(momentum) -> optional PGD projection.  The last partial batch is trained on, not dropped (DataLoader default).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ops
from .models.graph import GraphNet


def _agent_round_seed(seed: int, agent_id: int, rnd: int) -> int:
    return (int(seed) * 1_000_003 + (int(agent_id) + 1) * 7_919 + int(rnd) * 104_729) % (2 ** 63 - 1)


class TorchTrainer:
    name = "torch"

    def __init__(self, layout, args, device, max_shard: int, use_graphs: bool | None = None):
        self.layout, self.args = layout, args
        self.device = torch.device(device)
        cuda = self.device.type == "cuda"
        n = layout.n_total
        self.w = torch.zeros(n, dtype=torch.float32, device=device)
        self.g = torch.zeros(n, dtype=torch.float32, device=device)
        self.m = torch.zeros(n, dtype=torch.float32, device=device)
        self.compute_dtype = torch.bfloat16 if (cuda and args.dtype == "bf16") else torch.float32
        self.net = GraphNet(layout, self.w, self.g, self.compute_dtype)
        self.opt = ops.FlatSGD(n, device, args.client_lr, args.client_moment, 10.0, args.clip, n_pgd=layout.n_vote)
        self.loss_sum = torch.zeros(1, dtype=torch.float32, device=device)
        self.bs = args.bs
        self.use_graphs = cuda and not args.no_graphs if use_graphs is None else use_graphs
        self.max_shard = max_shard
        self._graphs = {}
        self._w0 = None
        if cuda:
            torch.backends.cudnn.benchmark = True
            self.perm = torch.zeros(max(1, max_shard), dtype=torch.int64, device=device)
            self.cursor = torch.zeros(1, dtype=torch.int32, device=device)
            self.y = torch.zeros(self.bs, dtype=torch.int64, device=device)
            self.x = None

    # ---- one optimisation step on a ready batch --------------------------------------------------------------
    def _step(self, x, y, w0):
        self.g.zero_()
        logits = self.net(x)
        loss = F.cross_entropy(logits, y)
        loss.backward()
        self.opt.step(self.w, self.g, self.m, w0=w0)
        self.loss_sum += loss.detach()

    def _graph_body(self, dataset, B, w0):
        meta = dataset.meta
        ops.gather_normalize(dataset.data, self.perm, meta.mean, meta.std, out=self.x[:B], cursor=self.cursor,
                             targets=dataset.targets, out_labels=self.y, batch=B)
        ops.ext().advance_cursor(self.cursor, B)
        self._step(self.x[:B], self.y[:B], w0)

    def _get_graph(self, dataset, B, w0):
        key = (B, dataset.data.data_ptr(), w0.data_ptr())
        if key in self._graphs:
            return self._graphs[key]
        meta = dataset.meta
        if self.x is None:
            self.x = torch.zeros(self.bs, meta.channels, meta.height, meta.width, dtype=torch.float32, device=self.device)
        # warm-up on a side stream (cuDNN autotune, lazy inits), then capture; state is re-initialised afterwards
        keep = (self.w.clone(), self.m.clone(), self.cursor.clone(), self.loss_sum.clone())
        self.perm.zero_()   # warm-up / capture must only touch valid sample indices (perm may hold another dataset's indices)
        s = torch.cuda.Stream(self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(3):
                self.cursor.zero_()
                self._graph_body(dataset, B, w0)
        torch.cuda.current_stream(self.device).wait_stream(s)
        self.cursor.zero_()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, capture_error_mode="thread_local"):
            self._graph_body(dataset, B, w0)
        self.w.copy_(keep[0]); self.m.copy_(keep[1]); self.cursor.copy_(keep[2]); self.loss_sum.copy_(keep[3])
        self._graphs[key] = graph
        return graph

    # ---- public --------------------------------------------------------------------------------------------
    def train_agent(self, agent, w_global, out, rnd: int = 0):
        args, bs = self.args, self.bs
        dataset, n = agent.dataset, agent.n_data
        self.net.train()
        self.loss_sum.zero_()
        steps = 0
        graphs = self.use_graphs and n <= self.max_shard
        if graphs:  # capture (first call only) BEFORE the round state is set up: capture warm-up scribbles on w/m
            full = self._get_graph(dataset, bs, w_global) if n >= bs else None
            tail = self._get_graph(dataset, n % bs, w_global) if n % bs else None
        ops.round_init(w_global, self.w, None, self.m)
        # independent dropout masks per (agent, round): the reference draws them from one sequential RNG (src/federated.py:68-72);
        # here agents of a round run on different ranks that were all seeded alike at start-up
        torch.manual_seed(_agent_round_seed(args.seed, agent.id, rnd))
        for ep in range(args.local_ep):
            idx = agent.epoch_indices(args.seed, rnd, ep)
            if graphs:
                self.perm[:n].copy_(idx)
                self.cursor.zero_()
                for _ in range(n // bs):
                    full.replay()
                if n % bs:
                    tail.replay()
                steps += (n + bs - 1) // bs
            else:
                for start in range(0, n, bs):
                    x, y = dataset.batch(idx[start:start + bs], dtype=torch.float32)
                    self._step(x, y, w_global)
                    steps += 1
        if out.data_ptr() != self.w.data_ptr():
            out.copy_(self.w)
        return {"loss_sum": self.loss_sum, "steps": steps}

    def launches_per_step(self):
        """Number of OUR kernels per local step (gather, cursor, ||g||^2, fused SGD [+ PGD]); forward/backward of this
        trainer are torch/cuDNN library calls and are not counted."""
        return (4 + (1 if self.args.clip > 0 else 0)) if self.device.type == "cuda" else 0

    @torch.no_grad()
    def eval_forward(self, w):
        """``forward(x)`` closure evaluating parameters ``w`` in eval mode (running BN statistics)."""
        net = GraphNet(self.layout, w, None, self.compute_dtype)
        net.eval()
        return lambda x: net(x)


def make_trainer(kind, layout, args, device, max_shard):
    dev = torch.device(device)
    if kind == "auto":
        kind = "torch"
        if dev.type == "cuda":
            try:
                from .models.native import NativeTrainer, native_supported
                if native_supported(layout):
                    kind = "native"
            except ImportError:
                pass
    if kind == "native":
        from .models.native import NativeTrainer
        return NativeTrainer(layout, args, device, max_shard)
    return TorchTrainer(layout, args, device, max_shard)
