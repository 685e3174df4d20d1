"""Model IR, flat parameter layout and the PyTorch executor of the IR.

A model is a short list of ``Node``s over named activation slots.  The same IR drives

* ``GraphNet`` (this file): a ``torch.nn.Module`` that interprets the IR with torch ops -- the CPU / oracle /
  "torch trainer" path -- whose parameters are *views into one flat fp32 buffer*, and
* ``models.native.NativeNet``: the sm_90a executor (hand-written forward/backward kernels, no autograd).

Flat layout (one buffer per role: params ``w``, grads ``g``, momentum ``m``):

    [ param_0 | pad | param_1 | pad | ... | (n_vote) | bn running stats ... | pad (n_total) ]

Every tensor starts at a multiple of 64 elements.  Coordinates ``< n_vote`` take part in the sign vote / robust
aggregation; BatchNorm running statistics live behind ``n_vote`` and are plainly averaged (SURVEY.md quirk 13).  GroupNorm
(op ``gn``) has no running state: a model without BatchNorm has ``n_total == n_vote``, every coordinate is voted on.
Because parameters already live in one vector, the reference's ``parameters_to_vector`` / ``vector_to_parameters``
round trips (src/federated.py:59,66,72; src/agent.py:35,56-63; src/aggregation.py:38-40) disappear.

Conv weights are stored OHWI (``[Cout][kh][kw][Cin]``, the K-major GEMM operand layout) and exposed to torch as a
channels-last ``[Cout,Cin,kh,kw]`` view; ``flatten`` uses NHWC order.  ``to_reference_vector`` converts to the
reference's OIHW / NCHW-flatten coordinate order for interop.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch
import torch.nn as nn
import torch.nn.functional as F

ALIGN = 64
TOTAL_ALIGN = 4096


@dataclass
class Node:
    op: str                     # conv | bn | gn | relu | maxpool | avgpool | flatten | dropout | linear | save | add
    name: str = ""
    inp: str = "x"
    out: str = "x"
    attrs: dict = field(default_factory=dict)


@dataclass
class ParamInfo:
    name: str
    shape: tuple        # storage shape (OHWI for conv weights)
    offset: int
    numel: int
    kind: str           # conv_w | linear_w | bias | bn_w | bn_b | bn_mean | bn_var | gn_w | gn_b
    node: int


def _ceil(x, a):
    return (x + a - 1) // a * a


class FlatLayout:
    """Offsets of every parameter / buffer of an IR in the flat vector."""

    def __init__(self, nodes, in_shape):
        self.nodes = nodes
        self.in_shape = tuple(in_shape)  # (C,H,W)
        self.params: list[ParamInfo] = []
        self.buffers: list[ParamInfo] = []
        off = 0

        def add(lst, name, shape, kind, node):
            nonlocal off
            n = int(math.prod(shape))
            lst.append(ParamInfo(name, tuple(shape), off, n, kind, node))
            off = _ceil(off + n, ALIGN)

        for i, nd in enumerate(nodes):
            a = nd.attrs
            if nd.op == "conv":
                add(self.params, nd.name + ".weight", (a["cout"], a["k"], a["k"], a["cin"]), "conv_w", i)
                if a.get("bias", True):
                    add(self.params, nd.name + ".bias", (a["cout"],), "bias", i)
            elif nd.op == "linear":
                add(self.params, nd.name + ".weight", (a["cout"], a["cin"]), "linear_w", i)
                if a.get("bias", True):
                    add(self.params, nd.name + ".bias", (a["cout"],), "bias", i)
            elif nd.op == "bn":
                add(self.params, nd.name + ".weight", (a["c"],), "bn_w", i)
                add(self.params, nd.name + ".bias", (a["c"],), "bn_b", i)
            elif nd.op == "gn":         # torch.nn.GroupNorm(groups, c, eps, affine=True): per-channel affine, no buffers
                assert a["c"] % a["groups"] == 0, f"{nd.name}: {a['groups']} groups do not divide {a['c']} channels"
                add(self.params, nd.name + ".weight", (a["c"],), "gn_w", i)
                add(self.params, nd.name + ".bias", (a["c"],), "gn_b", i)
        self.n_params = sum(p.numel for p in self.params)        # true parameter count (reference n_model_params)
        self.n_vote = _ceil(off, TOTAL_ALIGN)
        off = self.n_vote
        for i, nd in enumerate(nodes):
            if nd.op == "bn":
                add(self.buffers, nd.name + ".running_mean", (nd.attrs["c"],), "bn_mean", i)
                add(self.buffers, nd.name + ".running_var", (nd.attrs["c"],), "bn_var", i)
        self.n_buffers = sum(b.numel for b in self.buffers)
        self.n_total = _ceil(off, TOTAL_ALIGN)
        self.by_name = {p.name: p for p in self.params + self.buffers}

    # ---- views -------------------------------------------------------------------------------------------
    def view(self, flat, info: ParamInfo):
        return flat[info.offset:info.offset + info.numel].view(info.shape)

    def views(self, flat):
        return {p.name: self.view(flat, p) for p in self.params + self.buffers}

    # ---- init (torch default initialisers, like the reference's plain nn.Conv2d / nn.Linear) ----------------
    def init_(self, flat, seed=0):
        gen = torch.Generator(device="cpu").manual_seed(int(seed))
        cpu = torch.zeros(self.n_total, dtype=torch.float32)
        fan_in = {}
        for p in self.params:
            v = self.view(cpu, p)
            if p.kind in ("conv_w", "linear_w"):
                fi = int(math.prod(p.shape[1:]))
                fan_in[p.node] = fi
                bound = 1.0 / math.sqrt(fi)  # kaiming_uniform_(a=sqrt(5)) == U(-1/sqrt(fan_in), 1/sqrt(fan_in))
                v.uniform_(-bound, bound, generator=gen)
            elif p.kind == "bias":
                bound = 1.0 / math.sqrt(fan_in[p.node])
                v.uniform_(-bound, bound, generator=gen)
            elif p.kind in ("bn_w", "gn_w"):
                v.fill_(1.0)
            else:
                v.zero_()
        for b in self.buffers:
            self.view(cpu, b).fill_(1.0 if b.kind == "bn_var" else 0.0)
        flat.copy_(cpu.to(flat.device))
        return flat

    # ---- interop with the reference's coordinate order -----------------------------------------------------
    def _flatten_perm(self):
        """For the first linear after `flatten`: column permutation NHWC-flatten -> NCHW-flatten, or None."""
        shape = self.in_shape
        c, h, w = shape
        perm = {}
        for i, nd in enumerate(self.nodes):
            a = nd.attrs
            if nd.op == "conv":
                h = (h + 2 * a.get("pad", 0) - a["k"]) // a.get("stride", 1) + 1
                w = (w + 2 * a.get("pad", 0) - a["k"]) // a.get("stride", 1) + 1
                c = a["cout"]
            elif nd.op == "maxpool":
                h, w = h // 2, w // 2
            elif nd.op == "avgpool":
                h, w = 1, 1
            elif nd.op == "flatten":
                # our column j = (y*w + x)*c + ch ; reference column = ch*h*w + y*w + x
                idx = torch.arange(c * h * w).view(c, h, w).permute(1, 2, 0).reshape(-1)
                nxt = next((j for j in range(i + 1, len(self.nodes)) if self.nodes[j].op == "linear"), None)
                if nxt is not None and h * w > 1:
                    perm[nxt] = idx
        return perm

    def to_reference_vector(self, flat):
        """Concatenate parameters in the reference's ``parameters_to_vector`` order/layout (OIHW, NCHW flatten)."""
        perm = self._flatten_perm()
        out = []
        for p in self.params:
            v = self.view(flat, p)
            if p.kind == "conv_w":
                v = v.permute(0, 3, 1, 2)
            elif p.kind == "linear_w" and p.node in perm:
                ref = torch.empty_like(v)
                ref[:, perm[p.node].to(v.device)] = v
                v = ref
            out.append(v.reshape(-1))
        return torch.cat(out)

    def from_reference_vector(self, vec, flat):
        perm = self._flatten_perm()
        off = 0
        for p in self.params:
            src = vec[off:off + p.numel]
            off += p.numel
            dst = self.view(flat, p)
            if p.kind == "conv_w":
                o, kh, kw, i = p.shape
                dst.copy_(src.view(o, i, kh, kw).permute(0, 2, 3, 1))
            elif p.kind == "linear_w" and p.node in perm:
                dst.copy_(src.view(p.shape)[:, perm[p.node].to(src.device)])
            else:
                dst.copy_(src.view(p.shape))
        return flat


def head_index(layout) -> int:
    """Index of the model's last ``linear`` node (the head); its input is the penultimate-layer representation."""
    return max(i for i, nd in enumerate(layout.nodes) if nd.op == "linear")


def feature_dim(layout) -> int:
    """Width d of the penultimate-layer representation: the input features of the last ``linear`` node."""
    return int(layout.nodes[head_index(layout)].attrs["cin"])


def head_slices(layout):
    """``(w_off, b_off, P, d)`` of the model's head (the last ``linear`` node): its weight ``[P][d]`` and bias ``[P]`` in the flat vector.
    DeepSight reads both, so a head without a bias is refused."""
    nd = layout.nodes[head_index(layout)]
    if nd.name + ".bias" not in layout.by_name:
        raise ValueError(f"--aggr deepsight needs a head with a bias; {nd.name} has none")
    a = nd.attrs
    return layout.by_name[nd.name + ".weight"].offset, layout.by_name[nd.name + ".bias"].offset, int(a["cout"]), int(a["cin"])


class GraphNet(nn.Module):
    """PyTorch interpreter of the IR; parameters/buffers are views into the flat buffers ``w`` (and ``g``)."""

    def __init__(self, layout: FlatLayout, w: torch.Tensor, g: torch.Tensor | None = None, compute_dtype=torch.float32):
        super().__init__()
        self.layout = layout
        self.compute_dtype = compute_dtype
        self._names = []
        self.bind(w, g)

    def bind(self, w, g=None):
        """(Re)point every parameter at flat buffer ``w`` and its gradient at ``g``."""
        self.w, self.g = w, g
        for p in self.layout.params:
            key = p.name.replace(".", "__")
            v = self.layout.view(w, p)
            if p.kind == "conv_w":
                v = v.permute(0, 3, 1, 2)  # logical OIHW, channels-last strides
            if key in self._parameters:
                self._parameters[key].data = v
            else:
                self.register_parameter(key, nn.Parameter(v, requires_grad=True))
                self._names.append(key)
            if g is not None:
                gv = self.layout.view(g, p)
                if p.kind == "conv_w":
                    gv = gv.permute(0, 3, 1, 2)
                self._parameters[key].grad = gv
        self._bufs = {b.name: self.layout.view(w, b) for b in self.layout.buffers}

    def P(self, name):
        return self._parameters[name.replace(".", "__")]

    def forward(self, x, tap: bool = False):
        """Logits of ``x`` (fp32); with ``tap`` the input of the last ``linear`` node instead (the penultimate-layer representation
        FLARE compares, fp32 ``[B, d]``), the head itself not run."""
        cd = self.compute_dtype
        slots = {"x": x.to(cd)}
        if x.dim() == 4 and x.is_cuda:
            slots["x"] = slots["x"].contiguous(memory_format=torch.channels_last)
        head = head_index(self.layout) if tap else -1
        for i, nd in enumerate(self.layout.nodes):
            a = nd.attrs
            t = slots[nd.inp]
            if i == head:
                return t.float()
            if nd.op == "conv":
                b = self.P(nd.name + ".bias").to(cd) if a.get("bias", True) else None
                t = F.conv2d(t, self.P(nd.name + ".weight").to(cd), b, stride=a.get("stride", 1), padding=a.get("pad", 0))
            elif nd.op == "bn":
                rm, rv = self._bufs[nd.name + ".running_mean"], self._bufs[nd.name + ".running_var"]
                t = F.batch_norm(t, rm, rv, self.P(nd.name + ".weight"), self.P(nd.name + ".bias"),
                                 self.training, a.get("momentum", 0.1), a.get("eps", 1e-5))
            elif nd.op == "gn":
                # fp32 statistics and affine whatever the compute dtype (the bf16 torch trainer), result cast back
                t = F.group_norm(t.float(), a["groups"], self.P(nd.name + ".weight"), self.P(nd.name + ".bias"),
                                 a.get("eps", 1e-5)).to(cd)
            elif nd.op == "relu":
                t = F.relu(t)
            elif nd.op == "maxpool":
                t = F.max_pool2d(t, 2, 2)
            elif nd.op == "avgpool":
                t = t.mean(dim=(2, 3), keepdim=True)
            elif nd.op == "flatten":
                t = t.permute(0, 2, 3, 1).reshape(t.shape[0], -1)  # NHWC order (see module docstring)
            elif nd.op == "dropout":
                t = F.dropout(t, a["p"], self.training)  # reference Dropout2d on 2-D input == element-wise dropout
            elif nd.op == "linear":
                b = self.P(nd.name + ".bias").to(cd) if a.get("bias", True) else None
                t = F.linear(t, self.P(nd.name + ".weight").to(cd), b)
            elif nd.op == "save":
                pass
            elif nd.op == "add":
                t = t + slots[a["other"]]
            else:
                raise ValueError(nd.op)
            slots[nd.out] = t
        return slots["x"].float()
