"""GroupNorm models (resnet18_gn / resnet34_gn / vgg11_gn / vgg16_gn) on CPU: flat layout, the torch executor against an independent
``torch.nn`` definition, the native plan against autograd, the contract of the GroupNorm bindings (emulated extension) and a few
engine rounds with the RLR defence.  The sm_90a kernels themselves are tested in tests/test_gpu_groupnorm.py."""
import pytest
import torch
import torch.nn as tnn
import torch.nn.functional as F

import rlr_b200  # noqa: F401
from rlr_b200 import ops
from rlr_b200.models import GraphNet, get_layout
from rlr_b200.models.native import NativeNet
from rlr_b200.ops import nn

GN_MODELS = ("resnet18_gn", "resnet34_gn", "vgg11_gn", "vgg16_gn")


@pytest.mark.parametrize("name", GN_MODELS)
def test_gn_layouts_have_no_buffers_and_bn_twin_parameters(name):
    lay, twin = get_layout(name), get_layout(name[:-3])
    assert lay.n_params == twin.n_params
    assert [(p.name, p.shape) for p in lay.params] == [(p.name, p.shape) for p in twin.params]
    assert lay.n_buffers == 0 and lay.buffers == [] and lay.n_total == lay.n_vote
    assert {p.kind for p in lay.params if p.kind.startswith(("gn", "bn"))} == {"gn_w", "gn_b"}
    assert all(nd.attrs["groups"] == 32 for nd in lay.nodes if nd.op == "gn")
    if name == "resnet18_gn":
        assert lay.n_params == 11_173_962
    w = lay.init_(torch.zeros(lay.n_total), 0)
    assert all(float(lay.view(w, p).min()) == 1.0 for p in lay.params if p.kind == "gn_w")
    assert all(float(lay.view(w, p).abs().max()) == 0.0 for p in lay.params if p.kind == "gn_b")


# ---- independent oracle: plain torch.nn definitions (parameters registered in the reference vector's order) ----------------------
class _Block(tnn.Module):
    def __init__(self, cin, cout, stride):
        super().__init__()
        self.conv1 = tnn.Conv2d(cin, cout, 3, stride, 1, bias=False)
        self.bn1 = tnn.GroupNorm(32, cout)
        self.conv2 = tnn.Conv2d(cout, cout, 3, 1, 1, bias=False)
        self.bn2 = tnn.GroupNorm(32, cout)
        self.downsample = (tnn.Sequential(tnn.Conv2d(cin, cout, 1, stride, bias=False), tnn.GroupNorm(32, cout))
                           if stride != 1 or cin != cout else None)

    def forward(self, x):
        out = F.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        return F.relu(out + (self.downsample(x) if self.downsample is not None else x))


class _ResNet18GN(tnn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = tnn.Conv2d(3, 64, 3, 1, 1, bias=False)
        self.bn1 = tnn.GroupNorm(32, 64)
        cin, layers = 64, []
        for cout, stride in ((64, 1), (128, 2), (256, 2), (512, 2)):
            layers.append(tnn.Sequential(_Block(cin, cout, stride), _Block(cout, cout, 1)))
            cin = cout
        self.layer1, self.layer2, self.layer3, self.layer4 = layers
        self.fc = tnn.Linear(512, 10)

    def forward(self, x):
        x = F.relu(self.bn1(self.conv1(x)))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.fc(x.mean((2, 3)))


class _VGG11GN(tnn.Module):
    def __init__(self):
        super().__init__()
        mods, cin = [], 3
        for v in (64, "M", 128, "M", 256, 256, "M", 512, 512, "M", 512, 512, "M"):
            if v == "M":
                mods.append(tnn.MaxPool2d(2, 2))
            else:
                mods += [tnn.Conv2d(cin, v, 3, padding=1), tnn.GroupNorm(32, v), tnn.ReLU()]
                cin = v
        self.features = tnn.Sequential(*mods)
        self.classifier = tnn.Linear(512, 10)

    def forward(self, x):
        return self.classifier(self.features(x).flatten(1))


@pytest.mark.parametrize("name,oracle", [("resnet18_gn", _ResNet18GN), ("vgg11_gn", _VGG11GN)])
def test_graphnet_matches_independent_torch_definition(name, oracle):
    torch.manual_seed(0)
    lay = get_layout(name)
    w = lay.init_(torch.zeros(lay.n_total), 4)
    w[: lay.n_vote] += 0.05 * torch.randn(lay.n_vote)              # non-trivial affine parameters
    g = torch.zeros(lay.n_total)
    net = GraphNet(lay, w, g).train()
    ref = oracle()
    assert [n for n, _ in ref.named_parameters()] == [p.name for p in lay.params]
    torch.nn.utils.vector_to_parameters(lay.to_reference_vector(w), ref.parameters())
    with torch.no_grad():
        back = lay.from_reference_vector(torch.nn.utils.parameters_to_vector(ref.parameters()), torch.zeros(lay.n_total))
    assert all(torch.equal(lay.view(back, p), lay.view(w, p)) for p in lay.params)
    x, y = torch.randn(5, 3, 32, 32), torch.randint(0, 10, (5,))
    out, out_ref = net(x), ref(x)
    torch.testing.assert_close(out, out_ref, rtol=1e-4, atol=1e-4)
    F.cross_entropy(out, y).backward()
    F.cross_entropy(out_ref, y).backward()
    g_ref = torch.cat([p.grad.reshape(-1) for p in ref.parameters()])
    torch.testing.assert_close(lay.to_reference_vector(g), g_ref, rtol=1e-3, atol=1e-5)


@pytest.mark.parametrize("name,tol", [("resnet18_gn", 3e-2), ("vgg11_gn", 1e-4)])
def test_native_plan_matches_autograd_and_eval_equals_train(name, tol):
    torch.manual_seed(0)
    lay = get_layout(name)
    w = lay.init_(torch.zeros(lay.n_total), 1)
    w[: lay.n_vote] += 0.02 * torch.randn(lay.n_vote)
    g_ref, g_nat = torch.zeros(lay.n_total), torch.zeros(lay.n_total)
    ref = GraphNet(lay, w.clone(), g_ref).train()
    nat = NativeNet(lay, "cpu", 8, impl="aten", act_dtype=torch.float32)
    w2 = w.clone()
    nat.bind(w2, w2, g_nat)
    x, y = torch.randn(6, 3, 32, 32), torch.randint(0, 10, (6,))
    logits_ref = ref(x)
    F.cross_entropy(logits_ref, y).backward()
    xh = x.permute(0, 2, 3, 1).contiguous()
    logits = nat.forward(xh, True).clone()
    _, dl = ops.softmax_xent(logits, y)
    nat.backward(dl)
    torch.testing.assert_close(logits, logits_ref.detach(), atol=1e-4, rtol=1e-4)
    # ResNet: fp32 rounding differences flip a few ReLU masks near zero in the residual chain (as for the BatchNorm twin) -> looser bound
    assert float((g_nat - g_ref).abs().max()) <= tol * max(1.0, float(g_ref.abs().max()))
    assert float((g_nat - g_ref).norm() / g_ref.norm()) < 2e-2
    torch.testing.assert_close(nat.forward(xh, False), logits)                  # no running state: evaluation == training forward
    assert torch.equal(w2, w)                                                    # and the forward writes nothing into the flat vector


def test_gn_plan_shape_resnet18():
    lay = get_layout("resnet18_gn")
    net = NativeNet(lay, "cpu", 4, impl="aten", act_dtype=torch.float32)
    kinds = [op.kind for op in net.plan]
    assert kinds.count("conv") == 20 and kinds.count("gn") == 20 and "bn" not in kinds
    fused_add = [op for op in net.plan if op.kind == "gn" and op.res is not None]
    assert len(fused_add) == 8 and all(op.relu for op in fused_add)
    side = [op for op in net.plan if op.saved.get("side_branch")]
    forks = [op for op in net.plan if op.saved.get("fork_before")]
    assert len(forks) == 3 and [op.kind for op in side] == ["conv", "gn"] * 3
    assert not any(op.saved.get("want_stats") or "stats" in op.saved or "dsum" in op.saved for op in net.plan)
    assert net.stats_arena.numel() == 1 and net.dsum_arena.numel() == 1          # placeholders: no statistics arena
    assert all(op.saved["mean_rstd"].shape == (4, 2, 32) for op in net.plan if op.kind == "gn")


# ---- contract of the gn_fwd / gn_bwd bindings (ops/csrc/gemm_binding.cpp), emulated in fp32 ---------------------------------------
class FakeGnExt:
    def __init__(self):
        self.calls = []

    def gn_fwd(self, x, res, y, gamma, beta, mean_rstd, groups, eps, relu):
        self.calls.append("gn_fwd")
        assert isinstance(groups, int) and isinstance(relu, bool) and mean_rstd.shape == (x.shape[0], 2, groups)
        xn = x.permute(0, 3, 1, 2).float()
        out = F.group_norm(xn, groups, gamma, beta, eps).permute(0, 2, 3, 1)
        if res is not None:
            out = out + res
        y.copy_(out.clamp_min(0) if relu else out)
        xg = xn.reshape(x.shape[0], groups, -1)
        mean_rstd[:, 0] = xg.mean(-1)
        mean_rstd[:, 1] = torch.rsqrt(xg.var(-1, unbiased=False) + eps)

    def gn_bwd(self, dy, y, x, gamma, mean_rstd, dx, dres, dgamma, dbeta, groups, relu):
        self.calls.append("gn_bwd")
        assert (y is not None) == relu
        dz = dy * (y > 0) if relu else dy
        if dres is not None:
            dres.copy_(dz)
        B, C = x.shape[0], x.shape[-1]
        xn = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
        g = gamma.clone().requires_grad_(True)
        b = torch.zeros_like(gamma, requires_grad=True)
        # eps recovered from the saved statistics: rstd = 1 / sqrt(var + eps)
        var = xn.detach().reshape(B, groups, -1).var(-1, unbiased=False)
        eps = float((1.0 / mean_rstd[:, 1] ** 2 - var).mean())
        F.group_norm(xn, groups, g, b, eps).backward(dz.permute(0, 3, 1, 2))
        dx.copy_(xn.grad.permute(0, 2, 3, 1))
        dgamma += g.grad                                                         # ADDED into (binding contract)
        dbeta += b.grad

    def memset_zero(self, t):
        t.zero_()


@pytest.fixture
def fake(monkeypatch):
    ext = FakeGnExt()
    monkeypatch.setattr(nn, "_ext", lambda: ext)
    return ext


@pytest.mark.parametrize("groups,relu,with_res", [(1, True, True), (4, False, False), (16, True, False), (32, False, True)])
def test_gn_wrappers_hand_the_kernels_the_right_problem(fake, groups, relu, with_res):
    torch.manual_seed(groups)
    B, H, W, C = 3, 5, 4, 32
    x = torch.randn(B, H, W, C) * 1.5 + 0.3
    res = torch.randn(B, H, W, C) if with_res else None
    gamma, beta = torch.rand(C) + 0.5, torch.randn(C) * 0.2
    dy = torch.randn(B, H, W, C)
    out = {}
    for impl in ("aten", "sm100"):
        y, mr = torch.empty_like(x), torch.zeros(B, 2, groups)
        nn.gn_fwd(x, y, res, gamma, beta, mr, groups, 1e-5, relu, impl)
        dx, dres = torch.empty_like(x), (torch.empty_like(x) if with_res else None)
        dg, db = torch.full((C,), 0.5), torch.full((C,), -0.25)
        nn.gn_bwd(dy, y, x, gamma, mr, dx, dres, dg, db, groups, relu, impl, zero=False)
        out[impl] = (y, mr, dx, dres, dg, db)
    for a, b in zip(out["aten"], out["sm100"]):
        if a is not None:
            torch.testing.assert_close(b, a, rtol=1e-4, atol=1e-4)
    assert fake.calls == ["gn_fwd", "gn_bwd"]


def test_gn_unsupported_shape_is_a_recorded_fallback(fake, monkeypatch):
    x = torch.randn(2, 3, 3, 12)                                                 # C % 8 != 0: no kernel
    y, mr = torch.empty_like(x), torch.zeros(2, 2, 4)
    ops.reset_fallbacks()
    nn.gn_fwd(x, y, None, torch.ones(12), torch.zeros(12), mr, 4, 1e-5, False, "sm100")
    assert fake.calls == [] and ops.fallback_calls() == {"gn_fwd": 1}
    monkeypatch.setenv("RLR_STRICT", "1")
    with pytest.raises(RuntimeError, match="gn_fwd"):
        nn.gn_fwd(x, y, None, torch.ones(12), torch.zeros(12), mr, 4, 1e-5, False, "sm100")
    ops.reset_fallbacks()


def test_native_plan_drives_gn_bindings_like_the_library_path(fake):
    """Whole resnet18_gn plan with the normalisation layers on the (emulated) kernels against the same plan on the library path:
    catches wrong buffers / ragged-batch views / residual-gradient plumbing in how models/native.py drives gn_fwd / gn_bwd."""
    torch.manual_seed(0)
    lay = get_layout("resnet18_gn")
    w = lay.init_(torch.zeros(lay.n_total), 1)
    w[: lay.n_vote] += 0.02 * torch.randn(lay.n_vote)
    x, t = torch.randn(3, 32, 32, 3), torch.randint(0, 10, (3,))
    res = {}
    for bn_impl in ("aten", "sm100"):
        impl = dict(conv_fwd="aten", conv_dgrad="aten", conv_wgrad="aten", bn=bn_impl, pool="aten", linear="aten", dropout="aten")
        net = NativeNet(lay, "cpu", 4, impl=impl, act_dtype=torch.float32)          # batch 3 of max 4: ragged views
        wi, g = w.clone(), torch.zeros_like(w)
        net.bind(wi, wi.clone(), g)
        logits = net.forward(x, True).clone()
        _, dl = ops.softmax_xent(logits, t)
        net.backward(dl)
        res[bn_impl] = (logits, g.clone())
    torch.testing.assert_close(res["sm100"][0], res["aten"][0], rtol=1e-4, atol=1e-4)
    cos = F.cosine_similarity(res["sm100"][1].double(), res["aten"][1].double(), dim=0)     # ReLU-mask flips near zero: see above
    assert float(cos) > 0.9999, float(cos)
    assert fake.calls.count("gn_fwd") == 20 and fake.calls.count("gn_bwd") == 20


def test_gn_model_engine_rounds_with_rlr_and_checkpoint(tmp_path):
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    ck = str(tmp_path / "ck.pt")
    common = dict(data="cifar10", model="resnet18_gn", synthetic=96, synthetic_val=32, num_agents=3, num_corrupt=1, poison_frac=0.5,
                  robustLR_threshold=2, local_ep=1, bs=16, log_dir="", device="cpu")
    eng = FLEngine(make_args(rounds=2, checkpoint=ck, snap=1, **common), verbose=False)
    lay = eng.layout
    assert lay.n_total == lay.n_vote
    hist = eng.fit()
    _, flipped = eng.round_result()
    assert 0 < flipped <= lay.n_params
    assert 0.0 < hist[-1]["frac_flipped"] <= 1.0
    assert torch.isfinite(eng.w_global).all()
    eng2 = FLEngine(make_args(rounds=3, resume=ck, **common), verbose=False)
    assert eng2.start_round == 3
    assert torch.equal(eng2.w_global, eng.w_global)
    assert len(eng2.fit()) == 1
    eng.close(); eng2.close()
