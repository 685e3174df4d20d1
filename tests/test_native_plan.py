"""The native executor's plan (fusion, hand-derived backward, residual gradient accumulation) against PyTorch autograd, run on
CPU in fp32 through the `aten` back-end.  The sm_90a kernels behind the same plan are checked in tests/test_gpu_native.py."""
import pytest
import torch

from rlr_b200 import ops
from rlr_b200.models import GraphNet, get_layout
from rlr_b200.models.native import NativeNet


@pytest.mark.parametrize("name,tol", [("cnn_mnist", 1e-5), ("cnn_cifar", 1e-5), ("vgg11", 1e-4), ("resnet18", 3e-2), ("vgg16", 3e-2), ("resnet34", 1e-1)])
def test_plan_matches_autograd(name, tol):
    torch.manual_seed(0)
    lay = get_layout(name)
    for nd in lay.nodes:
        if nd.op == "dropout":
            nd.attrs["p"] = 0.0
    w = lay.init_(torch.zeros(lay.n_total), 1)
    g_ref, g_nat = torch.zeros(lay.n_total), torch.zeros(lay.n_total)
    ref = GraphNet(lay, w.clone(), g_ref)
    ref.train()
    nat = NativeNet(lay, "cpu", 8, impl="aten", act_dtype=torch.float32)
    w2 = w.clone()
    nat.bind(w2, w2, g_nat)
    C, H, W = lay.in_shape
    x, y = torch.randn(6, C, H, W), torch.randint(0, 10, (6,))
    logits_ref = ref(x)
    torch.nn.functional.cross_entropy(logits_ref, y).backward()
    logits = nat.forward(x.permute(0, 2, 3, 1).contiguous(), True)
    _, dl = ops.softmax_xent(logits, y)
    nat.backward(dl)
    nv = lay.n_vote
    torch.testing.assert_close(logits, logits_ref.detach(), atol=1e-4, rtol=1e-4)
    # ResNet: BatchNorm backward on 6 samples is ill-conditioned (near-zero channel variances) -> looser bound
    assert float((g_nat[:nv] - g_ref[:nv]).abs().max()) <= tol * max(1.0, float(g_ref[:nv].abs().max()))
    torch.testing.assert_close(w2[nv:], ref.w[nv:], atol=1e-4, rtol=1e-4)          # BN running statistics


def test_plan_fusion_shapes_resnet():
    lay = get_layout("resnet18")
    nat = NativeNet(lay, "cpu", 2, impl="aten", act_dtype=torch.float32)
    kinds = [op.kind for op in nat.plan]
    assert kinds.count("conv") == 20 and kinds.count("bn") == 20 and kinds.count("linear") == 1
    fused_add = [op for op in nat.plan if op.kind == "bn" and op.res is not None]
    assert len(fused_add) == 8 and all(op.relu for op in fused_add)      # one bn+add+relu per BasicBlock
    assert sum(op.acc_dx for op in nat.plan if op.kind == "conv") == 8   # conv1 of every block accumulates into the skip grad
    assert all(op.saved["want_stats"] for op in nat.plan if op.kind == "conv")


def test_eval_mode_uses_running_stats_and_no_dropout():
    lay = get_layout("cnn_cifar")
    w = lay.init_(torch.zeros(lay.n_total), 3)
    nat = NativeNet(lay, "cpu", 4, impl="aten", act_dtype=torch.float32)
    nat.bind(w, w, None)
    x = torch.randn(4, 32, 32, 3)
    a, b = nat.forward(x, False).clone(), nat.forward(x, False).clone()
    ref = GraphNet(lay, w.clone(), None).eval()
    torch.testing.assert_close(a, b)
    torch.testing.assert_close(a, ref(x.permute(0, 3, 1, 2)).detach(), atol=1e-4, rtol=1e-4)


def test_dropout_layers_are_fused_into_their_producers():
    """SURVEY.md K5: every dropout of the reference CNNs follows a max-pool or a Linear+ReLU (src/models.py:25-30,50-57) and is folded
    into that producer -- the plan has no stand-alone dropout op and no mask tensor; evaluation mode applies no dropout; training mode
    drops about p of the fused output and the backward pass zeroes exactly the dropped positions."""
    import torch
    from rlr_b200.models import get_layout
    from rlr_b200.models import native as nat
    for model, n_drop in (("cnn_mnist", 2), ("cnn_cifar", 3)):
        lay = get_layout(model)
        net = nat.NativeNet(lay, "cpu", 16, impl="aten", act_dtype=torch.float32)
        assert sum(op.kind == "dropout" for op in net.plan) == 0
        assert sum("drop" in op.saved for op in net.plan) == n_drop
        w = lay.init_(torch.zeros(lay.n_total), 3)
        g = torch.zeros_like(w)
        net.bind(w, w.clone(), g)
        C, H, W = lay.in_shape
        x = torch.randn(16, H, W, C)
        torch.manual_seed(0)
        a = net.forward(x, False).clone()
        b = net.forward(x, False).clone()
        assert torch.equal(a, b)                                   # evaluation: deterministic, no dropout
        t1 = net.forward(x, True).clone()
        t2 = net.forward(x, True).clone()
        assert not torch.equal(t1, t2)                             # training: fresh masks
        fused = [op for op in net.plan if "drop" in op.saved and op.kind == "linear"][0]
        y = net.T(fused.y, 16)
        frac_zero = float((y == 0).float().mean())
        assert frac_zero > 0.45                                    # >= p dropped (+ ReLU zeros)
        _, dl = __import__("rlr_b200").ops.softmax_xent(t2, torch.randint(0, 10, (16,)))
        net.backward(dl)
        gy = net.G(fused.y, 16)
        assert float(gy[y == 0].abs().max()) == 0.0               # gradient is zero exactly where the output was dropped / clamped
    old = nat.FUSE_DROPOUT
    try:
        nat.FUSE_DROPOUT = False
        net = nat.NativeNet(get_layout("cnn_mnist"), "cpu", 4, impl="aten", act_dtype=torch.float32)
        assert sum(op.kind == "dropout" for op in net.plan) == 2
    finally:
        nat.FUSE_DROPOUT = old


def test_shortcut_branches_and_relu_pool_fusion_are_planned_where_they_are_legal():
    """Static plan analysis behind two graph-level optimisations of models/native.py:
    * projection shortcuts (1x1 conv + BatchNorm on the block input) become a parallel branch: forked before the block's conv1 (which
      reads the same input), joined at the fused bn2 + add that consumes the shortcut output -- ResNet-18 / -34 have three, every other
      model none;
    * the ReLU of a conv whose ONLY consumer is a max-pool is back-propagated by the pooling backward (reference CNNs), never for
      BatchNorm models (their ReLU is fused into the BatchNorm op)."""
    impl = dict(conv_fwd="aten", conv_dgrad="aten", conv_wgrad="aten", bn="aten", pool="aten", linear="aten", dropout="aten")
    for name, n_branch, n_relu_pool in (("resnet18", 3, 0), ("resnet34", 3, 0), ("vgg11", 0, 0), ("cnn_mnist", 0, 1), ("cnn_cifar", 0, 3)):
        net = NativeNet(get_layout(name), "cpu", 2, impl=impl, act_dtype=torch.float32)
        plan = net.plan
        side = [op for op in plan if op.saved.get("side_branch")]
        forks = [op for op in plan if op.saved.get("fork_before")]
        joins = [op for op in plan if op.saved.get("join_before")]
        assert len(forks) == len(joins) == n_branch and len(side) == 2 * n_branch, name
        for f, j in zip(forks, joins):
            i_f, i_j = plan.index(f), plan.index(j)
            mine = [op for op in side if i_f < plan.index(op) < i_j]
            assert [op.kind for op in mine] == ["conv", "bn"] and ".downsample." in mine[0].name, name
            assert mine[0].x == f.x and mine[1].x == mine[0].y and j.res == mine[1].y            # same input as conv1; feeds the add
            assert all(op.x != mine[0].y and op.x != mine[1].y for op in plan[i_f:i_j] if op not in mine)   # nobody on the main path reads it
        pools = [op for op in plan if op.kind == "maxpool" and op.saved.get("relu_bwd_here")]
        convs = [op for op in plan if op.kind == "conv" and op.saved.get("relu_bwd_fused")]
        assert len(pools) == len(convs) == n_relu_pool, name
        for pool in pools:
            prod = next(q for q in plan if q.y == pool.x)
            assert prod in convs and prod.relu and sum(1 for q in plan if q.x == pool.x or q.res == pool.x) == 1
