"""GPU numerics of the GroupNorm kernels (groupnorm.cu) against fp32 ``F.group_norm`` autograd, their run-to-run bit-reproducibility,
the four GroupNorm models through the native executor against fp32 autograd, and federated training of ``resnet18_gn``."""
import pytest
import torch
import torch.nn.functional as F

import rlr_b200  # noqa: F401
from rlr_b200 import ops
from rlr_b200.models import get_layout
from rlr_b200.models.graph import GraphNet
from rlr_b200.models.native import NativeNet

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16


def _rel(a, b):
    """max-norm relative error."""
    return float((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-6))


def _rms_rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-12))


def _problem(B, H, W, C, groups, res, seed):
    g = torch.Generator(DEV).manual_seed(seed)
    x = (torch.randn(B, H, W, C, device=DEV, generator=g) * 1.5 + 0.4).to(BF)
    r = torch.randn(B, H, W, C, device=DEV, generator=g).to(BF) if res else None
    gamma = torch.rand(C, device=DEV, generator=g) + 0.5
    beta = torch.randn(C, device=DEV, generator=g) * 0.2
    dy = torch.randn(B, H, W, C, device=DEV, generator=g).to(BF)
    return x, r, gamma, beta, dy


def _run(impl, x, r, gamma, beta, dy, groups, relu):
    B, C = x.shape[0], x.shape[-1]
    y, mr = torch.empty_like(x), torch.zeros(B, 2, groups, device=DEV)
    ops.gn_fwd(x, y, r, gamma, beta, mr, groups, 1e-5, relu, impl)
    dx, dres = torch.empty_like(x), (torch.empty_like(x) if r is not None else None)
    dg, db = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    ops.gn_bwd(dy, y, x, gamma, mr, dx, dres, dg, db, groups, relu, impl)
    return dict(y=y, mr=mr, dx=dx, dres=dres, dg=dg, db=db)


CASES = [  # B, H, W, C, groups, relu, res
    (256, 32, 32, 64, 32, True, False), (256, 16, 16, 128, 32, True, True), (256, 8, 8, 256, 32, False, False),
    (256, 4, 4, 512, 32, True, True), (37, 2, 2, 512, 32, True, False), (37, 32, 32, 64, 1, True, True),
    (37, 16, 16, 128, 8, False, True), (37, 8, 8, 256, 256, True, False), (1, 32, 32, 64, 64, False, False),
    (1, 4, 4, 512, 8, True, True), (37, 1, 1, 512, 32, False, False),
    (8, 64, 64, 64, 32, True, True), (8, 64, 64, 64, 1, True, False),                  # tiles that do not fit in shared memory
    (5, 7, 9, 24, 3, True, True), (3, 5, 5, 40, 20, False, False),                    # odd sizes, groups across 8-channel vectors
]


@pytest.mark.parametrize("B,H,W,C,groups,relu,res", CASES)
def test_gn_kernels_vs_fp32_autograd(B, H, W, C, groups, relu, res):
    """Forward / backward against fp32 ``F.group_norm`` autograd fed the same bf16-rounded inputs; the aten back-end in bf16 is the
    yardstick (x1.5 + bf16 output rounding), as for the BatchNorm kernels."""
    x, r, gamma, beta, dy = _problem(B, H, W, C, groups, res, B + C + groups)
    xf = x.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    rf = r.float().permute(0, 3, 1, 2).clone().requires_grad_(True) if res else None
    gf, bf_ = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    z = F.group_norm(xf, groups, gf, bf_, 1e-5)
    if res:
        z = z + rf
    yf = F.relu(z) if relu else z
    yf.backward(dy.float().permute(0, 3, 1, 2))
    nhwc = lambda t: t.permute(0, 2, 3, 1)
    xg = x.float().reshape(B, -1, groups, C // groups)
    ref = dict(y=nhwc(yf.detach()), dx=nhwc(xf.grad), dres=nhwc(rf.grad) if res else None, dg=gf.grad, db=bf_.grad,
               mr=torch.stack([xg.mean((1, 3)), torch.rsqrt(xg.var((1, 3), unbiased=False) + 1e-5)], 1))
    ops.reset_fallbacks()
    sm, at = _run("sm100", x, r, gamma, beta, dy, groups, relu), _run("aten", x, r, gamma, beta, dy, groups, relu)
    assert ops.fallback_calls() == {}
    for k in ("y", "mr", "dx", "dres", "dg", "db"):
        if ref[k] is None:
            continue
        want = ref[k].reshape(sm[k].shape)
        e_sm, e_at = _rms_rel(sm[k], want), _rms_rel(at[k], want)
        print(f"gn B={B} {H}x{W}x{C} G={groups} {k}: rms-rel sm100 {e_sm:.2e} aten-bf16 {e_at:.2e}  max-rel sm100 {_rel(sm[k], want):.2e}")
        assert e_sm < 1.5 * e_at + 4e-3, (k, e_sm, e_at)
        assert _rel(sm[k], want) < 2e-2, (k, _rel(sm[k], want))


@pytest.mark.parametrize("B,H,W,C,groups", [(256, 32, 32, 64, 32), (37, 4, 4, 512, 32), (8, 64, 64, 64, 1)])
def test_gn_kernels_are_bitwise_reproducible(B, H, W, C, groups):
    x, r, gamma, beta, dy = _problem(B, H, W, C, groups, True, 7)
    a = _run("sm100", x, r, gamma, beta, dy, groups, True)
    b = _run("sm100", x, r, gamma, beta, dy, groups, True)
    for k in ("y", "mr", "dx", "dres", "dg", "db"):
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("model,B", [("resnet18_gn", 64), ("vgg11_gn", 48), ("resnet34_gn", 32), ("vgg16_gn", 32)])
def test_gn_native_net_sm100_vs_fp32_autograd(model, B):
    """Whole forward / backward of every GroupNorm model on our kernels against fp32 autograd, per parameter tensor, with the library
    bf16 path (aten back-end) as the yardstick: at most 1.5x as far from fp32 (+ 1 %).  No library fall-through in the sm100 run."""
    torch.manual_seed(0)
    lay = get_layout(model)
    w = lay.init_(torch.zeros(lay.n_total, device=DEV), 1)
    w[: lay.n_vote] = w[: lay.n_vote].to(BF).float()
    C, H, W = lay.in_shape
    x = torch.randn(B, H, W, C, device=DEV).to(BF)
    y = torch.randint(0, 10, (B,), device=DEV)
    wr, g32 = w.clone(), torch.zeros_like(w)
    net32 = GraphNet(lay, wr, g32, torch.float32).train()
    l32 = net32(x.float().permute(0, 3, 1, 2).contiguous())
    F.cross_entropy(l32, y).backward()
    l32 = l32.detach()
    res = {}
    for impl in ("aten", "sm100"):
        ops.reset_fallbacks()
        net = NativeNet(lay, DEV, B, impl=impl)
        wi, g = w.clone(), torch.zeros_like(w)
        net.bind(wi, wi.to(BF), g)
        logits = net.forward(x, True).clone()
        _, dl = ops.softmax_xent(logits, y)
        net.backward(dl)
        res[impl] = (logits, g.clone())
        if impl == "sm100":
            assert ops.fallback_calls() == {}, f"library fall-throughs in the sm100 plan of {model}: {ops.fallback_calls()}"
            torch.testing.assert_close(net.forward(x, False), logits, rtol=0, atol=0)    # evaluation == training forward
    (la, ga), (ls, gs) = res["aten"], res["sm100"]
    print(model, "logits rms-rel vs fp32: sm100", _rms_rel(ls, l32), "aten-bf16", _rms_rel(la, l32),
          "| gradient: sm100", _rms_rel(gs, g32), "aten-bf16", _rms_rel(ga, g32))
    assert _rms_rel(ls, l32) < 1.5 * _rms_rel(la, l32) + 1e-2
    bad = []
    for p in lay.params:
        want = lay.view(g32, p)
        e_sm, e_at = _rms_rel(lay.view(gs, p), want), _rms_rel(lay.view(ga, p), want)
        if not e_sm <= 1.5 * e_at + 1e-2:
            bad.append((p.name, round(e_sm, 4), round(e_at, 4)))
    assert not bad, f"{model}: parameters whose sm100 gradient is > 1.5x further from fp32 than the library bf16 path: {bad[:8]}"


def test_gn_trainers_learn_and_native_rounds_are_reproducible():
    """Native and torch trainers on resnet18_gn learn synthetic data (CUDA-graph capture, ragged last batch, evaluation); two
    identical native runs give bit-identical global parameters."""
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    accs, finals = {}, []
    for trainer in ("native", "torch", "native"):
        args = make_args(data="cifar10", model="resnet18_gn", num_agents=2, local_ep=2, bs=64, synthetic=1000, synthetic_val=200,
                         log_dir="", device=DEV, trainer=trainer, seed=2)
        eng = FLEngine(args, verbose=False)
        assert eng.trainer.name == trainer and eng.layout.n_total == eng.layout.n_vote
        ops.reset_fallbacks()
        for r in range(1, 11):
            eng.run_round(r)
        if trainer == "native":
            assert ops.fallback_calls() == {}
            finals.append(eng.global_params().clone())
        accs[trainer] = eng.evaluate(10)["val_acc"]
        eng.close()
    print("resnet18_gn", accs)
    assert accs["native"] > 0.85 and accs["torch"] > 0.85
    assert torch.equal(finals[0], finals[1])
