"""Server-clip update norms on the H100: ``ops.update_norms`` runs the trust pass (``trust_stats_kernel``, ops/csrc/trust.cu) with the
root parameters at ``w_global``.  Run-to-run bitwise equality, the fp64 statement for participant counts on both sides of the kernel's
1024-entry tables (more participants are launched in chunks and stay on the device), and a ``--server_clip --diagnostics`` server
step that is bitwise reproducible, ``Norms/*`` scalars included."""
import pytest
import torch

from rlr_b200 import ops
from rlr_b200.aggregation import Aggregation
from rlr_b200.options import make_args

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-7          # relative error of the squared norms: the tolerance tests/test_gpu_fltrust.py holds q_k to


def _participants(K, n, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randn(n, generator=gen, device=DEV)
    return g, [g + 0.01 * (1 + k % 5) * torch.randn(n, generator=gen, device=DEV) for k in range(K)]


def test_two_launches_are_bitwise_equal():
    g, ws = _participants(40, 1 << 20, 3)
    a = ops.update_norms(g, ws, (1 << 20) - 256)
    b = ops.update_norms(g, ws, (1 << 20) - 256)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


@pytest.mark.parametrize("K", [1, 10, 40, 1500])
def test_update_norms_match_fp64_statement(K):
    ops.reset_fallbacks()
    n = 1 << 20 if K <= 40 else 1 << 16
    nv = n - 1024                                                    # BatchNorm-style tail coordinates do not count
    g, ws = _participants(K, n, K + 7)
    for w in ws:
        w[nv:] += 100.0
    q = ops.update_norms(g, ws, nv) ** 2
    ref = torch.stack([(w[:nv].double() - g[:nv].double()).norm() for w in ws]) ** 2
    err = float(((q - ref).abs() / ref).max())
    print(f"K={K}: max rel err of the squared norms {err:.2e}")
    assert q.shape == (K,) and err <= TOL
    assert ops.fallback_calls() == {}


def test_server_clip_step_is_bitwise_reproducible():
    K, n, nv = 10, 1 << 20, (1 << 20) - 4096
    g, ws = _participants(K, n, 11)
    a = make_args(num_agents=K, num_corrupt=3, robustLR_threshold=2, server_lr=0.5, clip=25.0, server_clip=True, diagnostics=True,
                  device=DEV)
    runs = []
    for _ in range(2):
        wg = g.clone()
        agg = Aggregation({i: 100 + 13 * i for i in range(K)}, n, None, a)
        agg.aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=nv)
        torch.cuda.synchronize()
        runs.append((wg, agg.last_norms))
    norms = ops.update_norms(g, ws, nv)
    assert float(norms.min()) < a.clip < float(norms.max())         # some updates are clipped, some are not
    assert torch.equal(runs[0][0], runs[1][0]) and not torch.equal(runs[0][0], g)
    assert set(runs[0][1]) == {"Norms/Avg_Honest_L2", "Norms/Avg_Corrupt_L2"} and runs[0][1] == runs[1][1]
