"""Server step semantics (src/aggregation.py:19-75; SURVEY.md 3.4) incl. differential tests against the reference class."""
import pytest
import torch
from hypothesis import given, settings, strategies as st

from rlr_b200 import ops
from rlr_b200.aggregation import Aggregation
from rlr_b200.options import make_args


def _mk(K, n, seed=0, zeros=0.2):
    g = torch.Generator().manual_seed(seed)
    w0 = torch.randn(n, generator=g)
    ws = [w0 + 0.1 * torch.randn(n, generator=g) * (torch.rand(n, generator=g) > zeros) for _ in range(K)]
    return w0, ws


def test_lower_median_rule():
    w0 = torch.zeros(4)
    ws = [torch.full((4,), v) for v in (1.0, 2.0, 3.0, 4.0)]
    out, _ = ops.aggregate_oracle(w0, ws, [1, 1, 1, 1], "comed")
    assert torch.equal(out, torch.full((4,), 2.0)), "torch.median -> LOWER median for even K"


def test_rlr_flips_sign_not_zero_and_zero_abstains():
    w0 = torch.zeros(4)
    # coord0: 3 agree (+) -> keep; coord1: 2 vs 1 -> |s|=1 < 2 -> flip; coord2: two zeros + one + -> |s|=1 -> flip; coord3: all zero
    ws = [torch.tensor([1.0, 1.0, 0.0, 0.0]), torch.tensor([1.0, 1.0, 0.0, 0.0]), torch.tensor([1.0, -1.0, 3.0, 0.0])]
    out, nflip = ops.aggregate_oracle(w0, ws, [1, 1, 1], "avg", theta=2)
    torch.testing.assert_close(out, torch.tensor([1.0, -1.0 / 3, -1.0, 0.0]))
    assert nflip == 3  # coord3 has s=0 < theta: lr flipped too (update is 0 anyway), as in the reference


@pytest.mark.parametrize("aggr", ["avg", "comed", "sign"])
@pytest.mark.parametrize("theta", [0, 1, 3, 5])
def test_matches_reference_class(reference_outputs, aggr, theta):
    K, n = 5, 2000
    w0, ws = _mk(K, n, seed=theta)
    sizes = {i: 100 + 7 * i for i in range(K)}
    server_lr = 0.7 if aggr == "sign" else 1.0
    ref = reference_outputs[f"aggregate/{aggr}/{theta}"]       # the reference class's aggregate_updates on a Linear model holding w0
    ours, _ = ops.aggregate_oracle(w0, ws, [sizes[i] for i in range(K)], aggr, theta, server_lr)
    torch.testing.assert_close(ours, ref, atol=1e-7, rtol=1e-6)
    # and the public class (CPU path of the fused op)
    a = make_args(aggr=aggr, robustLR_threshold=theta, server_lr=0.7)
    wg = w0.clone()
    Aggregation(sizes, n, None, a).aggregate_updates(wg, {i: ws[i] for i in range(K)}, 1, n_vote=n)
    torch.testing.assert_close(wg, ref, atol=1e-7, rtol=1e-6)


def test_reference_named_helpers_match_reference(reference_outputs):
    K, n = 4, 500
    w0, ws = _mk(K, n, seed=3)
    ups = {i: (ws[i].double() - w0) for i in range(K)}
    sizes = {i: 10 * (i + 1) for i in range(K)}
    ref = lambda name: reference_outputs[f"helpers/{name}"]  # noqa: E731  (reference Aggregation, robustLR_threshold=3, clip=0.5)
    ours = Aggregation(sizes, n, None, make_args(robustLR_threshold=3, clip=0.5))
    torch.testing.assert_close(ours.compute_robustLR(ups), ref("robustLR"))
    torch.testing.assert_close(ours.agg_avg(ups), ref("avg"))
    torch.testing.assert_close(ours.agg_comed(ups), ref("comed"))
    torch.testing.assert_close(ours.agg_sign(ups), ref("sign"))
    a = {k: v.clone() for k, v in ups.items()}
    ours.clip_updates(a)
    for k in a:
        torch.testing.assert_close(a[k], ref("clipped")[k])


def test_tail_coordinates_get_plain_mean_and_no_vote():
    w0 = torch.zeros(8)
    ws = [torch.cat([torch.ones(4), torch.full((4,), 2.0)]), torch.cat([-torch.ones(4), torch.full((4,), 4.0)])]
    out, nflip = ops.aggregate_oracle(w0, ws, [1, 3], "comed", theta=2, n_vote=4)
    torch.testing.assert_close(out[4:], torch.full((4,), 3.5))      # weighted mean, not median, no flip
    torch.testing.assert_close(out[:4], torch.full((4,), 1.0))      # lower median -1, flipped (|s|=0<2) -> +1
    assert nflip == 4


def test_noise_is_added_before_lr_multiply():
    w0 = torch.zeros(2)
    ws = [torch.tensor([1.0, 1.0]), torch.tensor([1.0, -1.0])]
    noise = torch.tensor([0.5, 0.5])
    out, _ = ops.aggregate_oracle(w0, ws, [1, 1], "avg", theta=2, noise=noise)
    torch.testing.assert_close(out, torch.tensor([1.5, -0.5]))       # flipped coordinate gets NEGATED noise


def test_server_clip_and_diagnostics_run():
    from rlr_b200.data import make_synthetic, make_poisoned_val
    from rlr_b200.models import get_layout
    lay = get_layout("cnn_mnist")
    a = make_args(clip=0.5, server_clip=True, diagnostics=True, robustLR_threshold=2, num_corrupt=1, top_frac=50)
    _, va = make_synthetic("fmnist", 200, 100)
    pv = make_poisoned_val(va, a)
    w0 = lay.init_(torch.zeros(lay.n_total), 0)
    ws = {i: w0 + 0.01 * (i + 1) * torch.randn(lay.n_total) for i in range(3)}
    agg = Aggregation({0: 10, 1: 10, 2: 10}, lay.n_params, pv, a, None, lay)
    agg.aggregate_updates(w0, ws, 1)
    assert "Norms/Avg_Honest_L2" in agg.last_norms and "Norms/Avg_Corrupt_L2" in agg.last_norms
    assert set(agg.last_sign_stats) >= {"Sign/Hon_Maxim_L2", "Sign/Adv_Maxim_L2", "Sign/Adv_Minim_L2", "Sign/Hon_Minim_L2",
                                        "Sign/Adv_Net_L2", "Sign/Hon_Net_L2", "Sign/Model_Net_L2_Cumulative"}


@settings(max_examples=40, deadline=None)
@given(K=st.integers(1, 9), theta=st.integers(0, 9), seed=st.integers(0, 1000), aggr=st.sampled_from(["avg", "comed", "sign"]))
def test_property_oracle_invariants(K, theta, seed, aggr):
    n = 64
    w0, ws = _mk(K, n, seed, zeros=0.4)
    out, nflip = ops.aggregate_oracle(w0, ws, [1.0] * K, aggr, theta, 1.0)
    ups = torch.stack([w.double() - w0.double() for w in ws])
    s = torch.sign(ups).sum(0).abs()
    step = out.double() - w0.double()
    if aggr == "avg":
        base = ups.mean(0)
    elif aggr == "comed":
        base = ups.sort(0).values[(K - 1) // 2]
    else:
        base = torch.sign(torch.sign(ups).sum(0))
    lr = torch.where(s >= theta, 1.0, -1.0) if theta > 0 else torch.ones(n)
    torch.testing.assert_close(step, (lr * base), atol=1e-6, rtol=1e-5)
    assert nflip == (int((s < theta).sum()) if theta > 0 else 0)
    if theta > K:  # unreachable threshold: every coordinate is flipped
        assert nflip == n


def test_more_participants_than_the_kernel_limit_uses_exact_fallback():
    K, n = ops.MAX_FUSED_AGENTS + 22, 64
    w0, ws = _mk(K, n, seed=9)
    wt = [1.0 + (i % 3) for i in range(K)]
    for mode in ("avg", "comed", "sign"):
        ref, nflip = ops.aggregate_oracle(w0, ws, wt, mode, 40, 1.0)
        out = torch.empty_like(w0)
        flipped = torch.zeros(1, dtype=torch.int64)
        ops.fused_aggregate(w0, ws, wt, mode, 40, 1.0, out=out, flipped=flipped)
        torch.testing.assert_close(out, ref)
        assert int(flipped) == nflip


@settings(max_examples=40, deadline=None)
@given(K=st.integers(1, 9), splits=st.integers(1, 4), theta=st.integers(0, 9), seed=st.integers(0, 1000), aggr=st.sampled_from(["avg", "sign"]),
       tail=st.integers(0, 16))
def test_property_partial_sums_reproduce_the_oracle(K, splits, theta, seed, aggr, tail):
    """The all-reduce transport's algebra: splitting the participants over any number of ranks, summing their (vote, weighted sum)
    partials and finishing with aggregate_from_partials equals the oracle on the full list (weights, zeros, RLR, BN-style tail)."""
    n = 64
    w0, ws = _mk(K, n, seed, zeros=0.3)
    wt = [1.0 + (i * 7 % 5) for i in range(K)]
    ref, nflip = ops.aggregate_oracle(w0, ws, wt, aggr, theta, 0.5, None, n - tail)
    vote, wsum = torch.zeros(n), torch.zeros(n, dtype=torch.float64)
    for r in range(splits):
        mine = list(range(r, K, splits))
        v, s = ops.aggregate_partials(w0, [ws[j] for j in mine], [wt[j] for j in mine])
        vote += v
        wsum += s
    out, nf = ops.aggregate_from_partials(w0, vote, wsum, sum(wt), aggr, theta, 0.5, None, n - tail)
    torch.testing.assert_close(out, ref, atol=1e-6, rtol=1e-6)
    assert nf == nflip
    with pytest.raises(ValueError):
        ops.aggregate_from_partials(w0, vote, wsum, sum(wt), "comed", theta, 0.5)
