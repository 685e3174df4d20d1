"""SparseFed (``--server_topk``) on CPU: option validation and the banner, ``ops.sparsefed_statement`` on hand-built vectors (ties at tau,
keys that differ only in their low bits, signed zeros, NaN, k = 1 and k = n_vote, the BatchNorm tail), error-feedback conservation with
dyadic values, p = 1, the in-process ``Aggregation.aggregate_updates`` against a loop over the statement, engine runs with the torch
trainer (log fields, checkpoint / resume bit for bit, a checkpoint without the state refused), and 2 gloo ranks against one process on
the gather and reduce transports."""
import math
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from rlr_b200 import ops
from rlr_b200.options import make_args, print_exp_details

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- options ------------------------------------------------------------------------------------------------------------
def test_default_is_off_and_the_banner(capsys):
    a = make_args()
    assert a.server_topk == 0.0
    print_exp_details(a)
    assert "SparseFed" not in capsys.readouterr().out
    b = make_args(server_topk=0.01)
    print_exp_details(b, 1000)
    assert "Server top-k (SparseFed): 0.01 / 10" in capsys.readouterr().out
    print_exp_details(b)
    assert "Server top-k (SparseFed): 0.01 / -" in capsys.readouterr().out
    assert make_args(server_topk=1).server_topk == 1.0


@pytest.mark.parametrize("p", [-0.1, 1.5, float("nan"), float("inf")])
def test_rejects_out_of_range_values(p):
    with pytest.raises(ValueError, match="--server_topk"):
        make_args(server_topk=p)


def test_k_sizing_and_the_engine_refusing_k_zero():
    assert ops.sparsefed_k(0.01, 1000) == 10 and ops.sparsefed_k(1.0, 7) == 7
    with pytest.raises(ValueError, match="n_params 1000.*smallest usable p is 1/1000"):
        ops.sparsefed_k(0.0005, 1000)
    with pytest.raises(ValueError, match="n_params"):
        _engine(server_topk=1e-9)


# ---- the statement ------------------------------------------------------------------------------------------------------------
def _brute(w, wn, e, n_vote, k):
    """Per-coordinate Python form of the statement (sorted keys, explicit loops)."""
    w, wn, e = (np.asarray(x, dtype=np.float32) for x in (w, wn, e))
    with np.errstate(invalid="ignore", over="ignore"):
        e1 = np.array([np.float32(e[c] + np.float32(wn[c] - w[c])) for c in range(n_vote)], dtype=np.float32)
    keys = [int(x) & 0x7FFFFFFF for x in e1.view(np.uint32)]
    tau = sorted(keys, reverse=True)[k - 1]
    out, e2 = wn.copy(), e1.copy()
    applied = 0
    for c in range(n_vote):
        if keys[c] >= max(tau, 1):
            with np.errstate(invalid="ignore", over="ignore"):
                out[c] = np.float32(w[c] + e1[c])
            e2[c] = 0.0
            applied += 1
        else:
            out[c] = w[c]
    return out, e2, applied, tau


def _check(w, wn, e, n_vote, k):
    out, e2, applied, tau, norm = ops.sparsefed_statement(torch.from_numpy(w), torch.from_numpy(wn), torch.from_numpy(e), n_vote, k)
    bo, be, ba, bt = _brute(w, wn, e, n_vote, k)
    assert out.tobytes() == bo.tobytes() and e2.tobytes() == be.tobytes()
    assert applied == ba and (applied >= k or bt == 0) and np.float32(tau).view(np.uint32) == bt
    ref = math.sqrt(sum(float(x) ** 2 for x in be))
    assert (math.isnan(norm) and math.isnan(ref)) or math.isclose(norm, ref, rel_tol=1e-12)
    return out, e2, applied, tau


@pytest.mark.parametrize("k", [1, 7, 100, 256])
def test_statement_matches_a_sort_on_random_data(k):
    rs = np.random.RandomState(k)
    n, nv = 264, 256
    w = rs.randn(n).astype(np.float32)
    wn = (w + 0.01 * rs.randn(n)).astype(np.float32)
    e = (0.01 * rs.randn(nv)).astype(np.float32)
    out, _, applied, _ = _check(w, wn, e, nv, k)
    assert applied == k                                               # continuous data: no ties
    assert out[nv:].tobytes() == wn[nv:].tobytes()                    # the BatchNorm tail keeps the plain step


def test_ties_at_tau_are_all_taken():
    nv = 16
    w = np.zeros(nv, dtype=np.float32)
    wn = np.array([0.5, -0.5, 0.5, 0.25, -0.5, 0.125] + [0.0625] * 10, dtype=np.float32)
    e = np.zeros(nv, dtype=np.float32)
    _, e2, applied, tau = _check(w, wn, e, nv, 2)
    assert applied == 4 and tau == 0.5 and np.count_nonzero(e2) == nv - 4


def test_keys_that_differ_in_their_low_bits():
    nv = 8
    base = np.float32(1.0).view(np.uint32)
    d = (base + np.array([0, 1, 2, 3, 0x100, 0x1FF, 0x1FE, 5], dtype=np.uint32)).view(np.float32)
    sign = np.array([1, -1, 1, -1, 1, -1, 1, -1], dtype=np.float32)
    w = np.zeros(nv, dtype=np.float32)
    _, e2, applied, tau = _check(w, (d * sign).astype(np.float32), np.zeros(nv, dtype=np.float32), nv, 3)
    assert applied == 3 and np.float32(tau).view(np.uint32) == base + 0x100
    assert list(np.flatnonzero(e2 == 0)) == [4, 5, 6]


def test_signed_zeros_are_never_applied_and_nan_sorts_first():
    nv = 8
    w = np.zeros(nv, dtype=np.float32)
    wn = np.array([0.0, -0.0, 0.0, 1.0, np.nan, -0.0, 0.0, 0.0], dtype=np.float32)
    e = np.array([0.0, 0.0, -0.0, 0.0, 0.0, -0.0, 0.0, 0.0], dtype=np.float32)
    out, e2, applied, tau = _check(w, wn, e, nv, nv)                  # k = n_vote: tau is a zero key
    assert applied == 2 and tau == 0.0
    assert out[3] == 1.0 and np.isnan(out[4]) and e2[3] == 0 and e2[4] == 0
    _, _, applied, tau = _check(w, wn, e, nv, 1)                      # k = 1: only the NaN
    assert applied == 1 and math.isnan(tau)


def test_k_out_of_range_is_refused():
    z = torch.zeros(8)
    for k in (0, 9):
        with pytest.raises(ValueError, match="k ="):
            ops.sparsefed_statement(z, z, z, 8, k)


def test_error_feedback_conserves_the_steps_with_dyadic_values():
    """Dyadic steps are exact in fp32, so sum of the applied steps + e_R = sum of the plain steps u_t, coordinate by coordinate."""
    rs = np.random.RandomState(3)
    nv, R, k = 64, 6, 5
    w = (rs.randint(-64, 64, nv) / 8.0).astype(np.float32)
    e = np.zeros(nv, dtype=np.float32)
    applied_sum, u_sum = np.zeros(nv), np.zeros(nv)
    for _ in range(R):
        u = (rs.randint(-16, 16, nv) / 64.0).astype(np.float32)
        wn = (w + u).astype(np.float32)
        out, e, _, _ = _check(w, wn, e, nv, k)
        applied_sum += out.astype(np.float64) - w
        u_sum += u
        w = out
    assert np.array_equal(applied_sum + e, u_sum)


def test_p_one_keeps_no_error():
    rs = np.random.RandomState(4)
    n, nv = 40, 32
    w = rs.randn(n).astype(np.float32)
    wn = (w + rs.randn(n)).astype(np.float32)
    out, e2, applied, _, norm = ops.sparsefed_statement(torch.from_numpy(w), torch.from_numpy(wn), torch.zeros(nv), nv, nv)
    assert applied == nv and not e2.any() and norm == 0.0
    assert out[:nv].tobytes() == (w[:nv] + (wn[:nv] - w[:nv])).astype(np.float32).tobytes()


def test_cpu_step_writes_in_place():
    rs = np.random.RandomState(5)
    n, nv, k = 48, 40, 6
    w, wn = torch.from_numpy(rs.randn(n).astype(np.float32)), torch.from_numpy(rs.randn(n).astype(np.float32))
    e = torch.from_numpy((0.1 * rs.randn(nv)).astype(np.float32))
    ref = ops.sparsefed_statement(w, wn, e, nv, k)
    stats, wb = torch.zeros(3, dtype=torch.float64), torch.zeros(n, dtype=torch.bfloat16)
    ops.sparsefed_step(w, wn, e, nv, k, stats, wb)
    assert np.array_equal(w.numpy(), ref[0]) and np.array_equal(e.numpy(), ref[1]) and torch.equal(wb, w.to(torch.bfloat16))
    assert stats.tolist() == [ref[2], ref[3], ref[4]]


# ---- in-process aggregation ---------------------------------------------------------------------------------------------------
def test_in_process_aggregation_against_a_loop_over_the_statement():
    from rlr_b200.aggregation import Aggregation
    p, n, nv, n_params = 0.05, 200, 192, 190
    args = make_args(server_topk=p, robustLR_threshold=2, server_opt="adam", server_lr=0.5, aggr="avg")
    sizes = {i: 10 + i for i in range(4)}
    agg = Aggregation(sizes, n_params, None, args)
    g = torch.Generator().manual_seed(9)
    w = torch.randn(n, generator=g)
    ref_w, ref_e = w.clone(), torch.zeros(nv)
    ref_opt = ops.ServerOptState(n=n, **{"kind": "adam", "beta1": 0.9, "beta2": 0.99, "tau": 1e-3})
    k = math.floor(p * n_params)
    for rnd in (1, 2, 3, 4):
        ws = {i: w + 0.1 * torch.randn(n, generator=g) for i in sizes}
        plain = ops.fused_aggregate(ref_w, [x - w + ref_w for x in ws.values()], [float(s) for s in sizes.values()], "avg", 2, 0.5,
                                    n_vote=nv, out=torch.empty(n), opt=ref_opt)
        out, e2, applied, tau, norm = ops.sparsefed_statement(ref_w, plain, ref_e, nv, k)
        ref_w, ref_e = torch.from_numpy(out), torch.from_numpy(e2)
        agg.aggregate_updates(w, {i: x - w + w for i, x in ws.items()}, rnd, n_vote=nv)
        assert torch.equal(w, ref_w) and torch.equal(agg.sparse_e, ref_e)
        assert agg.last_sparse == {"sparse_applied": applied, "sparse_threshold": tau, "sparse_error_norm": norm}
        assert applied >= k and ref_e.any()


# ---- engine runs ----------------------------------------------------------------------------------------------------------
def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="fmnist", synthetic=800, synthetic_val=200, num_agents=5, local_ep=1, bs=64, device="cpu", num_corrupt=1,
                poison_frac=0.5, robustLR_threshold=2, log_dir="", seed=5, trainer="torch")
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def test_engine_runs_log_and_resume_bit_for_bit(tmp_path):
    kw = dict(server_topk=0.02, server_opt="momentum", server_lr=1.0, rounds=3, server_clip=True, clip=1.0)
    full = _engine(**kw)
    hist = full.fit()
    k = math.floor(0.02 * full.layout.n_params)
    assert full.topk_k == k and full.fused.sparse_e.shape == (full.layout.n_vote,)
    for h in hist:
        assert h["sparse_applied"] >= k and h["sparse_threshold"] > 0 and h["sparse_error_norm"] > 0
    ck = str(tmp_path / "ck.pt")
    first = _engine(checkpoint=ck, **{**kw, "rounds": 2})
    first.fit()
    assert torch.equal(torch.load(ck, weights_only=False)["extra"]["sparsefed_error"], first.fused.sparse_e)
    second = _engine(resume=ck, **kw)
    assert second.start_round == 3
    hist2 = second.fit()
    assert torch.equal(second.w_global, full.w_global) and torch.equal(second.fused.sparse_e, full.fused.sparse_e)
    assert {k_: v for k_, v in hist2[-1].items() if k_.startswith("sparse")} == {k_: v for k_, v in hist[-1].items() if k_.startswith("sparse")}
    for e in (full, first, second):
        e.close()


def test_off_allocates_nothing_and_a_checkpoint_without_the_state_is_refused(tmp_path):
    ck = str(tmp_path / "ck.pt")
    plain = _engine(rounds=1, checkpoint=ck)
    plain.fit()
    assert plain.fused.scratch is None and plain.fused.sparse_e is None and plain.last_sparse is None
    assert "sparsefed_error" not in torch.load(ck, weights_only=False)["extra"]
    with pytest.raises(ValueError, match="checkpoint has no SparseFed state"):
        _engine(rounds=2, resume=ck, server_topk=0.02)
    plain.close()


# ---- 2 gloo ranks against one process ---------------------------------------------------------------------------------------
CASES = [  # (transport, n, n_vote, n_part, mode, theta, kind)
    ("gather", 4096, 4000, 5, "avg", 2, "adam"),
    ("reduce", 4096, 4096, 4, "sign", 2, "momentum"),
]


def _run(fa, rank, seed, n, n_part, mode, theta, k):
    g = torch.Generator().manual_seed(seed)
    fa.w_global.copy_(torch.randn(n, generator=g))
    stats = []
    for rnd in (1, 2, 3):
        for j in range(n_part):
            a = fa.w_global + 0.1 * torch.randn(n, generator=g)
            r, s = fa.slot_owner(j)
            if r == rank:
                fa.slots[s].copy_(a)
        fa.aggregate([float(10 + 3 * j) for j in range(n_part)], mode, theta, 0.25, 0.0, seed=5, rnd=rnd)
        stats.append(fa.sparse_stats.tolist())
    return fa.w_global.clone(), fa.sparse_e.clone(), stats


def _gloo_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.parallel import FusedAggregator, init_distributed
    ctx = init_distributed("cpu")
    out = {}
    for ci, (transport, n, nv, n_part, mode, theta, kind) in enumerate(CASES):
        fa = FusedAggregator(ctx, n, nv, (n_part + world - 1) // world, "gloo", transport=transport, server_opt=dict(kind=kind),
                             topk_k=40)
        out[ci] = _run(fa, rank, 100 + ci, n, n_part, mode, theta, 40)
        fa.close()
    torch.save(out, os.path.join(outdir, f"r{rank}.pt"))
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_ranks_equal_one_process(tmp_path):
    from rlr_b200.parallel import FusedAggregator
    from rlr_b200.parallel.comm import DistContext
    world = 2
    mp.spawn(_gloo_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"r{r}.pt") for r in range(world)]
    for ci, (transport, n, nv, n_part, mode, theta, kind) in enumerate(CASES):
        solo = FusedAggregator(DistContext(), n, nv, n_part, "local", server_opt=dict(kind=kind), topk_k=40)
        ref = _run(solo, 0, 100 + ci, n, n_part, mode, theta, 40)
        assert ref[1].any() and all(s[0] >= 40 for s in ref[2])
        for o in outs:
            assert torch.equal(o[ci][0], ref[0]) and torch.equal(o[ci][1], ref[1]), transport
            assert o[ci][2] == ref[2]
