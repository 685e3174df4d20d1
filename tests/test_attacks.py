"""Model-poisoning attackers (``--attack_boost``, ``--attack_neurotoxin``) on CPU: option validation and the banner, Neurotoxin's mask
statement against a brute-force sort (random data, ties, edge values), the masked optimizer step against an fp64 statement, the boost
statement against per-coordinate Python arithmetic, and engine runs (defaults unchanged, boosted and masked rounds against unattacked
ones, resume, 2 ranks over gloo, Multi-Krum against a boosted update, JSONL fields and TensorBoard tags)."""
import json
import math
import os
import socket
import subprocess
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
def test_defaults_are_off_and_the_banner(capsys):
    a = make_args()
    assert a.attack_boost == 1.0 and a.attack_neurotoxin == 0.0
    print_exp_details(a)
    assert "Attack" not in capsys.readouterr().out
    print_exp_details(make_args(num_corrupt=1, attack_boost=8))
    assert "Attack (boost / neurotoxin): 8.0 / 0.0" in capsys.readouterr().out
    print_exp_details(make_args(num_corrupt=1, attack_neurotoxin=0.01))
    assert "Attack (boost / neurotoxin): 1.0 / 0.01" in capsys.readouterr().out


@pytest.mark.parametrize("kw", [
    dict(attack_boost=0.0), dict(attack_boost=-2.0), dict(attack_boost=float("inf")), dict(attack_boost=float("nan")),
    dict(attack_neurotoxin=-0.1), dict(attack_neurotoxin=1.0), dict(attack_neurotoxin=1.5), dict(attack_neurotoxin=float("nan")),
    dict(attack_neurotoxin=float("inf")),
])
def test_rejects_out_of_range_values(kw):
    with pytest.raises(ValueError):
        make_args(num_corrupt=1, **kw)


@pytest.mark.parametrize("kw", [dict(attack_boost=4.0), dict(attack_neurotoxin=0.01)])
def test_rejects_an_attack_without_corrupt_agents(kw):
    with pytest.raises(ValueError, match="num_corrupt"):
        make_args(num_corrupt=0, **kw)
    make_args(num_corrupt=1, **kw)


# ---- Neurotoxin's mask statement ----------------------------------------------------------------------------------------------
def _brute(w_g, w_prev, n_vote, k):
    d = (w_g[:n_vote].numpy() - w_prev[:n_vote].numpy()).astype(np.float32)
    a = [int(x) & 0x7FFFFFFF for x in d.view(np.uint32)]
    tau = sorted(a, reverse=True)[k - 1] if k > 0 else None
    bits = [tau is not None and x >= max(tau, 1) for x in a]
    words = np.zeros(ops.mask_words(n_vote), dtype=np.uint32)
    for c, b in enumerate(bits):
        if b:
            words[c // 32] |= np.uint32(1 << (c % 32))
    return words, sum(bits)


def _check_statement(w_g, w_prev, n_vote, k):
    words, count = ops.neurotoxin_statement(w_g, w_prev, n_vote, k)
    ref_words, ref_count = _brute(w_g, w_prev, n_vote, k)
    assert words.dtype == np.uint32 and np.array_equal(words, ref_words) and count == ref_count
    assert torch.equal(ops.mask_bits(torch.from_numpy(words.view(np.int32)), n_vote).sum(), torch.tensor(count))
    return words, count


@pytest.mark.parametrize("n", [1000, 1003, 4096])
def test_statement_matches_a_sort_on_random_data(n):
    g = torch.Generator().manual_seed(n)
    w_prev = torch.randn(n, generator=g)
    w_g = w_prev + 1e-3 * torch.randn(n, generator=g)
    for k in (1, int(0.01 * n), int(0.5 * n), n):
        _, count = _check_statement(w_g, w_prev, n, k)
        assert count == k                                           # continuous data: no ties


def test_statement_with_heavy_ties_includes_every_tie():
    n = 2000
    g = torch.Generator().manual_seed(1)
    levels = torch.tensor([0.0, 1e-3, 2e-3])
    w_prev = torch.zeros(n)
    w_g = levels[torch.randint(0, 3, (n,), generator=g)] * torch.where(torch.rand(n, generator=g) < 0.5, 1.0, -1.0)
    n_top = int((w_g.abs() == 2e-3).sum())
    n_nonzero = int((w_g != 0).sum())
    for k in (1, n_top, n_top + 1, n_nonzero, n):
        _, count = _check_statement(w_g, w_prev, n, k)
        assert count == (n_top if k <= n_top else n_nonzero)        # ties at tau all in; zero changes never


def test_statement_on_edge_values():
    n = 96
    w_prev = torch.zeros(n)
    assert _check_statement(w_prev.clone(), w_prev, n, 10)[1] == 0  # no change at all: empty mask
    assert _check_statement(w_prev, w_prev, n, 0)[1] == 0           # k = 0: empty mask
    w_g = torch.zeros(n)
    w_g[0], w_g[1] = 0.0, -0.0                                      # |+-0| = 0: never masked
    w_g[2], w_g[3] = 1e-45, -1e-44                                  # denormals
    w_g[4], w_g[5] = float("inf"), -float("inf")
    w_g[6] = float("nan")
    w_g[7:20] = torch.linspace(-1, 1, 13)
    for k in (1, 2, 3, 5, 10, 20, n):
        _check_statement(w_g, w_prev, n, k)
    words, _ = _check_statement(w_g, w_prev, n, 1)
    assert ops.mask_bits(torch.from_numpy(words.view(np.int32)), n).nonzero().flatten().tolist() == [6]   # NaN sorts above +inf


def test_neurotoxin_mask_refreshes_w_prev():
    n = 200
    w_prev = torch.zeros(n)
    w_g = torch.randn(n, generator=torch.Generator().manual_seed(2))
    mask = torch.full((ops.mask_words(n),), -1, dtype=torch.int32)
    count = torch.zeros(1, dtype=torch.int64)
    ref, ref_count = ops.neurotoxin_statement(w_g, w_prev, n, 7)
    ops.neurotoxin_mask(w_g, w_prev, n, 7, mask, count)
    assert np.array_equal(mask.numpy().view(np.uint32), ref) and int(count) == ref_count == 7
    assert torch.equal(w_prev, w_g)


# ---- the masked optimizer step --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pgd", [0.0, 0.05])
def test_masked_step_matches_the_fp64_statement(pgd):
    n, n_pgd, lr, mom = 1000, 960, 0.1, 0.9
    g0 = torch.Generator().manual_seed(3)
    w0 = torch.randn(n, generator=g0)
    w0[5] = -0.0
    bits = torch.rand(n_pgd, generator=g0) < 0.2
    bits[5] = True
    words = torch.from_numpy(np.packbits(np.concatenate([bits.numpy(), np.zeros(ops.mask_words(n_pgd) * 32 - n_pgd, bool)]),
                                         bitorder="little").view(np.int32).copy())
    assert torch.equal(ops.mask_bits(words, n_pgd), bits)
    opt = ops.FlatSGD(n, "cpu", lr, mom, 10.0, pgd, n_pgd=n_pgd)
    w, m = w0.clone(), torch.zeros(n)
    w64, m64 = w0.double(), torch.zeros(n, dtype=torch.float64)
    for step in range(4):
        g = torch.randn(n, generator=g0) * 5
        opt.step(w, g, m, w0=w0, grad_mask=words)
        gm = g.double().clone()
        gm[:n_pgd][bits] = 0
        coef = min(1.0, 10.0 / (float(gm.norm()) + 1e-6))
        m64 = mom * m64 + coef * gm
        w64 = w64 - lr * m64
        if pgd > 0:
            d = w64[:n_pgd] - w0[:n_pgd].double()
            denom = max(1.0, float(d.norm()) / pgd)
            w64[:n_pgd] = torch.where(bits, w64[:n_pgd], w0[:n_pgd].double() + d / denom)
        torch.testing.assert_close(w.double(), w64, rtol=1e-5, atol=1e-6)
        assert torch.equal(w[:n_pgd][bits].view(torch.int32), w0[:n_pgd][bits].view(torch.int32))    # bitwise, -0 included


def test_empty_mask_step_equals_the_unmasked_step():
    n = 512
    g0 = torch.Generator().manual_seed(4)
    w0, g = torch.randn(n, generator=g0), torch.randn(n, generator=g0)
    opt = ops.FlatSGD(n, "cpu", 0.1, 0.9, 10.0, 0.01)
    a, ma, b, mb = w0.clone(), torch.zeros(n), w0.clone(), torch.zeros(n)
    opt.step(a, g, ma, w0=w0)
    opt.step(b, g, mb, w0=w0, grad_mask=torch.zeros(ops.mask_words(n), dtype=torch.int32))
    assert torch.equal(a, b) and torch.equal(ma, mb)


# ---- the boosted update ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gamma", [0.5, 3.0, 100.0, 1e-3])
def test_boost_update_matches_per_coordinate_fp64(gamma):
    n, nv = 300, 256
    g0 = torch.Generator().manual_seed(5)
    w_g = torch.randn(n, generator=g0)
    slot = w_g + 1e-2 * torch.randn(n, generator=g0)
    before = slot.clone()
    ops.boost_update(slot, w_g, gamma, nv)
    for c in range(nv):
        d = float(np.float32(before[c].numpy() - w_g[c].numpy()))
        assert slot[c].numpy().view(np.uint32) == np.float32(float(w_g[c]) + gamma * d).view(np.uint32)
    assert torch.equal(slot[nv:], before[nv:])                      # BatchNorm statistics are not boosted
    assert np.array_equal(ops.boost_statement(before, w_g, gamma, nv), slot[:nv].numpy())


# ---- engine runs ----------------------------------------------------------------------------------------------------------
def _engine(**kw):
    from rlr_b200.engine import FLEngine
    base = dict(data="fmnist", synthetic=800, synthetic_val=200, num_agents=5, local_ep=1, bs=64, device="cpu", num_corrupt=1,
                poison_frac=0.5, robustLR_threshold=0, log_dir="", seed=5, trainer="torch")
    base.update(kw)
    return FLEngine(make_args(**base), verbose=False)


def _slots(eng, chosen):
    return {a: eng.fused.slots[eng.fused.slot_owner(j)[1]].clone() for j, a in enumerate(chosen)}


def test_inactive_flags_are_the_plain_run_bit_for_bit():
    a, b = _engine(), _engine(attack_boost=1.0, attack_neurotoxin=0.0)
    for r in (1, 2):
        a.run_round(r); b.run_round(r)
    assert torch.equal(a.w_global, b.w_global) and b.neurotoxin_k is None
    a.close(); b.close()


def test_boosted_round_against_the_statement():
    a, b = _engine(), _engine(attack_boost=6.0)
    w_g = a.w_global.clone()
    assert torch.equal(w_g, b.w_global)
    ca, cb = a.run_round(1)["chosen"], b.run_round(1)["chosen"]
    assert ca == cb
    sa, sb = _slots(a, ca), _slots(b, cb)
    nv = a.layout.n_vote
    for agent, s in sa.items():
        if agent < 1:
            assert np.array_equal(sb[agent][:nv].numpy(), ops.boost_statement(s, w_g, 6.0, nv))
            assert torch.equal(sb[agent][nv:], s[nv:])
        else:
            assert torch.equal(sb[agent], s)
    assert not torch.equal(a.w_global, b.w_global)
    a.close(); b.close()


def test_neurotoxin_rounds_against_the_unattacked_run():
    p = 0.02
    a, b = _engine(), _engine(attack_neurotoxin=p)
    nv, k = a.layout.n_vote, math.floor(p * a.layout.n_params)
    assert b.neurotoxin_k == k
    a.run_round(1); b.run_round(1)
    assert torch.equal(a.w_global, b.w_global)                      # round 1: no w_prev, empty mask
    assert int(b.masked_coords) == 0
    w1 = b.w_prev.clone()
    w2 = b.w_global.clone()
    ca, cb = a.run_round(2)["chosen"], b.run_round(2)["chosen"]
    ref_words, ref_count = ops.neurotoxin_statement(w2, w1, nv, k)
    assert np.array_equal(b.attack_mask.numpy().view(np.uint32), ref_words) and int(b.masked_coords) == ref_count >= k
    assert torch.equal(b.w_prev, w2[:nv])
    bits = ops.mask_bits(b.attack_mask, nv)
    sa, sb = _slots(a, ca), _slots(b, cb)
    for agent in sa:
        if agent < 1:
            assert torch.equal(sb[agent][:nv][bits], w2[:nv][bits])  # the corrupt agent never moved the masked coordinates
            assert not torch.equal(sb[agent], sa[agent])
        else:
            assert torch.equal(sb[agent], sa[agent])                 # honest agents are never masked
    a.close(); b.close()


def test_resume_equals_an_uninterrupted_run(tmp_path):
    kw = dict(attack_neurotoxin=0.02, attack_boost=3.0, clip=1.0)
    full = _engine(rounds=4, **kw)
    full.fit()
    ck = str(tmp_path / "ck.pt")
    first = _engine(rounds=2, checkpoint=ck, **kw)
    first.fit()
    assert torch.equal(torch.load(ck, weights_only=False)["extra"]["neurotoxin_w_prev"], first.w_prev)
    second = _engine(rounds=4, resume=ck, **kw)
    assert second.start_round == 3
    second.fit()
    assert torch.equal(second.w_global, full.w_global) and torch.equal(second.w_prev, full.w_prev)
    assert second.last_masked_coords == full.last_masked_coords > 0
    for e in (full, first, second):
        e.close()


def test_resume_without_the_neurotoxin_state_is_an_error(tmp_path):
    ck = str(tmp_path / "ck.pt")
    plain = _engine(rounds=1, checkpoint=ck)
    plain.fit()
    assert "neurotoxin_w_prev" not in torch.load(ck, weights_only=False)["extra"]       # format unchanged without Neurotoxin
    with pytest.raises(ValueError, match="Neurotoxin"):
        _engine(rounds=2, resume=ck, attack_neurotoxin=0.02)
    plain.close()


def test_multikrum_never_admits_a_boosted_update():
    eng = _engine(num_agents=10, num_corrupt=1, select="multikrum", attack_boost=100.0, rounds=3, synthetic=1000)
    hist = eng.fit()
    assert [h["select_corrupt_participants"] for h in hist] == [1, 1, 1]
    assert [h["select_corrupt_admitted"] for h in hist] == [0, 0, 0]
    eng.close()


def _gloo_worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args as mk
    eng = FLEngine(mk(data="fmnist", synthetic=800, synthetic_val=200, num_agents=4, local_ep=1, bs=64, device="cpu", num_corrupt=1,
                      poison_frac=0.5, log_dir="", seed=3, attack_neurotoxin=0.02, attack_boost=2.0), verbose=False)
    counts = []
    for r in range(1, 4):
        eng.run_round(r)
        eng.round_result()
        counts.append(eng.last_masked_coords)
    torch.save({"w": eng.w_global.clone(), "counts": counts, "mask": eng.attack_mask.clone()}, os.path.join(outdir, f"r{rank}.pt"))
    eng.close()
    import torch.distributed as dist
    dist.barrier(); dist.destroy_process_group()


def test_gloo_ranks_agree_on_the_mask():
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_gloo_worker, args=(2, _free_port(), d), nprocs=2, join=True)
        outs = [torch.load(os.path.join(d, f"r{r}.pt")) for r in range(2)]
    assert outs[0]["counts"][0] == 0 and outs[0]["counts"][1] > 0
    assert outs[0]["counts"] == outs[1]["counts"]
    assert torch.equal(outs[0]["w"], outs[1]["w"]) and torch.equal(outs[0]["mask"], outs[1]["mask"])


def test_federated_py_writes_the_attack_field_and_tag(tmp_path):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "federated.py", "--data=fmnist", "--local_ep=1", "--bs=64", "--num_agents=4", "--rounds=2",
                        "--num_corrupt=1", "--poison_frac=0.5", "--synthetic=400", "--synthetic_val=80", "--attack_boost=4",
                        "--attack_neurotoxin=0.01", f"--log_dir={tmp_path}", "--device=cpu"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "Attack (boost / neurotoxin): 4.0 / 0.01" in r.stdout
    run_dirs = os.listdir(tmp_path)
    assert len(run_dirs) == 1
    recs = [json.loads(l) for l in open(tmp_path / run_dirs[0] / "metrics.jsonl")]
    assert [rec["round"] for rec in recs] == [1, 2]
    assert recs[0]["attack_masked_coords"] == 0 and recs[1]["attack_masked_coords"] > 0
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    acc = EventAccumulator(str(tmp_path / run_dirs[0]))
    acc.Reload()
    assert [(e.step, e.value) for e in acc.Scalars("Attack/Masked_Coords")] == [(1, 0.0), (2, float(recs[1]["attack_masked_coords"]))]
