"""Headline benchmark: FL rounds/sec (device-timed, max over ranks) -- CIFAR-10 ResNet-18, FedAvg, bf16,
num_agents = number of GPUs, local_ep=2, bs=256, 50,000 synthetic CIFAR-shaped training images (BASELINE.json).

    python bench.py [--gpus N --steps K --warmup W] [--impl ours|reference] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        bench.py --gpus N --steps K --warmup W

A "step" is one federated round = every agent trains local_ep epochs on its shard (one agent per GPU, all GPUs in
parallel) + fused aggregation / server step / parameter hand-off.  Total work per round is fixed (the 50k-image
dataset is split over the agents), so scaling is STRONG.  Evaluation is outside the timed region for both arms
(BASELINE.md section 2).  Rank 0 prints ONE JSON line.

--dump-outputs DIR (ours): after the timed rounds, rank 0 writes what the last timed round produced -- the global parameter
vector after aggregation, the round's summed training loss and its flipped-coordinate count -- as DIR/<name>.npy (float32 /
float64, at most 64 MB), so two builds run with the same arguments (same seeded inputs) can be compared output for output.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=3)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--impl", type=str, default="ours", choices=("ours", "reference"))
    p.add_argument("--model", type=str, default="resnet18")
    p.add_argument("--data", type=str, default="cifar10")
    p.add_argument("--train_size", type=int, default=50000)
    p.add_argument("--local_ep", type=int, default=2)
    p.add_argument("--bs", type=int, default=256)
    p.add_argument("--aggr", type=str, default="avg")
    p.add_argument("--theta", type=int, default=0)
    p.add_argument("--num_corrupt", type=int, default=0)
    p.add_argument("--poison_frac", type=float, default=0.0)
    p.add_argument("--trainer", type=str, default="auto")
    p.add_argument("--backend", type=str, default="auto")
    p.add_argument("--dtype", type=str, default="bf16")
    p.add_argument("--no_e2e", action="store_true")
    p.add_argument("--agents", type=int, default=0,
                   help="number of FL agents (default 0 = one per GPU, the headline config); more agents than GPUs are time-multiplexed "
                        "-- e.g. --agents 10 --gpus 1 is the reference README's FMNIST setting")
    p.add_argument("--agents_in_flight", type=int, default=0, help="agents a GPU trains concurrently (ours only; 0 = the engine's auto rule)")
    p.add_argument("--agent_frac", type=float, default=1.0, help="fraction of the agents sampled per round (reference --agent_frac)")
    p.add_argument("--pattern_type", type=str, default="plus")
    p.add_argument("--no_fused_handoff", action="store_true", help="ours: keep round_init + the aggregation kernel's barrier-out (A/B of the hand-off fusion)")
    p.add_argument("--dump-outputs", dest="dump_outputs", type=str, default=None, metavar="DIR",
                   help="ours: write the outputs of the last timed round as DIR/<name>.npy")
    return p.parse_args()


DUMP_LIMIT_BYTES = 64 << 20


def dump_outputs(eng, out_dir, write=True):
    """Outputs of the round that just ran, as a caller of FLEngine.run_round receives them: the global parameters (float32; a fixed,
    seeded sample of them if the whole vector would exceed the size limit), the summed training loss and the flipped count (float64)."""
    import numpy as np
    loss, flipped = eng.round_result()          # collective on multi-GPU runs: every rank takes part, rank 0 writes
    w = eng.global_params().float().cpu().numpy()
    if not write:
        return
    os.makedirs(out_dir, exist_ok=True)
    budget = (DUMP_LIMIT_BYTES - (1 << 20)) // 4
    if w.size > budget:
        idx = np.sort(np.random.default_rng(0).choice(w.size, size=budget, replace=False))
        np.save(os.path.join(out_dir, "global_params_sample_index.npy"), idx.astype(np.float64))
        w = w[idx]
    np.save(os.path.join(out_dir, "global_params.npy"), w)
    np.save(os.path.join(out_dir, "train_loss_sum.npy"), np.array([loss], dtype=np.float64))
    np.save(os.path.join(out_dir, "flipped.npy"), np.array([flipped], dtype=np.float64))


class ClockSampler:
    """nvidia-smi clock / throttle-reason sampler running DURING the timed region (clocks and throttle reasons are part of every timing)."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index=0):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        self.p = None
        try:
            self.p = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "200",
                                       "-i", str(gpu_index)], stdout=self.f, stderr=subprocess.DEVNULL)
        except Exception:  # noqa: BLE001
            self.p = None

    def stop(self):
        if self.p is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.25)
        self.p.terminate()
        try:
            self.p.wait(timeout=5)
        except Exception:  # noqa: BLE001
            self.p.kill()
        self.f.flush()
        rows = [r.strip().split(", ") for r in open(self.f.name).read().strip().splitlines() if r.strip()]
        os.unlink(self.f.name)
        sm, mx, power, reasons = [], [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in rows:
            try:
                sm.append(float(r[1])); mx.append(float(r[2])); power.append(float(r[3]))
                for nm, v in zip(names, r[5:9]):
                    if v.strip().lower().startswith("active"):
                        reasons.add(nm)
            except Exception:  # noqa: BLE001
                continue
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no samples"]}
        load = [s for s, pw in zip(sm, power) if pw > 0.5 * max(power)] or sm
        return {"sm_mhz": statistics.median(load), "sm_max_mhz": max(mx), "power_w_max": max(power),
                "samples": len(sm), "reasons": sorted(reasons)}


def config_dict(a, n, impl):
    k = a.agents or n                     # agents: one per GPU unless --agents
    return {"model": a.model, "dataset": f"{a.data} (synthetic, {a.train_size} train images)", "num_agents": k,
            "agents_per_gpu": (k + n - 1) // n if impl == "ours" else k, "agents_in_flight": (a.agents_in_flight or "auto") if impl == "ours" else 1,
            "global_batch": a.bs * n if impl == "ours" else a.bs,
            "local_batch": a.bs, "local_ep": a.local_ep, "aggr": a.aggr, "robustLR_threshold": a.theta,
            "num_corrupt": a.num_corrupt, "poison_frac": a.poison_frac, "agent_frac": a.agent_frac, "seq_len": None,
            "parallelism": f"agent-parallel: {k} agent(s) on {n} GPU(s)" if impl == "ours" else f"{k} agent(s) sequential on 1 GPU (reference design)",
            "l2_policy": "inputs larger than L2: each step streams a fresh batch from the 150 MB device-resident dataset plus "
                         "4x45 MB flat parameter/grad/momentum buffers and >100 MB of activations (H100 L2 = 50 MB)",
            "timed_region": "local training of all agents + aggregation + parameter hand-off; evaluation excluded"}


def run_reference(a):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return  # the reference is a single-process, single-GPU simulation: extra ranks have nothing to do
    sys.path.insert(0, os.path.join(ROOT, "baseline"))
    import run_reference as rr
    if not rr.reference_available():
        from install_reference import install
        if not install():
            print(json.dumps({"impl": "reference", "unavailable": "baseline/_ref missing and /root/reference not mounted"}))
            return
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"impl": "reference", "unavailable": "no CUDA device visible"}))
        return
    if a.data == "fedemnist":
        print(json.dumps({"impl": "reference", "unavailable": "the reference reads Fed-EMNIST from one pickled file per client (src/agent.py:16-20); "
                          "the dataset is not in this image and the synthetic shim only replaces utils.get_datasets"}))
        return
    clocks = ClockSampler(0)
    t0 = time.time()
    res = rr.run(data=a.data, model=a.model, num_agents=a.agents or a.gpus, local_ep=a.local_ep, bs=a.bs, aggr=a.aggr,
                 train_size=a.train_size, steps=a.steps, warmup=a.warmup, theta=a.theta, num_corrupt=a.num_corrupt,
                 poison_frac=a.poison_frac, device="cuda:0", agent_frac=a.agent_frac)
    ck = clocks.stop()
    out = {"impl": "reference", "metric": "fl_rounds_per_sec", "value": res["rounds_per_s"], "unit": "rounds/s",
           "n_gpus": a.gpus, "steps": a.steps, "warmup": a.warmup, "ms_per_step": res["ms_per_round"],
           "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "fp32 (reference has no AMP; cuDNN TF32 convs)",
           "data": "synthetic", "config": config_dict(a, a.gpus, "reference"), "clocks": ck,
           "e2e": {"value": a.steps / res["wall_s"], "unit": "rounds/s", "h2d_bytes_per_step": res["h2d_bytes_per_round"],
                   "d2h_bytes_per_step": 0, "note": "wall clock of the same rounds; the reference copies every batch from pageable host memory"},
           "gpu_launches": 0,
           "note": ("unmodified reference Agent/Aggregation loop on 1 GPU"
                    + ("; ResNet / VGG are not in the reference: plain torch.nn definition from baseline/torch_models.py" if a.model in ("resnet18", "resnet34", "vgg11", "vgg16") else "")),
           "wall_s_total": time.time() - t0}
    print(json.dumps(out))


def ops_fallbacks():
    """Library fall-throughs of the sm100 back-end recorded while the steps were built / captured ({} = none)."""
    from rlr_b200 import ops
    return ops.fallback_calls()


def aggregation_check(eng, ctx, a):
    """Correctness evidence for the multi-GPU fused path, OUTSIDE the timed region: one extra round in which every rank also
    recomputes the server step from an all_gather of the participants' parameters with the fp64 oracle (ops.aggregate_oracle,
    the re-statement of src/aggregation.py:19-45) and compares it with what the fused P2P/multicast kernel left in its
    ``w_global``; plus a bit-wise comparison of ``w_global`` across ranks."""
    import torch
    from rlr_b200 import ops
    try:
        rnd = 20_000
        chosen = eng.place_participants(eng.sample_agents(rnd))
        prev = eng.w_global.clone()
        # local training only (the engine's own code path), then gather BEFORE the fused kernel consumes the slots
        eng.args.noise, noise_keep = 0.0, eng.args.noise                      # Philox noise has no oracle stream: check without it
        eng.run_round(rnd)
        eng.args.noise = noise_keep
        ws = eng.fused.gather_participants(len(chosen))
        weights = [float(eng.agent_data_sizes[i]) for i in chosen]
        want, want_flipped = ops.aggregate_oracle(prev, ws, weights, eng.args.aggr, eng.args.robustLR_threshold, eng.args.server_lr,
                                                  None, eng.layout.n_vote)
        got = eng.global_params()
        err = (got.double() - want.double()).abs().max()
        scale = (want.double() - prev.double()).abs().max()
        allw = ctx.all_gather(got)
        same = bool((allw == allw[0:1]).all().item())
        stats = torch.stack([err, scale])
        ctx.all_reduce_max(stats)
        _, flipped = eng.round_result()
        pad = (eng.layout.n_vote - eng.layout.n_params) if eng.args.robustLR_threshold > 0 else 0
        return {"agg_check_max_abs_err": float(stats[0]), "max_abs_update": float(stats[1]), "all_ranks_equal": same,
                "flipped_kernel": flipped, "flipped_oracle": int(want_flipped) - pad, "participants": len(chosen),
                "oracle": "fp64 ops.aggregate_oracle on an NCCL all_gather of the slots (src/aggregation.py:19-45 semantics)"}
    except Exception as e:  # noqa: BLE001
        return {"error": f"{type(e).__name__}: {str(e)[:200]}"}


def run_ours(a):
    import torch
    from rlr_b200.engine import FLEngine
    from rlr_b200.options import make_args
    from rlr_b200.parallel import init_distributed

    ctx = init_distributed(None, None)
    n = ctx.world
    if n != a.gpus and ctx.is_main:
        print(f"[bench] warning: --gpus {a.gpus} but WORLD_SIZE={n}; using {n}", file=sys.stderr)
    def make_engine(trainer):
        args = make_args(data=a.data, model=a.model, num_agents=a.agents or n, agents_in_flight=a.agents_in_flight, local_ep=a.local_ep, bs=a.bs,
                         aggr=a.aggr,
                         robustLR_threshold=a.theta, num_corrupt=a.num_corrupt, poison_frac=a.poison_frac, agent_frac=a.agent_frac,
                         pattern_type=a.pattern_type, no_fused_handoff=a.no_fused_handoff,
                         synthetic=a.train_size, synthetic_val=1000, snap=10 ** 9, rounds=10 ** 9, log_dir="",
                         trainer=trainer, backend=a.backend, dtype=a.dtype, seed=0)
        return FLEngine(args, ctx=ctx, verbose=False)

    dev = ctx.device
    cuda = dev.type == "cuda"
    notes = []
    eng = make_engine(a.trainer)

    def sync():
        ctx.barrier()
        if cuda:
            torch.cuda.synchronize(dev)

    def timed(k, first_round, stream):
        sync()
        if cuda:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        t0 = time.perf_counter()
        h2d = d2h = 0
        res = None
        for r in range(k):
            info = eng.run_round(first_round + r, stream_inputs=stream)
            h2d += info["h2d_bytes"]
            if stream:
                res = eng.round_result()            # device -> host read of the round's result
                d2h += 16
        if cuda:
            e1.record()
        sync()
        ms = e0.elapsed_time(e1) if cuda else (time.perf_counter() - t0) * 1e3
        t = torch.tensor([ms], dtype=torch.float64, device=dev)
        ctx.all_reduce_max(t)
        return float(t.item()), h2d, d2h, res, info

    for r in range(a.warmup):
        eng.run_round(r + 1)
    eng.timer.elapsed()  # drop warm-up spans
    clocks = ClockSampler(dev.index or 0) if (ctx.is_main and cuda) else None
    ms, _, _, _, info = timed(a.steps, a.warmup + 1, False)
    ck = clocks.stop() if clocks else {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["cpu run"]}
    if a.dump_outputs:
        dump_outputs(eng, a.dump_outputs, write=ctx.is_main)
        ctx.barrier()
    phases = eng.timer.elapsed()
    e2e = None
    if not a.no_e2e:
      try:
        eng.enable_input_streaming()
        eng.run_round(10_000, stream_inputs=True)  # warm the streaming path (captures graphs for the streamed shards)
        ms2, h2d, d2h, res, _ = timed(a.steps, 10_001, True)
        tot = torch.tensor([float(h2d), float(d2h)], dtype=torch.float64, device=dev)
        ctx.all_reduce_sum(tot)
        e2e = {"value": a.steps * 1e3 / ms2, "unit": "rounds/s", "h2d_bytes_per_step": tot[0].item() / a.steps,
               "d2h_bytes_per_step": tot[1].item() / a.steps, "ms_per_step": ms2 / a.steps,
               "note": "every round re-uploads each trained shard (uint8 images + labels) from pinned host memory and reads "
                       "the round's training-loss / flipped-coordinate result back to the host",
               "last_result": {"train_loss_sum": res[0], "flipped": res[1]} if res else None}
      except Exception as e:  # noqa: BLE001  -- never lose the device-timed line because the end-to-end pass failed
        notes.append(f"e2e pass failed: {type(e).__name__}: {str(e)[:160]}")
    launches = eng.trainer.launches_per_step() * info["steps"] * a.steps + 2 * a.steps  # + round_init + fused aggregate
    agg_check = aggregation_check(eng, ctx, a) if n > 1 else None
    if ctx.is_main:
        out = {"impl": "ours", "metric": "fl_rounds_per_sec", "value": a.steps * 1e3 / ms, "unit": "rounds/s", "n_gpus": n,
               "steps": a.steps, "warmup": a.warmup, "ms_per_step": ms / a.steps, "higher_is_better": True,
               "scaling": "strong", "vs_baseline": None, "dtype": a.dtype if cuda else "fp32", "data": "synthetic",
               "config": {**config_dict(a, n, "ours"), "trainer": eng.trainer.name, "agg_backend": eng.fused.backend,
                          "symm_provider": eng.fused.buf.provider, "multicast": bool(getattr(eng.fused, "use_multimem", False)),
                          "local_steps_per_round_per_gpu": info["steps"], "n_params": eng.layout.n_params,
                          "fused_handoff": bool(eng.handoff), "agents_in_flight_used": len(eng.trainers)},
               "clocks": ck, "e2e": e2e, "gpu_launches": int(launches), "notes": notes,
               "library_fallbacks": ops_fallbacks(), "agg_check": agg_check,
               "phase_ms_per_round_rank0": {k: v / a.steps for k, v in phases.items()}}
        print(json.dumps(out))
    eng.close()
    if ctx.is_dist:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    a = parse()
    if a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)
