"""Record the reference implementation's outputs for the differential tests as tests/golden/reference_outputs.pt.

    python scripts/make_reference_golden.py REFERENCE_ROOT

REFERENCE_ROOT is a checkout of TinfoilHat0/Defending-Against-Backdoors-with-Robust-Learning-Rate (its src/ is imported).  The
inputs of every case are generated here exactly as the tests generate them (seeded), so the tests compare the project against these
stored outputs without the reference being present.  Large vectors are stored as a fixed, seeded sample of their coordinates.
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

LOCAL_TRAIN_SAMPLE = 8000     # coordinates of each local-training update vector kept (seeded choice, see local_train_sample_index)


def local_train_sample_index(numel):
    return torch.from_numpy(np.sort(np.random.default_rng(0).choice(numel, size=min(numel, LOCAL_TRAIN_SAMPLE), replace=False)))


def main(ref_root):
    src = os.path.join(ref_root, "src")
    sys.path.insert(0, src)
    import importlib
    utils, aggregation, models, options, agent = (importlib.import_module(m) for m in ("utils", "aggregation", "models", "options", "agent"))
    import rlr_b200  # noqa: F401
    from rlr_b200.data import make_synthetic
    from rlr_b200.models import get_layout, get_model
    import test_aggregation as ta
    import test_partition as tp
    import test_poison as tpo
    import test_reference_differential as trd

    out = {}
    # aggregation class (tests/test_aggregation.py::test_matches_reference_class)
    for aggr in ("avg", "comed", "sign"):
        for theta in (0, 1, 3, 5):
            K, n = 5, 2000
            w0, ws = ta._mk(K, n, seed=theta)
            sizes = {i: 100 + 7 * i for i in range(K)}
            args = SimpleNamespace(aggr=aggr, robustLR_threshold=theta, server_lr=0.7 if aggr == "sign" else 1.0, noise=0, clip=0, device="cpu")
            model = torch.nn.Linear(n, 1, bias=False)
            model.weight.data.copy_(w0.view(1, n))
            aggregation.Aggregation(sizes, n, None, args, None).aggregate_updates(model, {i: (ws[i].double() - w0) for i in range(K)}, 1)
            out[f"aggregate/{aggr}/{theta}"] = model.weight.data.view(-1).clone()
    # named helpers (test_reference_named_helpers_match_reference)
    K, n = 4, 500
    w0, ws = ta._mk(K, n, seed=3)
    ups = {i: (ws[i].double() - w0) for i in range(K)}
    sizes = {i: 10 * (i + 1) for i in range(K)}
    ref = aggregation.Aggregation(sizes, n, None, SimpleNamespace(aggr="avg", robustLR_threshold=3, server_lr=1.0, noise=0, clip=0.5,
                                                                   device="cpu"), None)
    out["helpers/robustLR"] = ref.compute_robustLR({k: v.clone() for k, v in ups.items()})
    out["helpers/avg"], out["helpers/comed"], out["helpers/sign"] = ref.agg_avg(ups), ref.agg_comed(ups), ref.agg_sign(ups)
    b = {k: v.clone() for k, v in ups.items()}
    ref.clip_updates(b)
    out["helpers/clipped"] = torch.stack([b[k] for k in range(K)])
    # option defaults (tests/test_options.py::test_defaults_match_reference_parser)
    argv, sys.argv = sys.argv, ["federated.py"]
    out["options/defaults"] = {k: v for k, v in vars(options.args_parser()).items() if k != "device"}
    sys.argv = argv
    # partitioner (tests/test_partition.py::test_matches_reference)
    for K, n in [(2, 1000), (7, 6000), (8, 5000), (10, 2000), (40, 4000)]:
        tr, _ = make_synthetic("cifar10", n)
        groups = utils.distribute_data(tp._Wrap(tr), SimpleNamespace(num_agents=K))
        out[f"partition/{K}/{n}"] = [torch.tensor(list(groups[u]), dtype=torch.int32) for u in range(K)]
    # trojan patterns (tests/test_poison.py::test_add_pattern_matches_reference); the reference reads its pattern images cwd-relative
    cwd = os.getcwd()
    os.chdir(src)
    try:
        for ds, pat, ag in tpo.PATTERN_CASES:
            x = tpo.pattern_input(ds)
            r = utils.add_pattern_bd(x.clone() if ds != "cifar10" else x.numpy().copy(), ds, pattern_type=pat, agent_idx=ag)
            out[f"pattern/{ds}/{pat}/{ag}"] = torch.from_numpy(np.array(np.asarray(r, dtype=np.float32 if ds == "fedemnist" else None)))
    finally:
        os.chdir(cwd)
    # model functions (tests/test_models.py::test_same_function_as_reference_module)
    for data in ("fmnist", "cifar10"):
        m = models.get_model(data).eval()
        net = get_model(data, seed=3).eval()
        torch.nn.utils.vector_to_parameters(net.layout.to_reference_vector(net.w), m.parameters())
        x = torch.randn(5, *net.layout.in_shape, generator=torch.Generator().manual_seed(0))
        with torch.no_grad():
            out[f"model/{data}/logits"] = m(x)
        out[f"model/{data}/n_ref_params"] = sum(p.numel() for p in m.parameters())
    # one local step of the reference Agent (test_local_train_update_matches_reference_agent)
    for data, clip in trd.LOCAL_TRAIN_CASES:
        n = 48
        train, _ = make_synthetic(data, n, 16, seed=4)
        ref_args = SimpleNamespace(num_corrupt=0, bs=n, local_ep=1, client_lr=0.1, client_moment=0.9, clip=clip, device="cpu", num_workers=0,
                                   data=data)
        m = models.get_model(data)
        for mod in m.modules():
            if isinstance(mod, torch.nn.Dropout2d):
                mod.p = 0.0
        lay = get_layout(data)
        torch.nn.utils.vector_to_parameters(lay.to_reference_vector(trd.local_train_init(lay)), m.parameters())
        upd = agent.Agent(0, ref_args, trd._RefView(train), list(range(n))).local_train(m, torch.nn.CrossEntropyLoss())
        out[f"local_train/{data}/{clip}"] = upd[local_train_sample_index(upd.numel())].clone()
        out[f"local_train/{data}/{clip}/norm"] = float(upd.norm())
    # evaluation (test_evaluation_matches_reference_function)
    _, val = make_synthetic("cifar10", 64, 90, seed=7)
    lay = get_layout("cnn_cifar")
    w = lay.init_(torch.zeros(lay.n_total), 5)
    m = models.get_model("cifar10").eval()
    torch.nn.utils.vector_to_parameters(lay.to_reference_vector(w), m.parameters())
    loader = torch.utils.data.DataLoader(trd._RefView(val), batch_size=32, shuffle=False)
    loss, (acc, pc) = utils.get_loss_n_accuracy(m, torch.nn.CrossEntropyLoss(), loader, SimpleNamespace(device="cpu"))
    out["evaluation"] = {"loss": float(loss), "acc": float(acc), "per_class": pc.float().clone()}

    dst = os.path.join(ROOT, "tests", "golden", "reference_outputs.pt")
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    torch.save(out, dst)
    print(dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
