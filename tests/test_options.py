"""CLI parity with the reference flag table (src/options.py:4-74, SURVEY.md 5.6)."""
import pytest

from rlr_b200.options import args_parser, finalize_args, make_args, print_exp_details

REF_DEFAULTS = dict(data="fmnist", num_agents=10, agent_frac=1, num_corrupt=0, rounds=200, aggr="avg", local_ep=2, bs=256,
                    client_lr=0.1, client_moment=0.9, server_lr=1, base_class=5, target_class=7, poison_frac=0.0,
                    pattern_type="plus", robustLR_threshold=0, clip=0, noise=0, top_frac=100, snap=1, num_workers=0)


def test_defaults_match_reference_table():
    a = args_parser([])
    for k, v in REF_DEFAULTS.items():
        assert getattr(a, k) == v, k


def test_defaults_match_reference_parser(reference_outputs):
    ref = reference_outputs["options/defaults"]          # vars(args_parser()) of the reference's options.py, without "device"
    ours = vars(args_parser([]))
    for k, v in ref.items():
        if k == "device":
            continue
        assert ours[k] == v, k


def test_runner_sh_command_lines_parse():
    for line in ["--data=fmnist --local_ep=2 --bs=256 --num_agents=10 --rounds=200 --num_corrupt=1 --poison_frac=0.5 --robustLR_threshold=4 --device=cuda:1",
                 "--data=cifar10 --local_ep=2 --bs=256 --num_agents=40 --rounds=200 --num_corrupt=4 --poison_frac=0.5 --robustLR_threshold=8",
                 "--data=fedemnist --num_agents=3383 --agent_frac=0.01 --num_corrupt=338 --poison_frac=0.5 --local_ep=10 --bs=64 --rounds=500 --snap=5"]:
        a = finalize_args(args_parser(line.split()))
        assert a.model in ("cnn_mnist", "cnn_cifar")


def test_server_lr_forced_to_one_unless_sign():
    assert make_args(aggr="avg", server_lr=0.3).server_lr == 1.0
    assert make_args(aggr="comed", server_lr=0.3).server_lr == 1.0
    assert make_args(aggr="sign", server_lr=0.3).server_lr == 0.3


def test_unknown_values_rejected():
    with pytest.raises(ValueError):
        make_args(aggr="krum")
    with pytest.raises(ValueError):
        make_args(data="imagenet")
    with pytest.raises(AttributeError):
        make_args(not_a_flag=1)


def test_banner_prints(capsys):
    print_exp_details(make_args())
    out = capsys.readouterr().out
    for field in ["Dataset", "Global Rounds", "Aggregation Function", "RobustLR_threshold", "Poison Frac", "Clip"]:
        assert field in out
