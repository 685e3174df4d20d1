"""Model zoo: parameter counts, flat-buffer views, interop with the reference's nn.Modules (src/models.py)."""
import pytest
import torch

from rlr_b200.models import get_layout, get_model


@pytest.mark.parametrize("name,n_params,shape", [("cnn_mnist", 1_199_882, (1, 28, 28)), ("cnn_cifar", 537_610, (3, 32, 32)),
                                                 ("resnet18", 11_173_962, (3, 32, 32)), ("vgg11", 9_231_114, (3, 32, 32)),
                                                 ("resnet34", 21_282_122, (3, 32, 32)), ("vgg16", 14_728_266, (3, 32, 32))])
def test_param_counts_and_forward_backward(name, n_params, shape):
    net = get_model(name, seed=1)
    lay = net.layout
    assert lay.n_params == n_params and lay.n_vote % 4096 == 0 and lay.n_total % 4096 == 0
    y = net(torch.randn(3, *shape))
    assert y.shape == (3, 10)
    y.logsumexp(1).sum().backward()
    assert float(net.g[: lay.n_vote].abs().sum()) > 0 and float(net.g[lay.n_vote:].abs().sum()) == 0
    for p in lay.params:   # every view aliases the flat buffer
        assert lay.view(net.w, p).data_ptr() == net.w.data_ptr() + 4 * p.offset


def test_dataset_to_model_mapping_like_reference():
    assert get_layout("fmnist").name == "cnn_mnist" and get_layout("fedemnist").name == "cnn_mnist"
    assert get_layout("cifar10").name == "cnn_cifar"
    with pytest.raises(ValueError):
        get_layout("svhn")


@pytest.mark.parametrize("data", ["fmnist", "cifar10"])
def test_same_function_as_reference_module(reference_outputs, data):
    """Our flat parameters loaded into the reference's nn.Module via to_reference_vector (stored logits of that module): logits must
    agree."""
    net = get_model(data, seed=3).eval()
    vec = net.layout.to_reference_vector(net.w)
    assert vec.numel() == reference_outputs[f"model/{data}/n_ref_params"]
    x = torch.randn(5, *net.layout.in_shape, generator=torch.Generator().manual_seed(0))
    torch.testing.assert_close(net(x), reference_outputs[f"model/{data}/logits"], atol=1e-4, rtol=1e-4)
    # and the round trip
    w2 = torch.zeros_like(net.w)
    net.layout.from_reference_vector(vec, w2)
    torch.testing.assert_close(w2[: net.layout.n_vote], net.w[: net.layout.n_vote])


def test_bn_buffers_live_behind_n_vote_and_update_in_train_mode():
    net = get_model("vgg11")
    lay = net.layout
    assert all(b.offset >= lay.n_vote for b in lay.buffers) and lay.n_buffers == 2 * 2752
    before = net.w[lay.n_vote:].clone()
    net.train()
    net(torch.randn(4, 3, 32, 32))
    assert not torch.equal(before, net.w[lay.n_vote:])
    net.eval()
    mid = net.w[lay.n_vote:].clone()
    net(torch.randn(4, 3, 32, 32))
    assert torch.equal(mid, net.w[lay.n_vote:])


def test_init_statistics_follow_torch_defaults():
    lay = get_layout("cnn_mnist")
    w = lay.init_(torch.zeros(lay.n_total), 0)
    fc1 = lay.view(w, lay.by_name["fc1.weight"])
    bound = 1.0 / (9216 ** 0.5)
    assert float(fc1.abs().max()) <= bound and abs(float(fc1.std()) - bound / 3 ** 0.5) < 0.1 * bound
