"""Model definitions as IR programs.

``cnn_mnist`` / ``cnn_cifar`` are the reference's two networks (src/models.py:11-31, :33-58), layer for layer.
``resnet18`` / ``vgg11`` are NOT in the reference (SURVEY.md fact 3): they are the CIFAR variants named by
BASELINE.json -- ResNet-18 with a 3x3 stem and no max-pool (11,173,962 parameters) and VGG-11-BN with a single
``Linear(512,10)`` head (9,231,114 parameters).  ``resnet34`` / ``vgg16`` are the deeper members of the same two
families (same layer types, hence the same kernels).

``resnet18_gn`` / ``resnet34_gn`` / ``vgg11_gn`` / ``vgg16_gn`` replace every BatchNorm of their twin by GroupNorm with 32 groups
(Wu & He 2018), the usual normalisation of these networks in federated learning (Hsieh et al. 2020; Reddi et al. 2021): no running
statistics, so every coordinate of the flat vector takes part in the robust aggregation and evaluation normalises exactly as
training does.  Parameter names and counts equal the BatchNorm twin's.
"""
from __future__ import annotations

from .graph import Node


def cnn_mnist():
    """reference CNN_MNIST: conv(1,32,3) relu conv(32,64,3) relu pool flatten drop fc(9216,128) relu drop fc(128,10)."""
    n = [
        Node("conv", "conv1", attrs=dict(cin=1, cout=32, k=3)), Node("relu"),
        Node("conv", "conv2", attrs=dict(cin=32, cout=64, k=3)), Node("relu"),
        Node("maxpool"), Node("flatten"), Node("dropout", attrs=dict(p=0.5)),
        Node("linear", "fc1", attrs=dict(cin=9216, cout=128)), Node("relu"), Node("dropout", attrs=dict(p=0.5)),
        Node("linear", "fc2", attrs=dict(cin=128, cout=10)),
    ]
    return n, (1, 28, 28)


def cnn_cifar():
    """reference CNN_CIFAR: [conv3 relu pool]x3 (3-64-128-256) flatten drop fc128 relu drop fc256 relu drop fc10."""
    n = []
    for i, (ci, co) in enumerate([(3, 64), (64, 128), (128, 256)], 1):
        n += [Node("conv", f"conv{i}", attrs=dict(cin=ci, cout=co, k=3)), Node("relu"), Node("maxpool")]
    n += [Node("flatten"), Node("dropout", attrs=dict(p=0.5)),
          Node("linear", "fc1", attrs=dict(cin=1024, cout=128)), Node("relu"), Node("dropout", attrs=dict(p=0.5)),
          Node("linear", "fc2", attrs=dict(cin=128, cout=256)), Node("relu"), Node("dropout", attrs=dict(p=0.5)),
          Node("linear", "fc3", attrs=dict(cin=256, cout=10))]
    return n, (3, 32, 32)


GN_GROUPS = 32


def _norm(norm, name, c, **kw):
    """Normalisation node: BatchNorm (``bn``) or GroupNorm with GN_GROUPS groups (``gn``)."""
    if norm == "bn":
        return Node("bn", name, attrs=dict(c=c), **kw)
    return Node("gn", name, attrs=dict(c=c, groups=GN_GROUPS), **kw)


def _resnet(blocks, num_classes=10, norm="bn"):
    n = [Node("conv", "conv1", attrs=dict(cin=3, cout=64, k=3, pad=1, bias=False)), _norm(norm, "bn1", 64), Node("relu")]
    cin = 64
    for li, (cout, stride) in enumerate([(64, 1), (128, 2), (256, 2), (512, 2)], 1):
        for bi in range(blocks[li - 1]):
            s = stride if bi == 0 else 1
            pre = f"layer{li}.{bi}"
            n.append(Node("save", out="id"))
            n += [Node("conv", pre + ".conv1", attrs=dict(cin=cin, cout=cout, k=3, stride=s, pad=1, bias=False)),
                  _norm(norm, pre + ".bn1", cout), Node("relu"),
                  Node("conv", pre + ".conv2", attrs=dict(cin=cout, cout=cout, k=3, pad=1, bias=False)),
                  _norm(norm, pre + ".bn2", cout)]
            if s != 1 or cin != cout:
                n += [Node("conv", pre + ".downsample.0", inp="id", out="id",
                           attrs=dict(cin=cin, cout=cout, k=1, stride=s, pad=0, bias=False)),
                      _norm(norm, pre + ".downsample.1", cout, inp="id", out="id")]
            n += [Node("add", attrs=dict(other="id")), Node("relu")]
            cin = cout
    n += [Node("avgpool"), Node("flatten"), Node("linear", "fc", attrs=dict(cin=512, cout=num_classes))]
    return n, (3, 32, 32)


def resnet18(num_classes=10):
    """CIFAR ResNet-18 (BasicBlock x [2,2,2,2], 3x3 stem, no max-pool): 11,173,962 parameters."""
    return _resnet((2, 2, 2, 2), num_classes)


def resnet34(num_classes=10):
    """CIFAR ResNet-34 (BasicBlock x [3,4,6,3]): same layer types as ResNet-18, so every layer runs on the same kernels."""
    return _resnet((3, 4, 6, 3), num_classes)


_VGG = {"vgg11": [64, "M", 128, "M", 256, 256, "M", 512, 512, "M", 512, 512, "M"],
        "vgg16": [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M"]}


def _vgg(cfg, num_classes=10, norm="bn"):
    n, cin, i = [], 3, 0
    for v in _VGG[cfg]:
        if v == "M":
            n.append(Node("maxpool"))
        else:
            n += [Node("conv", f"features.{i}", attrs=dict(cin=cin, cout=v, k=3, pad=1)),
                  _norm(norm, f"features.{i + 1}", v), Node("relu")]
            cin, i = v, i + 3
            continue
        i += 1
    n += [Node("flatten"), Node("linear", "classifier", attrs=dict(cin=512, cout=num_classes))]
    return n, (3, 32, 32)


def vgg11(num_classes=10):
    """VGG-11-BN with a single Linear(512, 10) head: 9,231,114 parameters."""
    return _vgg("vgg11", num_classes)


def vgg16(num_classes=10):
    """VGG-16-BN, same head."""
    return _vgg("vgg16", num_classes)


def resnet18_gn(num_classes=10):
    """ResNet-18 with GroupNorm(32) in place of every BatchNorm: 11,173,962 parameters, no buffers."""
    return _resnet((2, 2, 2, 2), num_classes, "gn")


def resnet34_gn(num_classes=10):
    """ResNet-34 with GroupNorm(32)."""
    return _resnet((3, 4, 6, 3), num_classes, "gn")


def vgg11_gn(num_classes=10):
    """VGG-11 with GroupNorm(32): 9,231,114 parameters, no buffers."""
    return _vgg("vgg11", num_classes, "gn")


def vgg16_gn(num_classes=10):
    """VGG-16 with GroupNorm(32)."""
    return _vgg("vgg16", num_classes, "gn")


ZOO = {"cnn_mnist": cnn_mnist, "cnn_cifar": cnn_cifar, "resnet18": resnet18, "resnet34": resnet34, "vgg11": vgg11, "vgg16": vgg16,
       "resnet18_gn": resnet18_gn, "resnet34_gn": resnet34_gn, "vgg11_gn": vgg11_gn, "vgg16_gn": vgg16_gn}
