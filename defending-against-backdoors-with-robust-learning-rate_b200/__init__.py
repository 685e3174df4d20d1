"""robust-fl: a Hopper-native federated-learning engine with the Robust Learning Rate defense.

Capabilities mirror TinfoilHat0/Defending-Against-Backdoors-with-Robust-Learning-Rate
(reference layer map: SURVEY.md section 1), re-designed for one-process-per-GPU execution on H100:

* ``options``      CLI flags (reference src/options.py:4-74) + engine flags
* ``data``         device-resident datasets, partitioner, backdoor poisoner (reference src/utils.py)
* ``models``       CNN_MNIST / CNN_CIFAR (reference src/models.py) + ResNet-18 / VGG-11, flat-buffer params
* ``ops``          hand-written sm_90a kernels (+ fp32 torch oracles used on CPU and in tests)
* ``parallel``     process groups, symmetric memory, fused P2P aggregate+broadcast
* ``agent`` / ``aggregation`` / ``engine`` / ``federated``   client, server and round driver
* ``utils``        evaluation, logging, timers, checkpointing
"""
__version__ = "0.1.0"
