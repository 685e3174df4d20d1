"""Evaluation, logging, timing, checkpointing (SURVEY.md section 5 auxiliary subsystems)."""
from .evaluate import backdoor_lifespan, get_loss_n_accuracy
from .logging import MetricLogger
from .timers import PhaseTimer
from .checkpoint import save_checkpoint, load_checkpoint, restore_server_opt



def __getattr__(name):
    """Name parity with the reference's ``utils`` module (src/utils.py): ``utils.get_datasets``, ``utils.distribute_data``,
    ``utils.poison_dataset``, ``utils.add_pattern_bd``, ``utils.DatasetSplit``, ``utils.H5Dataset``, ``utils.print_exp_details``
    resolve to their homes in ``data`` / ``options`` (lazily, to avoid import cycles)."""
    if name in ("get_datasets", "distribute_data", "poison_dataset", "add_pattern_bd", "DatasetSplit", "H5Dataset", "DeviceDataset"):
        from .. import data
        return getattr(data, name)
    if name == "print_exp_details":
        from ..options import print_exp_details
        return print_exp_details
    raise AttributeError(name)


__all__ = ["backdoor_lifespan", "get_loss_n_accuracy", "MetricLogger", "PhaseTimer", "save_checkpoint", "load_checkpoint", "restore_server_opt"]
