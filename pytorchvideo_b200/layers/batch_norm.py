"""Naive synchronised BatchNorm (reference layers/batch_norm.py): same constructors, attributes and state_dict.

The engine is eval-only, where these are plain BatchNorm: the lowering folds their running statistics into the GEMM or
convolution epilogue before them (engine/lower.py).  The cross-device statistics of training mode are not implemented,
so they have no forward of their own."""
import torch.distributed as dist
from torch import nn


def get_local_size() -> int:
    """Processes per machine (the reference's default, with no local process group: the world size), 1 when
    torch.distributed is not initialised."""
    if not dist.is_available() or not dist.is_initialized():
        return 1
    return dist.get_world_size()


def _sync_args(bn, num_sync_devices, global_sync):
    bn.global_sync = global_sync
    if bn.global_sync and num_sync_devices is not None:
        raise ValueError(f"Cannot set num_sync_devices separately when global_sync = {bn.global_sync}")
    if not bn.global_sync and num_sync_devices is None:
        raise ValueError(f"num_sync_devices cannot be None when global_sync = {bn.global_sync}")
    if not bn.global_sync:
        bn.num_sync_devices = num_sync_devices
        if bn.num_sync_devices > 0:
            assert get_local_size() % bn.num_sync_devices == 0, (get_local_size(), bn.num_sync_devices)
            bn.num_groups = get_local_size() // bn.num_sync_devices
        else:
            bn.num_sync_devices = get_local_size()
            bn.num_groups = 1


def _no_forward(self, input):
    raise RuntimeError("%s has no forward of its own: it runs folded into the layer before it inside a model the "
                       "pytorchvideo_b200 engine lowers" % type(self).__name__)


class NaiveSyncBatchNorm1d(nn.BatchNorm1d):
    """1-D naive sync BatchNorm: ``num_sync_devices`` local devices to sync, or ``global_sync`` over all."""

    def __init__(self, num_sync_devices=None, global_sync=True, **args):
        _sync_args(self, num_sync_devices, global_sync)
        super(NaiveSyncBatchNorm1d, self).__init__(**args)

    forward = _no_forward


class NaiveSyncBatchNorm2d(nn.BatchNorm2d):
    """2-D naive sync BatchNorm (see NaiveSyncBatchNorm1d)."""

    def __init__(self, num_sync_devices=None, global_sync=True, **args):
        _sync_args(self, num_sync_devices, global_sync)
        super(NaiveSyncBatchNorm2d, self).__init__(**args)

    forward = _no_forward


class NaiveSyncBatchNorm3d(nn.BatchNorm3d):
    """3-D naive sync BatchNorm (see NaiveSyncBatchNorm1d)."""

    def __init__(self, num_sync_devices=None, global_sync=True, **args):
        _sync_args(self, num_sync_devices, global_sync)
        super(NaiveSyncBatchNorm3d, self).__init__(**args)

    forward = _no_forward
