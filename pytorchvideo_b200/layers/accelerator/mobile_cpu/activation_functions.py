"""Activation functions of the mobile efficient blocks (reference layers/accelerator/mobile_cpu/activation_functions.py).

Each wrapper holds the activation as ``.act``, as the reference does, so ``state_dict`` keys and ``repr`` match.  Inside
a block the engine applies the activation in the producing kernel's epilogue; called on its own a wrapper is one
elementwise launch.  ``convert`` changes nothing: the reference's deployable swish (``_NaiveSwish``) computes the same
function."""
import torch.nn as nn

from ....accelerator.efficient_block_base import EfficientBlockBase
from ....module import B200Module
from ...swish import Swish as _SwishOp


class _Activation(B200Module, EfficientBlockBase):
    def convert(self, *args, **kwargs):
        pass


class Swish(_Activation):
    """x * sigmoid(x) (PV_ACT_SWISH)."""

    def __init__(self):
        super().__init__()
        self.act = _SwishOp()


class HardSwish(_Activation):
    """x * clamp(x + 3, 0, 6) / 6, torch.nn.Hardswish (PV_ACT_HSWISH)."""

    def __init__(self):
        super().__init__()
        self.act = nn.Hardswish()


class ReLU(_Activation):
    def __init__(self):
        super().__init__()
        self.act = nn.ReLU(inplace=True)


class Identity(_Activation):
    def __init__(self):
        super().__init__()
        self.act = nn.Identity()


supported_act_functions = {
    "relu": ReLU,
    "swish": Swish,
    "hswish": HardSwish,
    "identity": Identity,
}
