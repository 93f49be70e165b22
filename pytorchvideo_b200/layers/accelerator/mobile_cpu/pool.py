"""Pools of the mobile efficient blocks (reference layers/accelerator/mobile_cpu/pool.py).  The 3-D pools run on the
engine's pool kernel; ``AdaptiveAvgPool3dOutSize1.convert`` keeps ``nn.AdaptiveAvgPool3d(1)`` (the engine already pools
over the whole grid with a constant kernel).  The 2-D pools exist for the module trees only: lowering them raises
NotImplementedError."""
import torch.nn as nn

from ....accelerator.no_op_convert_block import MobileBlock, NoOpConvertBlock


class AdaptiveAvgPool3dOutSize1(MobileBlock):
    def __init__(self):
        super().__init__()
        self.pool = nn.AdaptiveAvgPool3d(1)
        self.convert_flag = False


class AdaptiveAvgPool2dOutSize1(MobileBlock):
    def __init__(self):
        super().__init__()
        self.pool = nn.AdaptiveAvgPool2d(1)
        self.convert_flag = False


class AdaptiveAvgPool3d(NoOpConvertBlock):
    """AdaptiveAvgPool3d(output_size); the engine takes output size 1 only."""

    def __init__(self, output_size):
        super().__init__(model=nn.AdaptiveAvgPool3d(output_size))


class AdaptiveAvgPool2d(NoOpConvertBlock):
    def __init__(self, output_size):
        super().__init__(model=nn.AdaptiveAvgPool2d(output_size))
