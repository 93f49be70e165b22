"""Squeeze-Excitation of the mobile efficient blocks (reference layers/accelerator/mobile_cpu/attention.py): this
package's 3-D SqueezeExcitation wrapped as ``.se``, so the keys are ``se.block.{0,2}.{weight,bias}``.  The engine runs it
as channel sums (fused into the producing depthwise convolution inside a block), the gate and one scale launch.
``convert`` keeps this tree: the reference's deployable form (Linear layers, ``_Reshape``, ``_SkipConnectMul``) is not
reproduced.  2-D SE is not supported."""
from ....accelerator.no_op_convert_block import MobileBlock
from ...squeeze_excitation import SqueezeExcitation as _SqueezeExcitation3d


class SqueezeExcitation(MobileBlock):
    def __init__(self, num_channels, num_channels_reduced=None, reduction_ratio=2.0, is_3d=False, activation=None):
        super().__init__()
        self.se = _SqueezeExcitation3d(num_channels, num_channels_reduced=num_channels_reduced,
                                       reduction_ratio=reduction_ratio, is_3d=is_3d, activation=activation)
        self.is_3d = is_3d
        self.convert_flag = False
