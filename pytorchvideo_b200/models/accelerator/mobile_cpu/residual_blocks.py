"""X3D bottleneck of the mobile efficient blocks (reference models/accelerator/mobile_cpu/residual_blocks.py).

    out = final_act(res + conv_2(act_func_1(se(conv_1(conv_0(x)))))),  res = x, _res_proj(x) or nothing

The engine runs conv_0 as a pointwise convolution with BatchNorm and activation in its epilogue, conv_1 as the
depthwise kernel (with SE: it also produces the channel sums, and ``act_func_1`` is applied by the SE scale launch;
without SE: ``act_func_1`` is in its epilogue), and conv_2 with the residual add and ``final_act`` in its epilogue.
``convert`` keeps this tree and builds the block's plan (accelerator/no_op_convert_block.py ``MobileBlock``); the
reference's deployable form (Conv2d decompositions, ``_SkipConnectMul``, fused ``ConvReLU``) is not reproduced, and
``_residual_add_func`` is kept for the ``repr`` only."""
from collections import OrderedDict

import torch.nn as nn

from ....accelerator.no_op_convert_block import MobileBlock
from ....layers.accelerator.mobile_cpu.activation_functions import supported_act_functions
from ....layers.accelerator.mobile_cpu.attention import SqueezeExcitation
from ....layers.accelerator.mobile_cpu.convolutions import (Conv3d3x3x3DwBnAct, Conv3dPwBnAct,
                                                             Conv3dTemporalKernel1BnAct)
from ....layers.utils import round_width


class X3dBottleneckBlock(MobileBlock):
    _ALREADY_CONVERTED = "already converted, cannot be converted twice"

    def __init__(self, in_channels, mid_channels, out_channels, use_residual=True, spatial_stride=1, se_ratio=0.0625,
                 act_functions=("relu", "relu", "relu"), bias=(False, False, False), use_bn=(True, True, True),
                 norm_eps=1e-5, norm_momentum=0.1):
        super().__init__()
        self._use_residual = use_residual
        self._res_proj = None
        if use_residual:
            self._residual_add_func = nn.quantized.FloatFunctional()
            if spatial_stride != 1 or in_channels != out_channels:
                self._res_proj = Conv3dTemporalKernel1BnAct(in_channels, out_channels, bias=False, groups=1,
                                                            spatial_kernel=1, spatial_stride=spatial_stride,
                                                            spatial_padding=0, spatial_dilation=1,
                                                            activation="identity", use_bn=True)
        for a in act_functions:
            assert a in supported_act_functions, "%s is not supported." % a
        layers = OrderedDict()
        layers["conv_0"] = Conv3dPwBnAct(in_channels, mid_channels, bias=bias[0], activation=act_functions[0],
                                         use_bn=use_bn[0], norm_eps=norm_eps, norm_momentum=norm_momentum)
        self._spatial_stride = spatial_stride
        self._mid_channels = mid_channels
        layers["conv_1"] = Conv3d3x3x3DwBnAct(mid_channels, spatial_stride=spatial_stride, bias=bias[1],
                                              activation="identity", use_bn=use_bn[1], norm_eps=norm_eps,
                                              norm_momentum=norm_momentum)
        if se_ratio > 0:
            layers["se"] = SqueezeExcitation(num_channels=mid_channels,
                                             num_channels_reduced=round_width(mid_channels, se_ratio), is_3d=True)
        layers["act_func_1"] = supported_act_functions[act_functions[1]]()
        self._out_channels = out_channels
        layers["conv_2"] = Conv3dPwBnAct(mid_channels, out_channels, bias=bias[2], activation="identity",
                                         use_bn=use_bn[2], norm_eps=norm_eps, norm_momentum=norm_momentum)
        self.final_act = supported_act_functions[act_functions[2]]()
        self.layers = nn.Sequential(layers)
        self.convert_flag = False
