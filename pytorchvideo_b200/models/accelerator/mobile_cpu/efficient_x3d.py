"""X3D built from the mobile efficient blocks (reference models/accelerator/mobile_cpu/efficient_x3d.py).

The same network as ``models.x3d.create_x3d`` at the X3D-XS / S / M widths (L: deeper stages) in the reference's
efficient-block module tree, so its ``efficient_x3d_*_original_form`` checkpoints load with ``load_state_dict``.  The
forward runs on the engine like every module of this package: s1 is the X3D stem (a 1x3x3 convolution and the temporal
depthwise kernel), s2-s5 are ``X3dBottleneckBlock`` stages, and the head runs conv_5, the global average pool, lin_5
and the projection (with ``head_act`` in its epilogue) on the ProjectedPool / head-reduce launches.  Note that this
``create_x3d`` is not ``models.x3d.create_x3d``."""
from collections import OrderedDict

import torch.nn as nn

from ....layers.accelerator.mobile_cpu.activation_functions import supported_act_functions
from ....layers.accelerator.mobile_cpu.convolutions import (Conv3d5x1x1BnAct, Conv3dPwBnAct,
                                                             Conv3dTemporalKernel1BnAct)
from ....layers.accelerator.mobile_cpu.fully_connected import FullyConnected
from ....layers.accelerator.mobile_cpu.pool import AdaptiveAvgPool3dOutSize1
from ....module import B200Module
from .residual_blocks import X3dBottleneckBlock

# (stage, in channels, mid channels, out channels, depth, depth for "L")
_STAGES = (("s2", 24, 54, 24, 3, 5), ("s3", 24, 108, 48, 5, 10), ("s4", 48, 216, 96, 11, 25),
           ("s5", 96, 432, 192, 7, 15))


class EfficientX3d(B200Module):
    """Args: num_classes, dropout (training only), expansion ("XS", "S", "M" or "L"), head_act (a key of
    supported_act_functions), enable_head (False: the forward returns the s5 feature map)."""

    def __init__(self, num_classes=400, dropout=0.5, expansion="XS", head_act="identity", enable_head=True):
        super().__init__()
        assert expansion in ("XS", "S", "M", "L"), f"Expansion {expansion} not supported."
        s1 = OrderedDict()
        s1["pathway0_stem_conv_xy"] = Conv3dTemporalKernel1BnAct(3, 24, bias=False, groups=1, spatial_kernel=3,
                                                                 spatial_stride=2, spatial_padding=1,
                                                                 activation="identity", use_bn=False)
        s1["pathway0_stem_conv"] = Conv3d5x1x1BnAct(24, 24, bias=False, groups=24, use_bn=True)
        self.s1 = nn.Sequential(s1)
        for stage, c_in, c_mid, c_out, depth, depth_l in _STAGES:
            blocks = OrderedDict()
            for i in range(depth_l if expansion == "L" else depth):
                blocks[f"pathway0_res{i}"] = X3dBottleneckBlock(
                    in_channels=c_in if i == 0 else c_out, mid_channels=c_mid, out_channels=c_out, use_residual=True,
                    spatial_stride=2 if i == 0 else 1, se_ratio=0.0625 if i % 2 == 0 else 0,
                    act_functions=("relu", "swish", "relu"), use_bn=(True, True, True))
            setattr(self, stage, nn.Sequential(blocks))
        self.enable_head = enable_head
        if enable_head:
            head = OrderedDict()
            head["conv_5"] = Conv3dPwBnAct(in_channels=192, out_channels=432, bias=False, use_bn=True)
            head["avg_pool"] = AdaptiveAvgPool3dOutSize1()
            head["lin_5"] = Conv3dPwBnAct(in_channels=432, out_channels=2048, bias=False, use_bn=False)
            self.head = nn.Sequential(head)
            if dropout > 0:
                self.dropout = nn.Dropout(dropout)
            self.projection = FullyConnected(2048, num_classes, bias=True)
            assert head_act in supported_act_functions, f"{head_act} is not supported."
            self.act = supported_act_functions[head_act]()

    def forward(self, x):
        # Blocks replaced one by one by the accelerator protocol (transmute_model(model, "b200")) each own a plan: the
        # stages then run in sequence, handing NCDHW tensors on, and the head compiles into a plan of its own.  An
        # untouched model compiles into ONE plan.
        stages = (self.s1, self.s2, self.s3, self.s4, self.s5)
        if not any(type(b).__name__ == "B200Block" for s in stages for b in s):
            return super().forward(x)
        for s in stages:
            x = s(x)
        return super().forward(x, "head") if self.enable_head else x


def create_x3d(*, num_classes=400, dropout=0.5, expansion="XS", head_act="identity", enable_head=True):
    """X3D with efficient blocks (reference models/accelerator/mobile_cpu/efficient_x3d.py create_x3d)."""
    return EfficientX3d(num_classes=num_classes, dropout=dropout, expansion=expansion, head_act=head_act,
                        enable_head=enable_head)
