"""Convolution blocks of the mobile efficient blocks (reference layers/accelerator/mobile_cpu/convolutions.py):
``kernel = Sequential(conv, [bn], act)``.  The engine runs each as one convolution launch with BatchNorm folded and the
activation in its epilogue (engine/lower.py ``mobile_conv``).  ``convert`` keeps this tree: the reference's Conv2d
decompositions of the deployable form (``_Conv3dTemporalKernel*Decomposed``, ``_Reshape``, the fused ``ConvReLU``) are
not reproduced (accelerator/no_op_convert_block.py ``MobileBlock``)."""
from collections import OrderedDict

import torch.nn as nn

from ....accelerator.no_op_convert_block import MobileBlock
from .activation_functions import supported_act_functions


def _kernel(block, conv, out_channels, activation, use_bn, norm_eps, norm_momentum):
    k = OrderedDict()
    k["conv"] = conv
    if use_bn:
        k["bn"] = nn.BatchNorm3d(out_channels, eps=norm_eps, momentum=norm_momentum)
    assert activation in supported_act_functions, \
        "%s: %s is not in supported_act_functions." % (type(block).__name__, activation)
    k["act"] = supported_act_functions[activation]()
    return nn.Sequential(k)


class Conv3dPwBnAct(MobileBlock):
    """1x1x1 convolution + optional BatchNorm + activation."""

    def __init__(self, in_channels, out_channels, bias=False, activation="relu", use_bn=True, norm_eps=1e-5,
                 norm_momentum=0.1):
        super().__init__()
        self._in_channels = in_channels
        self._out_channels = out_channels
        self.act = activation
        self.kernel = _kernel(self, nn.Conv3d(in_channels, out_channels, kernel_size=1, bias=bias), out_channels,
                              activation, use_bn, norm_eps, norm_momentum)
        self.convert_flag = False


class Conv3d3x3x3DwBnAct(MobileBlock):
    """Depthwise 3x3x3 convolution, padding 1, stride (1, s, s) + optional BatchNorm + activation."""

    _ALREADY_CONVERTED = "already converted, cannot be converted twice."

    def __init__(self, in_channels, spatial_stride=1, bias=False, activation="relu", use_bn=True, norm_eps=1e-5,
                 norm_momentum=0.1):
        super().__init__()
        conv = nn.Conv3d(in_channels, in_channels, kernel_size=(3, 3, 3), stride=(1, spatial_stride, spatial_stride),
                         groups=in_channels, padding=1, bias=bias)
        self.kernel = _kernel(self, conv, in_channels, activation, use_bn, norm_eps, norm_momentum)
        self.convert_flag = False


class Conv3dTemporalKernel1BnAct(MobileBlock):
    """(1, k, k) convolution, temporal stride 1 and padding 0 + optional BatchNorm + activation."""

    def __init__(self, in_channels, out_channels, bias=False, groups=1, spatial_kernel=1, spatial_stride=1,
                 spatial_padding=0, spatial_dilation=1, activation="relu", use_bn=True, norm_eps=1e-5,
                 norm_momentum=0.1):
        super().__init__()
        conv = nn.Conv3d(in_channels, out_channels, kernel_size=(1, spatial_kernel, spatial_kernel),
                         padding=(0, spatial_padding, spatial_padding), stride=(1, spatial_stride, spatial_stride),
                         dilation=(1, spatial_dilation, spatial_dilation), groups=groups, bias=bias)
        self.kernel = _kernel(self, conv, out_channels, activation, use_bn, norm_eps, norm_momentum)
        self.convert_flag = False


class Conv3d3x1x1BnAct(MobileBlock):
    """(3, 1, 1) convolution, padding (1, 0, 0) + optional BatchNorm + activation."""

    _ALREADY_CONVERTED = "already converted, cannot be converted twice"

    def __init__(self, in_channels, out_channels, groups=1, bias=False, activation="relu", use_bn=True, norm_eps=1e-5,
                 norm_momentum=0.1):
        super().__init__()
        conv = nn.Conv3d(in_channels, out_channels, kernel_size=(3, 1, 1), groups=groups, padding=(1, 0, 0), bias=bias)
        self.kernel = _kernel(self, conv, out_channels, activation, use_bn, norm_eps, norm_momentum)
        self.convert_flag = False


class Conv3d5x1x1BnAct(MobileBlock):
    """(5, 1, 1) convolution, padding (2, 0, 0) + optional BatchNorm + activation.  Depthwise (groups = channels) it
    runs on the temporal depthwise kernel (the X3D stem's temporal convolution)."""

    _ALREADY_CONVERTED = "already converted, cannot be converted twice"

    def __init__(self, in_channels, out_channels, groups=1, bias=False, activation="relu", use_bn=True, norm_eps=1e-5,
                 norm_momentum=0.1):
        super().__init__()
        conv = nn.Conv3d(in_channels, out_channels, kernel_size=(5, 1, 1), groups=groups, padding=(2, 0, 0), bias=bias)
        self.kernel = _kernel(self, conv, out_channels, activation, use_bn, norm_eps, norm_momentum)
        self.convert_flag = False
