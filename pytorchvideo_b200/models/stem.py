"""Stems (reference models/stem.py)."""
import torch.nn as nn

from ..layers.utils import set_attributes
from ..module import B200Module


class ResNetBasicStem(B200Module):
    """conv -> norm -> activation -> pool (stem.py:215-260)."""

    def __init__(self, *, conv=None, norm=None, activation=None, pool=None):
        super().__init__()
        set_attributes(self, locals())
        assert self.conv is not None


def create_res_basic_stem(*, in_channels, out_channels, conv_kernel_size=(3, 7, 7), conv_stride=(1, 2, 2),
                          conv_padding=(1, 3, 3), conv_bias=False, conv=nn.Conv3d, pool=nn.MaxPool3d,
                          pool_kernel_size=(1, 3, 3), pool_stride=(1, 2, 2), pool_padding=(0, 1, 1),
                          norm=nn.BatchNorm3d, norm_eps=1e-5, norm_momentum=0.1, activation=nn.ReLU):
    return ResNetBasicStem(
        conv=conv(in_channels=in_channels, out_channels=out_channels, kernel_size=conv_kernel_size,
                  stride=conv_stride, padding=conv_padding, bias=conv_bias),
        norm=None if norm is None else norm(num_features=out_channels, eps=norm_eps, momentum=norm_momentum),
        activation=None if activation is None else activation(),
        pool=None if pool is None else pool(kernel_size=pool_kernel_size, stride=pool_stride,
                                            padding=pool_padding),
    )


def create_acoustic_res_basic_stem(*, in_channels, out_channels, conv_kernel_size=(3, 7, 7), conv_stride=(1, 1, 1),
                                   conv_padding=(1, 3, 3), conv_bias=False, pool=nn.MaxPool3d,
                                   pool_kernel_size=(1, 3, 3), pool_stride=(1, 2, 2), pool_padding=(0, 1, 1),
                                   norm=nn.BatchNorm3d, norm_eps=1e-5, norm_momentum=0.1, activation=nn.ReLU):
    """Stem whose conv is a (kt,1,1) temporal and a (1,kh,kw) spatial convolution, summed (stem.py:110-212).
    On device the two branches run as one (kt,kh,kw) convolution."""
    from ..layers.convolutions import ConvReduce3D
    return ResNetBasicStem(
        conv=ConvReduce3D(in_channels=in_channels, out_channels=out_channels,
                          kernel_size=((conv_kernel_size[0], 1, 1), (1, conv_kernel_size[1], conv_kernel_size[2])),
                          stride=(conv_stride, conv_stride),
                          padding=((conv_padding[0], 0, 0), (0, conv_padding[1], conv_padding[2])),
                          bias=(conv_bias, conv_bias), reduction_method="sum"),
        norm=None if norm is None else norm(num_features=out_channels, eps=norm_eps, momentum=norm_momentum),
        activation=None if activation is None else activation(),
        pool=None if pool is None else pool(kernel_size=pool_kernel_size, stride=pool_stride, padding=pool_padding),
    )


class PatchEmbed(B200Module):
    """Patchifying conv; on device its NDHWC output already IS the (B, THW, C) token layout, so the
    reference's flatten(2).transpose(1, 2) (stem.py:289-292) costs nothing."""

    def __init__(self, *, patch_model=None):
        super().__init__()
        set_attributes(self, locals())
        assert self.patch_model is not None


def create_conv_patch_embed(*, in_channels, out_channels, conv_kernel_size=(1, 16, 16), conv_stride=(1, 4, 4),
                            conv_padding=(1, 7, 7), conv_bias=True, conv=nn.Conv3d):
    return PatchEmbed(patch_model=conv(in_channels=in_channels, out_channels=out_channels,
                                       kernel_size=conv_kernel_size, stride=conv_stride, padding=conv_padding,
                                       bias=conv_bias))
