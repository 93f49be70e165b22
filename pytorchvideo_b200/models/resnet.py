"""ResNet-style blocks, stages and the Slow / C2D / I3D family builder
(reference models/resnet.py).  Module trees and state_dict keys match the reference so hub
checkpoints (``checkpoint["model_state"]``) load with strict=True."""
from typing import Callable

import numpy as np
import torch
import torch.nn as nn

from ..layers.utils import set_attributes
from ..module import B200Module
from .head import create_res_basic_head
from .net import Net
from .stem import create_acoustic_res_basic_stem, create_res_basic_stem

_MODEL_STAGE_DEPTH = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3), 152: (3, 8, 36, 3)}


class BottleneckBlock(B200Module):
    """conv_a/norm_a/act_a -> conv_b/norm_b/act_b -> conv_c/norm_c (resnet.py:1288-1365)."""

    def __init__(self, *, conv_a=None, norm_a=None, act_a=None, conv_b=None, norm_b=None, act_b=None,
                 conv_c=None, norm_c=None):
        super().__init__()
        set_attributes(self, locals())
        assert all(op is not None for op in (self.conv_a, self.conv_b, self.conv_c))
        if self.norm_c is not None:
            self.norm_c.block_final_bn = True   # read by init_net_weights


class SeparableBottleneckBlock(B200Module):
    """conv_a/norm_a/act_a -> parallel conv_b[i]/norm_b[i]/act_b[i] reduced by "sum" or "cat" -> conv_c/norm_c
    (resnet.py:1192-1285).  On device both conv_b branches run as one convolution over their union of taps."""

    def __init__(self, *, conv_a, norm_a, act_a, conv_b, norm_b, act_b, conv_c, norm_c, reduce_method="sum"):
        super().__init__()
        set_attributes(self, locals())
        assert all(op is not None for op in (self.conv_b, self.conv_c)), (
            f"{self.conv_a}, {self.conv_b}, {self.conv_c} has None")
        assert reduce_method in ["sum", "cat"]
        if self.norm_c is not None:
            self.norm_c.block_final_bn = True   # read by init_net_weights


class ResBlock(B200Module):
    """shortcut (identity | conv+norm) + branch2, then activation (resnet.py:1137-1189)."""

    def __init__(self, branch1_conv=None, branch1_norm=None, branch2=None, activation=None,
                 branch_fusion=None):
        super().__init__()
        set_attributes(self, locals())
        assert self.branch2 is not None


class ResStage(B200Module):
    def __init__(self, res_blocks):
        super().__init__()
        self.res_blocks = res_blocks


def _norm(norm, c, eps, momentum):
    return None if norm is None else norm(num_features=c, eps=eps, momentum=momentum)


def create_bottleneck_block(*, dim_in, dim_inner, dim_out, conv_a_kernel_size=(3, 1, 1),
                            conv_a_stride=(2, 1, 1), conv_a_padding=(1, 0, 0), conv_a=nn.Conv3d,
                            conv_b_kernel_size=(1, 3, 3), conv_b_stride=(1, 2, 2), conv_b_padding=(0, 1, 1),
                            conv_b_num_groups=1, conv_b_dilation=(1, 1, 1), conv_b=nn.Conv3d, conv_c=nn.Conv3d,
                            norm=nn.BatchNorm3d, norm_eps=1e-5, norm_momentum=0.1, activation=nn.ReLU):
    act = (lambda: None) if activation is None else activation
    return BottleneckBlock(
        conv_a=conv_a(in_channels=dim_in, out_channels=dim_inner, kernel_size=conv_a_kernel_size,
                      stride=conv_a_stride, padding=conv_a_padding, bias=False),
        norm_a=_norm(norm, dim_inner, norm_eps, norm_momentum),
        act_a=act(),
        conv_b=conv_b(in_channels=dim_inner, out_channels=dim_inner, kernel_size=conv_b_kernel_size,
                      stride=conv_b_stride, padding=conv_b_padding, bias=False, groups=conv_b_num_groups,
                      dilation=conv_b_dilation),
        norm_b=_norm(norm, dim_inner, norm_eps, norm_momentum),
        act_b=act(),
        conv_c=conv_c(in_channels=dim_inner, out_channels=dim_out, kernel_size=(1, 1, 1), bias=False),
        norm_c=_norm(norm, dim_out, norm_eps, norm_momentum),
    )


def create_acoustic_bottleneck_block(*, dim_in, dim_inner, dim_out, conv_a_kernel_size=(3, 1, 1),
                                     conv_a_stride=(2, 1, 1), conv_a_padding=(1, 0, 0), conv_a=nn.Conv3d,
                                     conv_b_kernel_size=(1, 1, 1), conv_b_stride=(1, 1, 1), conv_b_padding=(0, 0, 0),
                                     conv_b_num_groups=1, conv_b_dilation=(1, 1, 1), conv_b=nn.Conv3d,
                                     conv_c=nn.Conv3d, norm=nn.BatchNorm3d, norm_eps=1e-5, norm_momentum=0.1,
                                     activation=nn.ReLU):
    """Bottleneck whose conv_b is a (kt,1,1) temporal and a (1,kh,kw) spatial convolution in parallel, summed
    (resnet.py:151-316).  ``conv_b`` / ``norm_b`` / ``act_b`` hold the spatial branch first, the temporal second."""
    act = (lambda: None) if activation is None else activation
    branch_t = dict(kernel_size=[conv_b_kernel_size[0], 1, 1], padding=[conv_b_padding[0], 0, 0],
                    dilation=[conv_b_dilation[0], 1, 1])
    branch_s = dict(kernel_size=[1, conv_b_kernel_size[1], conv_b_kernel_size[2]],
                    padding=[0, conv_b_padding[1], conv_b_padding[2]],
                    dilation=[1, conv_b_dilation[1], conv_b_dilation[2]])
    conv_b_1, conv_b_2 = (conv_b(in_channels=dim_inner, out_channels=dim_inner, stride=conv_b_stride, bias=False,
                                 groups=conv_b_num_groups, **kw) for kw in (branch_t, branch_s))
    norm_b_1 = _norm(norm, dim_inner, norm_eps, norm_momentum)
    act_b_1 = act()
    norm_b_2 = _norm(norm, dim_inner, norm_eps, norm_momentum)
    act_b_2 = act()
    return SeparableBottleneckBlock(
        conv_a=conv_a(in_channels=dim_in, out_channels=dim_inner, kernel_size=conv_a_kernel_size,
                      stride=conv_a_stride, padding=conv_a_padding, bias=False),
        norm_a=_norm(norm, dim_inner, norm_eps, norm_momentum),
        act_a=act(),
        conv_b=nn.ModuleList([conv_b_2, conv_b_1]),
        norm_b=nn.ModuleList([norm_b_2, norm_b_1]),
        act_b=nn.ModuleList([act_b_2, act_b_1]),
        conv_c=conv_c(in_channels=dim_inner, out_channels=dim_out, kernel_size=(1, 1, 1), bias=False),
        norm_c=_norm(norm, dim_out, norm_eps, norm_momentum),
    )


def create_res_block(*, dim_in, dim_inner, dim_out, bottleneck, use_shortcut=False,
                     branch_fusion=lambda x, y: x + y, conv_a_kernel_size=(3, 1, 1), conv_a_stride=(2, 1, 1),
                     conv_a_padding=(1, 0, 0), conv_a=nn.Conv3d, conv_b_kernel_size=(1, 3, 3),
                     conv_b_stride=(1, 2, 2), conv_b_padding=(0, 1, 1), conv_b_num_groups=1,
                     conv_b_dilation=(1, 1, 1), conv_b=nn.Conv3d, conv_c=nn.Conv3d, conv_skip=nn.Conv3d,
                     norm=nn.BatchNorm3d, norm_eps=1e-5, norm_momentum=0.1, activation_bottleneck=nn.ReLU,
                     activation_block=nn.ReLU):
    skip_stride = tuple(a * b for a, b in zip(conv_a_stride, conv_b_stride))
    changes_shape = dim_in != dim_out or int(np.prod(skip_stride)) != 1
    needs_proj = changes_shape or use_shortcut
    skip_norm = None
    if use_shortcut or (norm is not None and changes_shape):
        skip_norm = norm(num_features=dim_out, eps=norm_eps, momentum=norm_momentum)
    return ResBlock(
        branch1_conv=conv_skip(dim_in, dim_out, kernel_size=(1, 1, 1), stride=skip_stride, bias=False)
        if needs_proj else None,
        branch1_norm=skip_norm,
        branch2=bottleneck(dim_in=dim_in, dim_inner=dim_inner, dim_out=dim_out,
                           conv_a_kernel_size=conv_a_kernel_size, conv_a_stride=conv_a_stride,
                           conv_a_padding=conv_a_padding, conv_a=conv_a, conv_b_kernel_size=conv_b_kernel_size,
                           conv_b_stride=conv_b_stride, conv_b_padding=conv_b_padding,
                           conv_b_num_groups=conv_b_num_groups, conv_b_dilation=conv_b_dilation, conv_b=conv_b,
                           conv_c=conv_c, norm=norm, norm_eps=norm_eps, norm_momentum=norm_momentum,
                           activation=activation_bottleneck),
        activation=None if activation_block is None else activation_block(),
        branch_fusion=branch_fusion,
    )


def create_res_stage(*, depth, dim_in, dim_inner, dim_out, bottleneck, conv_a_kernel_size=(3, 1, 1),
                     conv_a_stride=(2, 1, 1), conv_a_padding=(1, 0, 0), conv_a=nn.Conv3d,
                     conv_b_kernel_size=(1, 3, 3), conv_b_stride=(1, 2, 2), conv_b_padding=(0, 1, 1),
                     conv_b_num_groups=1, conv_b_dilation=(1, 1, 1), conv_b=nn.Conv3d, conv_c=nn.Conv3d,
                     norm=nn.BatchNorm3d, norm_eps=1e-5, norm_momentum=0.1, activation=nn.ReLU):
    # a single kernel spec is cycled over the blocks of the stage
    a_kernels = [conv_a_kernel_size] if isinstance(conv_a_kernel_size[0], int) else list(conv_a_kernel_size)
    a_pads = [conv_a_padding] if isinstance(conv_a_padding[0], int) else list(conv_a_padding)
    blocks = []
    for i in range(depth):
        first = i == 0
        blocks.append(create_res_block(
            dim_in=dim_in if first else dim_out, dim_inner=dim_inner, dim_out=dim_out, bottleneck=bottleneck,
            conv_a_kernel_size=a_kernels[i % len(a_kernels)],
            conv_a_stride=conv_a_stride if first else (1, 1, 1),
            conv_a_padding=a_pads[i % len(a_pads)], conv_a=conv_a, conv_b_kernel_size=conv_b_kernel_size,
            conv_b_stride=conv_b_stride if first else (1, 1, 1), conv_b_padding=conv_b_padding,
            conv_b_num_groups=conv_b_num_groups, conv_b_dilation=conv_b_dilation, conv_b=conv_b, conv_c=conv_c,
            norm=norm, norm_eps=norm_eps, norm_momentum=norm_momentum, activation_bottleneck=activation,
            activation_block=activation))
    return ResStage(res_blocks=nn.ModuleList(blocks))


def _half_kernel_padding(kernel):
    if isinstance(kernel[0], int):
        return [k // 2 for k in kernel]
    return [[k // 2 for k in ks] for ks in kernel]


def _conv_b_padding(kernel, dilation):
    return (kernel[0] // 2,
            dilation[1] if dilation[1] > 1 else kernel[1] // 2,
            dilation[2] if dilation[2] > 1 else kernel[2] // 2)


def create_resnet(*, input_channel=3, model_depth=50, model_num_class=400, dropout_rate=0.5,
                  norm=nn.BatchNorm3d, activation=nn.ReLU, stem_dim_out=64, stem_conv_kernel_size=(3, 7, 7),
                  stem_conv_stride=(1, 2, 2), stem_pool=nn.MaxPool3d, stem_pool_kernel_size=(1, 3, 3),
                  stem_pool_stride=(1, 2, 2), stem=create_res_basic_stem, stage1_pool=None,
                  stage1_pool_kernel_size=(2, 1, 1),
                  stage_conv_a_kernel_size=((1, 1, 1), (1, 1, 1), (3, 1, 1), (3, 1, 1)),
                  stage_conv_b_kernel_size=((1, 3, 3), (1, 3, 3), (1, 3, 3), (1, 3, 3)),
                  stage_conv_b_num_groups=(1, 1, 1, 1),
                  stage_conv_b_dilation=((1, 1, 1), (1, 1, 1), (1, 1, 1), (1, 1, 1)),
                  stage_spatial_h_stride=(1, 2, 2, 2), stage_spatial_w_stride=(1, 2, 2, 2),
                  stage_temporal_stride=(1, 1, 1, 1), bottleneck=create_bottleneck_block,
                  head=create_res_basic_head, head_pool=nn.AvgPool3d, head_pool_kernel_size=(4, 7, 7),
                  head_output_size=(1, 1, 1), head_activation=None, head_output_with_global_average=True):
    """Slow / C2D / I3D-style 3-D ResNet (reference resnet.py:601-827)."""
    torch._C._log_api_usage_once("PYTORCHVIDEO.model.create_resnet")
    assert model_depth in _MODEL_STAGE_DEPTH, f"{model_depth} is not in {_MODEL_STAGE_DEPTH.keys()}"
    depths = _MODEL_STAGE_DEPTH[model_depth]
    n_stage = len(depths)
    if isinstance(stage_conv_a_kernel_size[0], int):
        stage_conv_a_kernel_size = (stage_conv_a_kernel_size,) * n_stage
    if isinstance(stage_conv_b_kernel_size[0], int):
        stage_conv_b_kernel_size = (stage_conv_b_kernel_size,) * n_stage
    if isinstance(stage_conv_b_dilation[0], int):
        stage_conv_b_dilation = (stage_conv_b_dilation,) * n_stage
    if isinstance(bottleneck, Callable):
        bottleneck = [bottleneck] * n_stage

    blocks = [stem(in_channels=input_channel, out_channels=stem_dim_out, conv_kernel_size=stem_conv_kernel_size,
                   conv_stride=stem_conv_stride, conv_padding=[k // 2 for k in stem_conv_kernel_size],
                   pool=stem_pool, pool_kernel_size=stem_pool_kernel_size, pool_stride=stem_pool_stride,
                   pool_padding=[k // 2 for k in stem_pool_kernel_size], norm=norm, activation=activation)]
    width_in, width_out = stem_dim_out, stem_dim_out * 4
    for s in range(n_stage):
        a_kernel = stage_conv_a_kernel_size[s]
        blocks.append(create_res_stage(
            depth=depths[s], dim_in=width_in, dim_inner=width_out // 4, dim_out=width_out,
            bottleneck=bottleneck[s], conv_a_kernel_size=a_kernel,
            conv_a_stride=(stage_temporal_stride[s], 1, 1), conv_a_padding=_half_kernel_padding(a_kernel),
            conv_b_kernel_size=stage_conv_b_kernel_size[s],
            conv_b_stride=(1, stage_spatial_h_stride[s], stage_spatial_w_stride[s]),
            conv_b_padding=_conv_b_padding(stage_conv_b_kernel_size[s], stage_conv_b_dilation[s]),
            conv_b_num_groups=stage_conv_b_num_groups[s], conv_b_dilation=stage_conv_b_dilation[s],
            norm=norm, activation=activation))
        width_in, width_out = width_out, width_out * 2
        if s == 0 and stage1_pool is not None:
            blocks.append(stage1_pool(kernel_size=stage1_pool_kernel_size, stride=stage1_pool_kernel_size,
                                      padding=(0, 0, 0)))
    if head is not None:
        blocks.append(head(in_features=width_in, out_features=model_num_class, pool=head_pool,
                           output_size=head_output_size, pool_kernel_size=head_pool_kernel_size,
                           dropout_rate=dropout_rate, activation=head_activation,
                           output_with_global_average=head_output_with_global_average))
    return Net(blocks=nn.ModuleList(blocks))


def create_acoustic_resnet(*, input_channel=1, model_depth=50, model_num_class=400, dropout_rate=0.5,
                           norm=nn.BatchNorm3d, activation=nn.ReLU, stem_dim_out=64, stem_conv_kernel_size=(9, 1, 9),
                           stem_conv_stride=(1, 1, 3), stem_pool=None, stem_pool_kernel_size=(3, 1, 3),
                           stem_pool_stride=(2, 1, 2), stem=create_acoustic_res_basic_stem, stage1_pool=None,
                           stage1_pool_kernel_size=(2, 1, 1), stage_conv_a_kernel_size=(3, 1, 1),
                           stage_conv_b_kernel_size=(3, 1, 3), stage_conv_b_num_groups=(1, 1, 1, 1),
                           stage_conv_b_dilation=(1, 1, 1), stage_spatial_h_stride=(1, 1, 1, 1),
                           stage_spatial_w_stride=(1, 2, 2, 2), stage_temporal_stride=(1, 2, 2, 2),
                           bottleneck=(create_acoustic_bottleneck_block, create_acoustic_bottleneck_block,
                                       create_bottleneck_block, create_bottleneck_block),
                           head_pool=nn.AvgPool3d, head_pool_kernel_size=(4, 1, 2),
                           head_output_size=(1, 1, 1), head_activation=None, head_output_with_global_average=True):
    """ResNet over a log-mel spectrogram (B, C, T, 1, F) (reference resnet.py:1022-1134)."""
    return create_resnet(**locals())


def create_resnet_with_roi_head(*, input_channel=3, model_depth=50, model_num_class=80, dropout_rate=0.5,
                                norm=nn.BatchNorm3d, activation=nn.ReLU, stem_dim_out=64,
                                stem_conv_kernel_size=(1, 7, 7), stem_conv_stride=(1, 2, 2), stem_pool=nn.MaxPool3d,
                                stem_pool_kernel_size=(1, 3, 3), stem_pool_stride=(1, 2, 2),
                                stem=create_res_basic_stem, stage1_pool=None, stage1_pool_kernel_size=(2, 1, 1),
                                stage_conv_a_kernel_size=((1, 1, 1), (1, 1, 1), (3, 1, 1), (3, 1, 1)),
                                stage_conv_b_kernel_size=((1, 3, 3), (1, 3, 3), (1, 3, 3), (1, 3, 3)),
                                stage_conv_b_num_groups=(1, 1, 1, 1),
                                stage_conv_b_dilation=((1, 1, 1), (1, 1, 1), (1, 1, 1), (1, 2, 2)),
                                stage_spatial_h_stride=(1, 2, 2, 1), stage_spatial_w_stride=(1, 2, 2, 1),
                                stage_temporal_stride=(1, 1, 1, 1), bottleneck=create_bottleneck_block,
                                head=None, head_pool=nn.AvgPool3d, head_pool_kernel_size=(4, 1, 1),
                                head_output_size=(1, 1, 1), head_activation=nn.Sigmoid,
                                head_output_with_global_average=False, head_spatial_resolution=(7, 7),
                                head_spatial_scale=1.0 / 16.0, head_sampling_ratio=0):
    """Slow-only detection network: ResNet trunk without head + RoI head (reference resnet.py:844-1017)."""
    from .head import create_res_roi_pooling_head
    from .net import DetectionBBoxNetwork
    if head is None:
        head = create_res_roi_pooling_head
    model = create_resnet(
        input_channel=input_channel, model_depth=model_depth, model_num_class=model_num_class,
        dropout_rate=dropout_rate, norm=norm, activation=activation, stem_dim_out=stem_dim_out,
        stem_conv_kernel_size=stem_conv_kernel_size, stem_conv_stride=stem_conv_stride, stem_pool=stem_pool,
        stem_pool_kernel_size=stem_pool_kernel_size, stem_pool_stride=stem_pool_stride, stem=stem,
        stage1_pool=stage1_pool, stage1_pool_kernel_size=stage1_pool_kernel_size,
        stage_conv_a_kernel_size=stage_conv_a_kernel_size, stage_conv_b_kernel_size=stage_conv_b_kernel_size,
        stage_conv_b_num_groups=stage_conv_b_num_groups, stage_conv_b_dilation=stage_conv_b_dilation,
        stage_spatial_h_stride=stage_spatial_h_stride, stage_spatial_w_stride=stage_spatial_w_stride,
        stage_temporal_stride=stage_temporal_stride, bottleneck=bottleneck, head=None)
    det_head = head(
        in_features=stem_dim_out * 2 ** (len(_MODEL_STAGE_DEPTH[model_depth]) + 1), out_features=model_num_class,
        pool=head_pool, output_size=head_output_size, pool_kernel_size=head_pool_kernel_size,
        dropout_rate=dropout_rate, activation=head_activation,
        output_with_global_average=head_output_with_global_average, resolution=head_spatial_resolution,
        spatial_scale=head_spatial_scale, sampling_ratio=head_sampling_ratio)
    return DetectionBBoxNetwork(model, det_head)
