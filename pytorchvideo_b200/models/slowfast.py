"""SlowFast (reference models/slowfast.py): two ResNet pathways with lateral Fast->Slow fusion."""
from typing import Callable

import torch
import torch.nn as nn

from ..layers.utils import set_attributes
from ..module import B200Module
from .head import create_res_basic_head
from .net import MultiPathWayWithFuse, Net
from .resnet import _MODEL_STAGE_DEPTH, _conv_b_padding, _half_kernel_padding, create_bottleneck_block, \
    create_res_stage
from .stem import create_res_basic_stem


class PoolConcatPathway(B200Module):
    """Pool every pathway, then concatenate along channels (slowfast.py:585-620)."""

    def __init__(self, retain_list=False, pool=None, dim=1):
        super().__init__()
        set_attributes(self, locals())


class FuseFastToSlow(B200Module):
    """Time-strided conv on the Fast pathway, concatenated onto the Slow one (slowfast.py:697-729).
    On device the concat is free: the conv writes into the Slow tensor's channel slice."""

    def __init__(self, conv_fast_to_slow, norm=None, activation=None):
        super().__init__()
        set_attributes(self, locals())


class FastToSlowFusionBuilder:
    def __init__(self, slowfast_channel_reduction_ratio, conv_fusion_channel_ratio, conv_kernel_size,
                 conv_stride, norm=nn.BatchNorm3d, norm_eps=1e-5, norm_momentum=0.1, activation=nn.ReLU,
                 max_stage_idx=3):
        set_attributes(self, locals())

    def create_module(self, fusion_dim_in, stage_idx):
        if stage_idx > self.max_stage_idx:
            return nn.Identity()
        c_fast = fusion_dim_in // self.slowfast_channel_reduction_ratio
        c_fuse = int(c_fast * self.conv_fusion_channel_ratio)
        return FuseFastToSlow(
            conv_fast_to_slow=nn.Conv3d(c_fast, c_fuse, kernel_size=self.conv_kernel_size,
                                        stride=self.conv_stride,
                                        padding=[k // 2 for k in self.conv_kernel_size], bias=False),
            norm=None if self.norm is None else self.norm(
                num_features=c_fast * self.conv_fusion_channel_ratio, eps=self.norm_eps,
                momentum=self.norm_momentum),
            activation=None if self.activation is None else self.activation(),
        )


_BB = create_bottleneck_block
# slowfast.py:14-19: SlowFast also builds at depth 18 (create_resnet does not)
_SLOWFAST_STAGE_DEPTH = {18: (1, 1, 1, 1), **_MODEL_STAGE_DEPTH}


def create_slowfast(*, slowfast_channel_reduction_ratio=(8,), slowfast_conv_channel_fusion_ratio=2,
                    slowfast_fusion_conv_kernel_size=(7, 1, 1), slowfast_fusion_conv_stride=(4, 1, 1),
                    fusion_builder=None, input_channels=(3, 3), model_depth=50, model_num_class=400,
                    dropout_rate=0.5, norm=nn.BatchNorm3d, activation=nn.ReLU,
                    stem_function=(create_res_basic_stem, create_res_basic_stem), stem_dim_outs=(64, 8),
                    stem_conv_kernel_sizes=((1, 7, 7), (5, 7, 7)), stem_conv_strides=((1, 2, 2), (1, 2, 2)),
                    stem_pool=(nn.MaxPool3d, nn.MaxPool3d), stem_pool_kernel_sizes=((1, 3, 3), (1, 3, 3)),
                    stem_pool_strides=((1, 2, 2), (1, 2, 2)),
                    stage_conv_a_kernel_sizes=(((1, 1, 1), (1, 1, 1), (3, 1, 1), (3, 1, 1)),
                                               ((3, 1, 1), (3, 1, 1), (3, 1, 1), (3, 1, 1))),
                    stage_conv_b_kernel_sizes=(((1, 3, 3),) * 4, ((1, 3, 3),) * 4),
                    stage_conv_b_num_groups=((1, 1, 1, 1), (1, 1, 1, 1)),
                    stage_conv_b_dilations=(((1, 1, 1),) * 4, ((1, 1, 1),) * 4),
                    stage_spatial_strides=((1, 2, 2, 2), (1, 2, 2, 2)),
                    stage_temporal_strides=((1, 1, 1, 1), (1, 1, 1, 1)),
                    bottleneck=((_BB, _BB, _BB, _BB), (_BB, _BB, _BB, _BB)), head=create_res_basic_head,
                    head_pool=nn.AvgPool3d, head_pool_kernel_sizes=((8, 7, 7), (32, 7, 7)),
                    head_output_size=(1, 1, 1), head_activation=None, head_output_with_global_average=True):
    """SlowFast network builder (reference slowfast.py:22-361); input is ``[slow_clip, fast_clip]``."""
    torch._C._log_api_usage_once("PYTORCHVIDEO.model.create_slowfast")
    n_path = len(input_channels)
    assert model_depth in _SLOWFAST_STAGE_DEPTH, f"{model_depth} is not in {_SLOWFAST_STAGE_DEPTH.keys()}"
    depths = _SLOWFAST_STAGE_DEPTH[model_depth]
    if isinstance(slowfast_channel_reduction_ratio, int):
        slowfast_channel_reduction_ratio = (slowfast_channel_reduction_ratio,)
    if isinstance(stem_pool, Callable):
        stem_pool = (stem_pool,) * n_path
    if isinstance(bottleneck, Callable):
        bottleneck = ((bottleneck,) * len(depths),) * n_path
    if fusion_builder is None:
        fusion_builder = FastToSlowFusionBuilder(
            slowfast_channel_reduction_ratio=slowfast_channel_reduction_ratio[0],
            conv_fusion_channel_ratio=slowfast_conv_channel_fusion_ratio,
            conv_kernel_size=slowfast_fusion_conv_kernel_size, conv_stride=slowfast_fusion_conv_stride,
            norm=norm, activation=activation, max_stage_idx=len(depths) - 1).create_module

    stems = [stem_function[p](in_channels=input_channels[p], out_channels=stem_dim_outs[p],
                              conv_kernel_size=stem_conv_kernel_sizes[p], conv_stride=stem_conv_strides[p],
                              conv_padding=[k // 2 for k in stem_conv_kernel_sizes[p]], pool=stem_pool[p],
                              pool_kernel_size=stem_pool_kernel_sizes[p], pool_stride=stem_pool_strides[p],
                              pool_padding=[k // 2 for k in stem_pool_kernel_sizes[p]], norm=norm,
                              activation=activation) for p in range(n_path)]
    stages = [MultiPathWayWithFuse(multipathway_blocks=nn.ModuleList(stems),
                                   multipathway_fusion=fusion_builder(fusion_dim_in=stem_dim_outs[0], stage_idx=0))]

    width_in, width_out = stem_dim_outs[0], stem_dim_outs[0] * 4
    ratio0 = slowfast_channel_reduction_ratio[0]
    for s in range(len(depths)):
        # Slow pathway input carries the fused lateral channels
        dims_in = [width_in + width_in * slowfast_conv_channel_fusion_ratio // ratio0]
        dims_inner = [width_out // 4]
        dims_out = [width_out]
        for r in slowfast_channel_reduction_ratio:
            dims_in.append(width_in // r)
            dims_inner.append(width_out // 4 // r)
            dims_out.append(width_out // r)
        paths = []
        for p in range(n_path):
            a_kernel = stage_conv_a_kernel_sizes[p][s]
            b_kernel = stage_conv_b_kernel_sizes[p][s]
            sp = stage_spatial_strides[p][s]
            paths.append(create_res_stage(
                depth=depths[s], dim_in=dims_in[p], dim_inner=dims_inner[p], dim_out=dims_out[p],
                bottleneck=bottleneck[p][s], conv_a_kernel_size=a_kernel,
                conv_a_stride=(stage_temporal_strides[p][s], 1, 1), conv_a_padding=_half_kernel_padding(a_kernel),
                conv_b_kernel_size=b_kernel, conv_b_stride=(1, sp, sp),
                conv_b_padding=_conv_b_padding(b_kernel, stage_conv_b_dilations[p][s]),
                conv_b_num_groups=stage_conv_b_num_groups[p][s], conv_b_dilation=stage_conv_b_dilations[p][s],
                norm=norm, activation=activation))
        stages.append(MultiPathWayWithFuse(multipathway_blocks=nn.ModuleList(paths),
                                           multipathway_fusion=fusion_builder(fusion_dim_in=width_out,
                                                                              stage_idx=s + 1)))
        width_in, width_out = width_out, width_out * 2

    if head_pool is None:
        pools = None
    elif head_pool == nn.AdaptiveAvgPool3d:
        pools = [head_pool(head_output_size[p]) for p in range(n_path)]
    elif head_pool == nn.AvgPool3d:
        pools = [head_pool(kernel_size=head_pool_kernel_sizes[p], stride=(1, 1, 1), padding=(0, 0, 0))
                 for p in range(n_path)]
    else:
        raise NotImplementedError(f"Unsupported pool_model type {head_pool}")
    stages.append(PoolConcatPathway(retain_list=False, pool=None if pools is None else nn.ModuleList(pools)))
    feat = width_in + sum(width_in // r for r in slowfast_channel_reduction_ratio)
    if head is not None:
        stages.append(head(in_features=feat, out_features=model_num_class, pool=None,
                           output_size=head_output_size, dropout_rate=dropout_rate, activation=head_activation,
                           output_with_global_average=head_output_with_global_average))
    return Net(blocks=nn.ModuleList(stages))


def create_slowfast_with_roi_head(*, slowfast_channel_reduction_ratio=(8,), slowfast_conv_channel_fusion_ratio=2,
                                  slowfast_fusion_conv_kernel_size=(7, 1, 1), slowfast_fusion_conv_stride=(4, 1, 1),
                                  fusion_builder=None, input_channels=(3, 3), model_depth=50, model_num_class=80,
                                  dropout_rate=0.5, norm=nn.BatchNorm3d, activation=nn.ReLU,
                                  stem_function=(create_res_basic_stem, create_res_basic_stem), stem_dim_outs=(64, 8),
                                  stem_conv_kernel_sizes=((1, 7, 7), (5, 7, 7)),
                                  stem_conv_strides=((1, 2, 2), (1, 2, 2)), stem_pool=(nn.MaxPool3d, nn.MaxPool3d),
                                  stem_pool_kernel_sizes=((1, 3, 3), (1, 3, 3)),
                                  stem_pool_strides=((1, 2, 2), (1, 2, 2)),
                                  stage_conv_a_kernel_sizes=(((1, 1, 1), (1, 1, 1), (3, 1, 1), (3, 1, 1)),
                                                             ((3, 1, 1), (3, 1, 1), (3, 1, 1), (3, 1, 1))),
                                  stage_conv_b_kernel_sizes=(((1, 3, 3),) * 4, ((1, 3, 3),) * 4),
                                  stage_conv_b_num_groups=((1, 1, 1, 1), (1, 1, 1, 1)),
                                  stage_conv_b_dilations=(((1, 1, 1), (1, 1, 1), (1, 1, 1), (1, 2, 2)),
                                                          ((1, 1, 1), (1, 1, 1), (1, 1, 1), (1, 2, 2))),
                                  stage_spatial_strides=((1, 2, 2, 1), (1, 2, 2, 1)),
                                  stage_temporal_strides=((1, 1, 1, 1), (1, 1, 1, 1)),
                                  bottleneck=((_BB, _BB, _BB, _BB), (_BB, _BB, _BB, _BB)), head=None,
                                  head_pool=nn.AvgPool3d, head_pool_kernel_sizes=((8, 1, 1), (32, 1, 1)),
                                  head_output_size=(1, 1, 1), head_activation=nn.Sigmoid,
                                  head_output_with_global_average=False, head_spatial_resolution=(7, 7),
                                  head_spatial_scale=1.0 / 16.0, head_sampling_ratio=0):
    """SlowFast detection network (reference slowfast.py:364-582): the SlowFast trunk ends in PoolConcatPathway
    (temporal average per pathway, channel concat), the RoI head follows.  NB: like the reference, the trunk is
    built with ``create_bottleneck_block`` regardless of ``bottleneck``."""
    from .head import create_res_roi_pooling_head
    from .net import DetectionBBoxNetwork
    model = create_slowfast(
        slowfast_channel_reduction_ratio=slowfast_channel_reduction_ratio,
        slowfast_conv_channel_fusion_ratio=slowfast_conv_channel_fusion_ratio,
        slowfast_fusion_conv_kernel_size=slowfast_fusion_conv_kernel_size,
        slowfast_fusion_conv_stride=slowfast_fusion_conv_stride, input_channels=input_channels,
        model_depth=model_depth, model_num_class=model_num_class, dropout_rate=dropout_rate, norm=norm,
        activation=activation, stem_dim_outs=stem_dim_outs, stem_conv_kernel_sizes=stem_conv_kernel_sizes,
        stem_conv_strides=stem_conv_strides, stem_pool=stem_pool, stem_pool_kernel_sizes=stem_pool_kernel_sizes,
        stem_pool_strides=stem_pool_strides, stage_conv_a_kernel_sizes=stage_conv_a_kernel_sizes,
        stage_conv_b_kernel_sizes=stage_conv_b_kernel_sizes, stage_conv_b_num_groups=stage_conv_b_num_groups,
        stage_conv_b_dilations=stage_conv_b_dilations, stage_spatial_strides=stage_spatial_strides,
        stage_temporal_strides=stage_temporal_strides, bottleneck=create_bottleneck_block, head=None,
        head_pool=head_pool, head_pool_kernel_sizes=head_pool_kernel_sizes)
    stage_dim_out = stem_dim_outs[0] * 2 ** (len(_MODEL_STAGE_DEPTH[model_depth]) + 1)
    beta = stem_dim_outs[0] // stem_dim_outs[1]
    det_head = create_res_roi_pooling_head(
        in_features=stage_dim_out + stage_dim_out // beta, out_features=model_num_class, pool=None,
        output_size=head_output_size, dropout_rate=dropout_rate, activation=head_activation,
        output_with_global_average=head_output_with_global_average, resolution=head_spatial_resolution,
        spatial_scale=head_spatial_scale, sampling_ratio=head_sampling_ratio)
    return DetectionBBoxNetwork(model, det_head)
