"""Audiovisual SlowFast (reference models/audio_visual_slowfast.py): SlowFast with a third, audio pathway over a
log-mel spectrogram (B, 1, T, 1, F) that fuses into the Slow pathway at every stage."""
from typing import Tuple

import torch
import torch.nn as nn

from ..layers.utils import set_attributes
from ..module import B200Module
from .resnet import create_acoustic_bottleneck_block, create_bottleneck_block
from .slowfast import create_slowfast
from .stem import create_acoustic_res_basic_stem, create_res_basic_stem

_BB, _AB = create_bottleneck_block, create_acoustic_bottleneck_block


def create_audio_visual_slowfast(*, slowfast_channel_reduction_ratio=(8, 2), slowfast_conv_channel_fusion_ratio=2,
                                 fusion_builder=None, input_channels=(3, 3, 1), model_depth=50, model_num_class=400,
                                 dropout_rate=0.5, norm=nn.BatchNorm3d, activation=nn.ReLU,
                                 stem_dim_outs=(64, 8, 32),
                                 stem_conv_kernel_sizes=((1, 7, 7), (5, 7, 7), (9, 1, 9)),
                                 stem_conv_strides=((1, 2, 2), (1, 2, 2), (1, 1, 1)),
                                 stem_pool=(nn.MaxPool3d, nn.MaxPool3d, None),
                                 stem_pool_kernel_sizes=((1, 3, 3), (1, 3, 3), (1, 3, 3)),
                                 stem_pool_strides=((1, 2, 2), (1, 2, 2), (1, 1, 1)),
                                 stage_conv_a_kernel_sizes=(((1, 1, 1), (1, 1, 1), (3, 1, 1), (3, 1, 1)),
                                                            ((3, 1, 1), (3, 1, 1), (3, 1, 1), (3, 1, 1)),
                                                            ((1, 1, 1), (1, 1, 1), (1, 1, 1), (1, 1, 1))),
                                 stage_conv_b_kernel_sizes=(((1, 3, 3),) * 4, ((1, 3, 3),) * 4, ((3, 1, 3),) * 4),
                                 stage_conv_b_num_groups=((1, 1, 1, 1), (1, 1, 1, 1), (1, 1, 1, 1)),
                                 stage_conv_b_dilations=(((1, 1, 1),) * 4, ((1, 1, 1),) * 4, ((1, 1, 1),) * 4),
                                 stage_spatial_strides=((1, 2, 2, 2), (1, 2, 2, 2), (1, 2, 2, 2)),
                                 stage_temporal_strides=((1, 1, 1, 1), (1, 1, 1, 1), (1, 2, 2, 2)),
                                 bottleneck=((_BB, _BB, _BB, _BB), (_BB, _BB, _BB, _BB), (_AB, _AB, _BB, _BB)),
                                 head_pool=nn.AvgPool3d, head_pool_kernel_sizes=((8, 7, 7), (32, 7, 7), (16, 1, 10)),
                                 head_output_size=(1, 1, 1), head_activation=None,
                                 head_output_with_global_average=True) -> nn.Module:
    """AVSlowFast builder (reference audio_visual_slowfast.py:20-237); input is ``[slow, fast, audio]`` with the
    audio as (B, 1, T, 1, F)."""
    torch._C._log_api_usage_once("PYTORCHVIDEO.model.create_audio_visual_slowfast")
    if fusion_builder is None:
        fusion_builder = AudioToSlowFastFusionBuilder(
            slowfast_channel_reduction_ratio=slowfast_channel_reduction_ratio[0],
            slowfast_audio_reduction_ratio=slowfast_channel_reduction_ratio[1],
            conv_fusion_channel_ratio=slowfast_conv_channel_fusion_ratio, conv_kernel_size=(7, 1, 1),
            conv_kernel_size_a=(5, 1, 1), conv_stride=(4, 1, 1),
            conv_stride_a=((16, 1, 1), (16, 1, 1), (8, 1, 1), (4, 1, 1), (2, 1, 1)), norm=norm,
            activation=activation).create_module
    return create_slowfast(
        slowfast_channel_reduction_ratio=slowfast_channel_reduction_ratio,
        slowfast_conv_channel_fusion_ratio=slowfast_conv_channel_fusion_ratio, fusion_builder=fusion_builder,
        input_channels=input_channels, model_depth=model_depth, model_num_class=model_num_class,
        dropout_rate=dropout_rate, norm=norm, activation=activation,
        stem_function=(create_res_basic_stem, create_res_basic_stem, create_acoustic_res_basic_stem),
        stem_dim_outs=stem_dim_outs, stem_conv_kernel_sizes=stem_conv_kernel_sizes,
        stem_conv_strides=stem_conv_strides, stem_pool=stem_pool, stem_pool_kernel_sizes=stem_pool_kernel_sizes,
        stem_pool_strides=stem_pool_strides, stage_conv_a_kernel_sizes=stage_conv_a_kernel_sizes,
        stage_conv_b_kernel_sizes=stage_conv_b_kernel_sizes, stage_conv_b_num_groups=stage_conv_b_num_groups,
        stage_conv_b_dilations=stage_conv_b_dilations, stage_spatial_strides=stage_spatial_strides,
        stage_temporal_strides=stage_temporal_strides, bottleneck=bottleneck, head_pool=head_pool,
        head_pool_kernel_sizes=head_pool_kernel_sizes, head_output_size=head_output_size,
        head_activation=head_activation, head_output_with_global_average=head_output_with_global_average)


class AudioToSlowFastFusionBuilder:
    """Builds the per-stage FuseAudioToFastSlow modules (audio_visual_slowfast.py:240-381)."""

    def __init__(self, slowfast_channel_reduction_ratio, slowfast_audio_reduction_ratio, conv_fusion_channel_ratio,
                 conv_kernel_size, conv_kernel_size_a, conv_stride, conv_stride_a,
                 conv_fusion_channel_interm_dim=0.25, conv_num_a=2, norm=nn.BatchNorm3d, norm_eps=1e-5,
                 norm_momentum=0.1, activation=nn.ReLU, max_stage_idx=3) -> None:
        set_attributes(self, locals())

    def create_module(self, fusion_dim_in: int, stage_idx: int) -> nn.Module:
        if stage_idx > self.max_stage_idx:
            return nn.Identity()
        conv_stride = self.conv_stride[stage_idx] if isinstance(self.conv_stride[0], Tuple) else self.conv_stride
        conv_stride_a = (self.conv_stride_a[stage_idx] if isinstance(self.conv_stride_a[0], Tuple)
                         else self.conv_stride_a)
        conv_dim_in = fusion_dim_in // self.slowfast_channel_reduction_ratio
        conv_dim_in_a = fusion_dim_in // self.slowfast_audio_reduction_ratio
        fastslow_module = [nn.Conv3d(conv_dim_in, int(conv_dim_in * self.conv_fusion_channel_ratio),
                                     kernel_size=self.conv_kernel_size, stride=conv_stride,
                                     padding=[k // 2 for k in self.conv_kernel_size], bias=False)]
        if self.norm is not None:
            fastslow_module.append(self.norm(num_features=conv_dim_in * self.conv_fusion_channel_ratio,
                                             eps=self.norm_eps, momentum=self.norm_momentum))
        if self.activation is not None:
            fastslow_module.append(self.activation())
        if isinstance(self.conv_fusion_channel_interm_dim, int):
            interm = self.conv_fusion_channel_interm_dim
        else:
            interm = int(conv_dim_in_a * self.conv_fusion_channel_interm_dim)
        block_audio_to_fastslow = []
        cur_dim_in = conv_dim_in_a
        for idx in range(self.conv_num_a):
            if idx == self.conv_num_a - 1:
                cur_stride, cur_dim_out = conv_stride_a, int(conv_dim_in * self.conv_fusion_channel_ratio + fusion_dim_in)
            else:
                cur_stride, cur_dim_out = (1, 1, 1), interm
            block_audio_to_fastslow.append(nn.Conv3d(cur_dim_in, cur_dim_out, kernel_size=self.conv_kernel_size_a,
                                                     stride=cur_stride,
                                                     padding=[k // 2 for k in self.conv_kernel_size_a], bias=False))
            if self.norm is not None:
                block_audio_to_fastslow.append(self.norm(num_features=cur_dim_out, eps=self.norm_eps,
                                                         momentum=self.norm_momentum))
            if self.activation is not None:
                block_audio_to_fastslow.append(self.activation())
            cur_dim_in = cur_dim_out
        return FuseAudioToFastSlow(block_fast_to_slow=nn.Sequential(*fastslow_module),
                                   block_audio_to_fastslow=nn.Sequential(*block_audio_to_fastslow))


class FuseAudioToFastSlow(B200Module):
    """``[fuse_a + cat(x_s, block_fast_to_slow(x_f)), x_f, x_a]`` with
    ``fuse_a = block_audio_to_fastslow(mean(x_a, dim=-1, keepdim=True))`` (audio_visual_slowfast.py:384-418).

    The reference's forward also prints the size of the concatenated tensor (a leftover debug ``print``); this
    module does not.  On device neither the concat nor the add is a separate pass: the two convolutions that write
    the concat buffer add ``fuse_a`` in their epilogues."""

    def __init__(self, block_fast_to_slow: nn.Module, block_audio_to_fastslow: nn.Module) -> None:
        super().__init__()
        set_attributes(self, locals())
