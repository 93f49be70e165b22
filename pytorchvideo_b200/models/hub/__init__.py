"""Named model configurations (reference models/hub/*.py).  ``pretrained=True`` needs network
access for the checkpoint download and is therefore rejected in this offline build; load a local
``checkpoint["model_state"]`` with ``model.load_state_dict`` instead (keys are identical)."""
import torch.nn as nn

from ..csn import create_csn
from ..r2plus1d import create_r2plus1d
from ..resnet import create_resnet, create_resnet_with_roi_head
from ..slowfast import create_slowfast, create_slowfast_with_roi_head
from ..x3d import create_x3d


def _build(builder, pretrained, **kwargs):
    if pretrained:
        raise RuntimeError("pretrained weights require a download; load a local state_dict instead")
    return builder(**kwargs)


def slow_r50(pretrained=False, progress=True, **kw):
    return _build(create_resnet, pretrained, stem_conv_kernel_size=(1, 7, 7), head_pool_kernel_size=(8, 7, 7),
                  model_depth=50, **kw)


def slow_r50_detection(pretrained=False, progress=True, **kw):
    """Slow-R50 4x16 detection model (AVA), reference hub/resnet.py:73-90."""
    return _build(create_resnet_with_roi_head, pretrained, **kw)


def c2d_r50(pretrained=False, progress=True, **kw):
    return _build(create_resnet, pretrained, stem_conv_kernel_size=(1, 7, 7), stage1_pool=nn.MaxPool3d,
                  stage_conv_a_kernel_size=((1, 1, 1),) * 4, **kw)


def i3d_r50(pretrained=False, progress=True, **kw):
    return _build(create_resnet, pretrained, stem_conv_kernel_size=(5, 7, 7), stage1_pool=nn.MaxPool3d,
                  stage_conv_a_kernel_size=((3, 1, 1), [(3, 1, 1), (1, 1, 1)], [(3, 1, 1), (1, 1, 1)],
                                            [(1, 1, 1), (3, 1, 1)]), **kw)


def slowfast_r50(pretrained=False, progress=True, **kw):
    return _build(create_slowfast, pretrained, model_depth=50, slowfast_fusion_conv_kernel_size=(7, 1, 1), **kw)


def slowfast_r50_detection(pretrained=False, progress=True, **kw):
    """SlowFast-R50 8x8 detection model (AVA), reference hub/slowfast.py:150-181."""
    return _build(create_slowfast_with_roi_head, pretrained, **kw)


def slowfast_r101(pretrained=False, progress=True, **kw):
    return _build(create_slowfast, pretrained, model_depth=101, slowfast_fusion_conv_kernel_size=(5, 1, 1), **kw)


def slowfast_16x8_r101_50_50(pretrained=False, progress=True, **kw):
    """SlowFast-R101 16x8 whose res4 has temporal conv_a kernels in its first 6 blocks only (reference
    hub/slowfast.py:101-147).  Inputs: 16 Slow and 64 Fast frames."""
    res4 = ((3, 1, 1),) * 6 + ((1, 1, 1),) * (23 - 6)
    return _build(create_slowfast, pretrained, model_depth=101, slowfast_fusion_conv_kernel_size=(5, 1, 1),
                  stage_conv_a_kernel_sizes=(((1, 1, 1), (1, 1, 1), res4, (3, 1, 1)),
                                             ((3, 1, 1), (3, 1, 1), res4, (3, 1, 1))),
                  head_pool_kernel_sizes=((16, 7, 7), (64, 7, 7)), **kw)


def x3d_xs(pretrained=False, progress=True, **kw):
    return _build(create_x3d, pretrained, input_clip_length=4, input_crop_size=160, **kw)


def x3d_s(pretrained=False, progress=True, **kw):
    return _build(create_x3d, pretrained, input_clip_length=13, input_crop_size=160, **kw)


def x3d_m(pretrained=False, progress=True, **kw):
    return _build(create_x3d, pretrained, input_clip_length=16, input_crop_size=224, **kw)


def x3d_l(pretrained=False, progress=True, **kw):
    return _build(create_x3d, pretrained, input_clip_length=16, input_crop_size=312, depth_factor=5.0, **kw)


def efficient_x3d_xs(pretrained=False, progress=True, **kw):
    """X3D-XS in the mobile efficient-block tree (reference hub/efficient_x3d_mobile_cpu.py)."""
    from ..accelerator.mobile_cpu.efficient_x3d import create_x3d as create_efficient_x3d
    return _build(create_efficient_x3d, pretrained, expansion="XS", **kw)


def efficient_x3d_s(pretrained=False, progress=True, **kw):
    """X3D-S in the mobile efficient-block tree (reference hub/efficient_x3d_mobile_cpu.py)."""
    from ..accelerator.mobile_cpu.efficient_x3d import create_x3d as create_efficient_x3d
    return _build(create_efficient_x3d, pretrained, expansion="S", **kw)


def csn_r101(pretrained=False, progress=True, **kw):
    return _build(create_csn, pretrained, model_depth=101, stem_pool=nn.MaxPool3d, head_pool_kernel_size=(4, 7, 7),
                  **kw)


def r2plus1d_r50(pretrained=False, progress=True, **kw):
    return _build(create_r2plus1d, pretrained, dropout_rate=0.5, **kw)


_MVIT_VIDEO_BASE = {
    "spatial_size": 224, "temporal_size": 16,
    "embed_dim_mul": [[1, 2.0], [3, 2.0], [14, 2.0]], "atten_head_mul": [[1, 2.0], [3, 2.0], [14, 2.0]],
    "pool_q_stride_size": [[1, 1, 2, 2], [3, 1, 2, 2], [14, 1, 2, 2]], "pool_kv_stride_adaptive": [1, 8, 8],
    "pool_kvq_kernel": [3, 3, 3],
}


def mvit_base_16x4(pretrained=False, progress=True, **kw):
    from ..vision_transformers import create_multiscale_vision_transformers
    cfg = dict(_MVIT_VIDEO_BASE)
    cfg.update(kw)
    return _build(create_multiscale_vision_transformers, pretrained, **cfg)


def mvit_base_32x3(pretrained=False, progress=True, **kw):
    from ..vision_transformers import create_multiscale_vision_transformers
    cfg = dict(_MVIT_VIDEO_BASE, temporal_size=32)
    cfg.update(kw)
    return _build(create_multiscale_vision_transformers, pretrained, **cfg)


_MVIT_IMAGE_BASE_16 = {
    "spatial_size": 224, "temporal_size": 1, "depth": 16,
    "conv_patch_embed_kernel": [7, 7], "conv_patch_embed_stride": [4, 4], "conv_patch_embed_padding": [3, 3],
    "use_2d_patch": True,
    "embed_dim_mul": [[1, 2.0], [3, 2.0], [14, 2.0]], "atten_head_mul": [[1, 2.0], [3, 2.0], [14, 2.0]],
    "pool_q_stride_size": [[1, 1, 2, 2], [3, 1, 2, 2], [14, 1, 2, 2]], "pool_kv_stride_adaptive": [1, 4, 4],
    "pool_kvq_kernel": [1, 3, 3],
}


def mvit_base_16(pretrained=False, progress=True, **kw):
    """Image MViT-B, depth 16 (reference hub/vision_transformers.py:41-54, 127-158): takes (B, 3, 224, 224) images."""
    from ..vision_transformers import create_multiscale_vision_transformers
    cfg = dict(_MVIT_IMAGE_BASE_16)
    cfg.update(kw)
    return _build(create_multiscale_vision_transformers, pretrained, **cfg)
