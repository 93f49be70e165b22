from .audio_visual_slowfast import AudioToSlowFastFusionBuilder, FuseAudioToFastSlow, create_audio_visual_slowfast  # noqa: F401
from .csn import create_csn  # noqa: F401
from .head import ResNetBasicHead, ResNetRoIHead, RoIAlign, create_res_basic_head, create_res_roi_pooling_head  # noqa: F401
from .net import DetectionBBoxNetwork, MultiPathWayWithFuse, Net  # noqa: F401
from .r2plus1d import create_2plus1d_bottleneck_block, create_r2plus1d  # noqa: F401
from .resnet import (BottleneckBlock, ResBlock, ResStage, SeparableBottleneckBlock,  # noqa: F401
                     create_acoustic_bottleneck_block, create_acoustic_resnet, create_bottleneck_block,
                     create_res_block, create_res_stage, create_resnet, create_resnet_with_roi_head)
from .slowfast import FuseFastToSlow, PoolConcatPathway, create_slowfast, create_slowfast_with_roi_head  # noqa: F401
from .stem import ResNetBasicStem, create_acoustic_res_basic_stem, create_res_basic_stem  # noqa: F401
from .weight_init import init_net_weights  # noqa: F401
from .x3d import (ProjectedPool, create_x3d, create_x3d_bottleneck_block, create_x3d_head,  # noqa: F401
                  create_x3d_res_block, create_x3d_res_stage, create_x3d_stem)
from .head import SequencePool, VisionTransformerBasicHead, create_vit_basic_head  # noqa: F401,E402
from .stem import PatchEmbed, create_conv_patch_embed  # noqa: F401,E402
from .vision_transformers import MultiscaleVisionTransformers, create_multiscale_vision_transformers  # noqa: F401,E402
from .masked_multistream import (LSTM, LearnMaskedDefault, MaskedMultiPathWay, MaskedSequential,  # noqa: F401,E402
                                 MaskedTemporalPooling, TransposeMultiheadAttention, TransposeTransformerEncoder)
