from .transforms import (ApplyTransformToKey, CenterCropVideo, ConvertUint8ToFloat, Div255,  # noqa: F401
                         FusedClipTransform, Normalize, RandomCropVideo, RandomShortSideScale, ShortSideScale,
                         UniformCropVideo, UniformTemporalSubsample, create_video_transform, SlowFastPackPathway,
                         RemoveKey, RandomResizedCrop, Permute, RandAugment, AugMix, FusedDetectionTransform)
from .mix import CutMix, MixUp, MixVideo  # noqa: F401
from .color import (ApplyTransformToKeyOnList, ColorJitterVideoSSl, FusedContrastiveTransform,  # noqa: F401
                    RepeatandConverttoList)
from . import functional  # noqa: F401
