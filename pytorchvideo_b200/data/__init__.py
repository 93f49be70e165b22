"""Input pipeline on the GPU: frame-folder videos decoded by the library's batched baseline-JPEG decoder, the
reference's datasets and clip samplers over them, and batch loaders that decode and transform a batch (of clips, or
of clips and their boxes) at once."""
from .ava import Ava  # noqa: F401
from .charades import Charades  # noqa: F401
from .clip_sampling import (  # noqa: F401
    ClipInfo,
    ClipInfoList,
    ClipSampler,
    ConstantClipsPerVideoSampler,
    make_clip_sampler,
    RandomClipSampler,
    RandomMultiClipSampler,
    RandomMultiClipSamplerTruncateFromStart,
    UniformClipSampler,
    UniformClipSamplerTruncateFromStart,
)
from .frame_video import ClipFrames, FrameVideo  # noqa: F401
from .jpeg import decode_jpeg_frames, parse_jpeg  # noqa: F401
from .labeled_video_dataset import Kinetics, labeled_video_dataset, LabeledVideoDataset, Ucf101  # noqa: F401
from .labeled_video_paths import LabeledVideoPaths  # noqa: F401
from .loader import ClipBatchLoader, DetectionBatchLoader  # noqa: F401
from .ssv2 import SSv2  # noqa: F401
from .utils import MultiProcessSampler  # noqa: F401
from .video import VideoPathHandler  # noqa: F401
