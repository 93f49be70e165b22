"""Input pipeline on the GPU: frame-folder videos decoded by the library's batched baseline-JPEG decoder."""
from .frame_video import FrameVideo  # noqa: F401
from .jpeg import decode_jpeg_frames, parse_jpeg  # noqa: F401
