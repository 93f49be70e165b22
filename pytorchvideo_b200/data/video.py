"""Videos by path: a directory of frame files is a ``FrameVideo``."""
import os

from .frame_video import FrameVideo


class VideoPathHandler:
    """Opens the video at a path and caches the frame order of every directory it has listed."""

    def __init__(self) -> None:
        self.path_order_cache = {}

    def video_from_path(self, filepath, decode_video=True, decode_audio=False, decoder="pyav", fps=30):
        """A ``FrameVideo`` at ``fps`` for a directory.  A file is an encoded video, which this engine has no
        decoder for: NotImplementedError.  A missing path: FileNotFoundError."""
        if os.path.isfile(filepath):
            raise NotImplementedError("%s is a video file; pytorchvideo_b200 has no video-file decoder and reads "
                                      "videos stored as directories of JPEG frames" % filepath)
        if os.path.isdir(filepath):
            assert not decode_audio, "decode_audio must be False when using FrameVideo"
            return FrameVideo.from_directory(filepath, fps, path_order_cache=self.path_order_cache)
        raise FileNotFoundError(f"{filepath} not found.")
