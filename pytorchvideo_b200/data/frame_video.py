"""FrameVideo: a video stored as one JPEG file per frame, decoded on the GPU.

Same public surface and clip rules as the reference's data/frame_video.py:
- frame i covers [i / fps, (i + 1) / fps), and the video lasts len(frames) / fps seconds
- a clip [start_sec, end_sec) holds frames ceil(fps * start_sec) up to, not including, ceil(fps * min(end_sec,
  duration)), and never past the last frame
- a start before 0 or after the duration gives None, after a logged warning
- an optional frame_filter maps that index list to the indices to load
The files are read on the host and decoded together by ``decode_jpeg_frames`` straight into float32; the clip is
(C, T, H, W) with THWC strides, the layout of the reference's ``thwc_to_cthw(frames).to(torch.float32)``.
"""
import logging
import math
import os
import re
from concurrent.futures import ThreadPoolExecutor
from typing import Callable, Dict, List, NamedTuple, Optional

import torch

from .jpeg import decode_jpeg_frames

logger = logging.getLogger(__name__)

FrameFilter = Callable[[List[int]], List[int]]


def natural_sort_key(name: str):
    """Orders names by their runs of digits as numbers ("f2" before "f10"); digit runs sit at the odd positions."""
    return [int(part) if i % 2 else part for i, part in enumerate(re.split(r"(\d+)", name))]


def clip_frame_indices(fps: float, duration: float, n_frames: int, start_sec: float, end_sec: float) -> Optional[List[int]]:
    """Indices of the frames in [start_sec, end_sec), or None when start_sec lies outside [0, duration]."""
    if not 0 <= start_sec <= duration:
        return None
    first = math.ceil(fps * start_sec)
    stop = min(math.ceil(fps * min(end_sec, duration)), n_frames)
    return list(range(first, stop))


class ClipFrames(NamedTuple):
    """A clip's frames as file bytes, not decoded: what a DataLoader worker can produce without the GPU."""

    data: List[bytes]            # file bytes of each kept frame, in clip order (a repeated frame repeats its bytes)
    paths: List[str]             # file of each kept frame
    frame_indices: List[int]     # the clip's frame indices, as get_clip returns them
    kept: List[int]              # the positions in frame_indices that data and paths hold


class FrameVideo:
    """A video whose frames are image files; get_clip returns clips on the current CUDA device."""

    def __init__(self, duration: float, fps: float, video_frame_to_path_fn: Callable[[int], str] = None,
                 video_frame_paths: List[str] = None, multithreaded_io: bool = False) -> None:
        """
        Args:
            duration: length of the video in seconds.
            fps: frame rate that maps frame indices to timestamps.
            video_frame_to_path_fn: the file path of a frame index.  Give this or video_frame_paths, not both.
            video_frame_paths: the file path of every frame, in order.
            multithreaded_io: read a clip's files on several threads.
        """
        assert (video_frame_to_path_fn is None) != (video_frame_paths is None), (
            "FrameVideo needs exactly one of video_frame_to_path_fn and video_frame_paths")
        self._duration = duration
        self._fps = fps
        self._multithreaded_io = multithreaded_io
        self._path_fn = video_frame_to_path_fn
        self._paths = video_frame_paths
        # named after the directory holding frame 0
        self._name = os.path.basename(os.path.dirname(self._frame_path(0)))

    @classmethod
    def from_directory(cls, path: str, fps: float = 30.0, multithreaded_io=False,
                       path_order_cache: Optional[Dict[str, List[str]]] = None):
        """Every file in directory ``path``, in natural order, as one video at ``fps``.

        ``path_order_cache`` maps a directory to its ordered frame paths: an entry for ``path`` is used instead of
        listing the directory, and a listing is stored in it.
        """
        cached = None if path_order_cache is None else path_order_cache.get(path)
        if cached is None:
            assert os.path.isdir(path), f"{path} is not a directory"
            cached = [os.path.join(path, name) for name in sorted(os.listdir(path), key=natural_sort_key)]
            if path_order_cache is not None:
                path_order_cache[path] = cached
        return cls.from_frame_paths(cached, fps, multithreaded_io)

    @classmethod
    def from_frame_paths(cls, video_frame_paths: List[str], fps: float = 30.0, multithreaded_io: bool = False):
        """A video made of the given frame files at ``fps``; it lasts len(video_frame_paths) / fps seconds."""
        assert len(video_frame_paths) > 0, "FrameVideo needs at least one frame path"
        return cls(len(video_frame_paths) / fps, fps, video_frame_paths=video_frame_paths,
                   multithreaded_io=multithreaded_io)

    @property
    def name(self) -> str:
        return self._name

    @property
    def duration(self) -> float:
        """Length of the video (its end time) in seconds."""
        return self._duration

    def frame_indices(self, start_sec: float, end_sec: float,
                      frame_filter: Optional[FrameFilter] = None) -> Optional[List[int]]:
        """The frame indices get_clip loads for [start_sec, end_sec): None (and a warning) when start_sec is outside
        [0, duration], else the indices in range, passed through frame_filter when one is given."""
        # len() of the path list, as the reference: a video built from video_frame_to_path_fn has no frame count
        indices = clip_frame_indices(self._fps, self._duration, len(self._paths), start_sec, end_sec)
        if indices is None:
            logger.warning("FrameVideo %s: no frames in [%s, %s) s; the video spans [0, %s] s",
                           self._name, start_sec, end_sec, self._duration)
            return None
        return frame_filter(indices) if frame_filter else indices

    def get_clip(self, start_sec: float, end_sec: float,
                 frame_filter: Optional[FrameFilter] = None) -> Optional[Dict]:
        """The frames in [start_sec, end_sec), subsampled by ``frame_filter`` before any file is read.

        Returns {"video": float32 (C, T, H, W) RGB values 0..255 on the current CUDA device, "frame_indices": the
        indices loaded, "audio": None}, or None when start_sec is outside the video.  An empty index list raises
        ValueError.  A frame that cannot be decoded, or frames of different sizes, raise RuntimeError naming the frame.
        """
        indices = self.frame_indices(start_sec, end_sec, frame_filter)
        if indices is None:
            return None
        if not indices:
            raise ValueError("FrameVideo %s: no frame to load for [%s, %s) s" % (self._name, start_sec, end_sec))
        files = _read_all([self._frame_path(i) for i in indices], self._multithreaded_io)
        thwc = decode_jpeg_frames(files, out_dtype=torch.float32)
        return {"video": thwc.permute(3, 0, 1, 2), "frame_indices": indices, "audio": None}

    def get_clip_frames(self, start_sec: float, end_sec: float, frame_filter: Optional[FrameFilter] = None,
                        keep: Optional[Callable[[int], List[int]]] = None) -> Optional[ClipFrames]:
        """The clip get_clip would load, as the files' bytes: reads, never decodes, so it runs on any host process.

        ``keep`` maps the clip's frame count to the positions to read (a temporal subsample), so frames a transform
        would drop are not read; by default every frame is.  Returns None, or raises ValueError, where get_clip does.
        """
        indices = self.frame_indices(start_sec, end_sec, frame_filter)
        if indices is None:
            return None
        if not indices:
            raise ValueError("FrameVideo %s: no frame to load for [%s, %s) s" % (self._name, start_sec, end_sec))
        kept = list(range(len(indices))) if keep is None else [int(k) for k in keep(len(indices))]
        paths = [self._frame_path(indices[k]) for k in kept]
        unique = list(dict.fromkeys(paths))
        read = dict(zip(unique, _read_all(unique, self._multithreaded_io)))
        return ClipFrames([read[p] for p in paths], paths, indices, kept)

    def close(self) -> None:
        """Nothing to release: a frame video holds no open file."""

    def _frame_path(self, index: int) -> str:
        if self._path_fn is not None:
            return self._path_fn(index)
        return self._paths[index]


def _read_bytes(path):
    with open(path, "rb") as f:
        return f.read()


def _read_all(paths, threaded):
    if threaded and len(paths) > 1:
        with ThreadPoolExecutor(max_workers=min(32, len(paths))) as pool:
            return list(pool.map(_read_bytes, paths))
    return [_read_bytes(p) for p in paths]
