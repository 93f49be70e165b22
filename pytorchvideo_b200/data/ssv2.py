"""Something-Something v2 stored as image frames."""
import functools
import json
import random
from collections import defaultdict
from typing import Any, Callable, List, Optional, Tuple, Type

import numpy as np
import torch
import torch.utils.data

from .charades import _read_frame_csv
from .clip_sampling import ClipSampler
from .frame_video import FrameVideo
from .utils import GpuClipDataset, MultiProcessSampler


class SSv2(GpuClipDataset, torch.utils.data.IterableDataset):
    """Clips of the SSv2 videos, decoded on the GPU.

    label_name_file maps template names to label indices (json), video_label_file lists {"id", "template"} per video
    (json), video_path_label_file is the space-separated frame csv (as Charades').  Only videos in both the json and
    the csv are kept, in the json's order.  Every clip is the whole video; with ``frames_per_clip`` it keeps one frame
    per equal segment, the middle one, or one drawn with ``random.randint`` when ``rand_sample_frames``.  A sample is
    {"video": float32 (C, T, H, W) on the GPU, "label", "video_name": str(video_index), "video_index", "clip_index",
    "aug_index"}.  ``host_only()`` yields file bytes instead (see ``GpuClipDataset``).
    """

    def __init__(self, label_name_file: str, video_label_file: str, video_path_label_file: str,
                 clip_sampler: ClipSampler,
                 video_sampler: Type[torch.utils.data.Sampler] = torch.utils.data.RandomSampler,
                 transform: Optional[Callable[[dict], Any]] = None, video_path_prefix: str = "",
                 frames_per_clip: Optional[int] = None, rand_sample_frames: bool = False) -> None:
        self._transform = transform
        self._clip_sampler = clip_sampler
        self._path_to_videos, self._labels = _read_video_paths_and_labels(
            label_name_file, video_label_file, video_path_label_file, prefix=video_path_prefix)
        self._video_sampler = video_sampler(self._path_to_videos)
        self._video_sampler_iter = None
        self._frame_filter = (functools.partial(SSv2._sample_clip_frames, frames_per_clip=frames_per_clip,
                                                rand_sample=rand_sample_frames)
                              if frames_per_clip is not None else None)
        self._loaded_video = None
        self._next_clip_start_time = 0.0

    @staticmethod
    def _sample_clip_frames(frame_indices: List[int], frames_per_clip: int, rand_sample: bool) -> List[int]:
        """One frame of each of frames_per_clip segments [round(s * i), round(s * (i + 1))], s = (n - 1) /
        frames_per_clip: a random.randint draw in it, or its midpoint."""
        seg = float(len(frame_indices) - 1) / frames_per_clip
        picks = []
        for i in range(frames_per_clip):
            lo, hi = int(np.round(seg * i)), int(np.round(seg * (i + 1)))
            picks.append(random.randint(lo, hi) if rand_sample else (lo + hi) // 2)
        return [frame_indices[p] for p in picks]

    @property
    def video_sampler(self):
        return self._video_sampler

    def __next__(self) -> dict:
        self._check_process()
        if not self._video_sampler_iter:
            self._video_sampler_iter = iter(MultiProcessSampler(self._video_sampler))
        if self._loaded_video:
            video, video_index = self._loaded_video
        else:
            video_index = next(self._video_sampler_iter)
            video = FrameVideo.from_frame_paths(self._path_to_videos[video_index])
            self._loaded_video = (video, video_index)

        clip_start, clip_end, clip_index, aug_index, is_last_clip = self._clip_sampler(
            self._next_clip_start_time, video.duration, {})
        if aug_index == 0:                 # the whole video; the other augmentations of a clip reuse it
            self._loaded_clip = self._load_clip(video, 0, video.duration, self._frame_filter)
        self._next_clip_start_time = clip_end
        if is_last_clip:
            self._loaded_video = None
            self._next_clip_start_time = 0.0

        sample = {"video": self._loaded_clip["video"], "label": self._labels[video_index],
                  "video_name": str(video_index), "video_index": video_index, "clip_index": clip_index,
                  "aug_index": aug_index}
        return self._apply_transform(sample)

    def __iter__(self):
        return self


def _read_video_paths_and_labels(label_name_file: str, video_label_file: str, video_path_label_file: str,
                                 prefix: str = "") -> Tuple[List[List[str]], List[int]]:
    """(frame paths per video, label per video) of the videos listed in both video_label_file and the csv."""
    paths = defaultdict(list)
    for name, path, _ in _read_frame_csv(video_path_label_file, prefix):
        paths[name].append(path)
    with open(label_name_file, "r") as f:
        label_of = json.load(f)
    with open(video_label_file, "r") as f:
        videos = json.load(f)
    image_paths, labels = [], []
    for video in videos:
        if video["id"] in paths:
            image_paths.append(paths[video["id"]])
            labels.append(int(label_of[video["template"].replace("[", "").replace("]", "")]))
    return image_paths, labels
