"""Charades stored as image frames (one JPEG per frame, listed in a csv)."""
import csv
import functools
import itertools
import os
from collections import defaultdict
from typing import Any, Callable, List, Optional, Tuple, Type

import torch
import torch.utils.data

from .clip_sampling import ClipSampler
from .frame_video import FrameVideo
from .utils import GpuClipDataset, MultiProcessSampler


class Charades(GpuClipDataset, torch.utils.data.IterableDataset):
    """Clips of the Charades videos, decoded on the GPU.

    ``data_path`` is the space-separated csv of the frame lists (columns original_vido_id, video_id, frame_id, path,
    labels); a frame's labels are a comma-separated list, possibly empty.  A sample is {"video": float32 (C, T, H, W)
    on the GPU, "label": the label lists of the frames from the clip's first to its last kept frame, "video_label":
    the video's labels, "video_name": str(video_index), "video_index", "clip_index", "aug_index"}.  With
    ``frames_per_clip`` a clip keeps that many frames at ``linspace`` positions.  ``host_only()`` yields file bytes
    instead (see ``GpuClipDataset``).
    """

    NUM_CLASSES = 157

    def __init__(self, data_path: str, clip_sampler: ClipSampler,
                 video_sampler: Type[torch.utils.data.Sampler] = torch.utils.data.RandomSampler,
                 transform: Optional[Callable[[dict], Any]] = None, video_path_prefix: str = "",
                 frames_per_clip: Optional[int] = None) -> None:
        self._transform = transform
        self._clip_sampler = clip_sampler
        self._path_to_videos, self._labels, self._video_labels = _read_video_paths_and_labels(
            data_path, prefix=video_path_prefix)
        self._video_sampler = video_sampler(self._path_to_videos)
        self._video_sampler_iter = None
        self._frame_filter = (functools.partial(Charades._sample_clip_frames, frames_per_clip=frames_per_clip)
                              if frames_per_clip is not None else None)
        self._loaded_video = None
        self._loaded_clip = None
        self._next_clip_start_time = 0.0

    @staticmethod
    def _sample_clip_frames(frame_indices: List[int], frames_per_clip: int) -> List[int]:
        """frames_per_clip of the indices at clamp(linspace(0, n - 1, frames_per_clip)).long() positions."""
        n = len(frame_indices)
        positions = torch.clamp(torch.linspace(0, n - 1, frames_per_clip), 0, n - 1).long()
        return [frame_indices[p] for p in positions]

    @property
    def video_sampler(self) -> torch.utils.data.Sampler:
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
        if aug_index == 0:                 # the other augmentations of a clip reuse it
            self._loaded_clip = self._load_clip(video, clip_start, clip_end, self._frame_filter)
        frame_indices = self._loaded_clip["frame_indices"]
        self._next_clip_start_time = clip_end
        if is_last_clip:
            self._loaded_video = None
            self._next_clip_start_time = 0.0

        labels = self._labels[video_index]
        sample = {"video": self._loaded_clip["video"],
                  "label": [labels[i] for i in range(min(frame_indices), max(frame_indices) + 1)],
                  "video_label": self._video_labels[video_index], "video_name": str(video_index),
                  "video_index": video_index, "clip_index": clip_index, "aug_index": aug_index}
        return self._apply_transform(sample)

    def __iter__(self):
        return self


def _read_frame_csv(path: str, prefix: str):
    """Rows of a space-separated frame csv (original_vido_id video_id frame_id path labels), each asserted to have five
    columns, as (video name, frame path under prefix, row)."""
    with open(path, "r") as f:
        for row in csv.DictReader(f, delimiter=" "):
            assert len(row) == 5
            yield row["original_vido_id"], os.path.join(prefix, row["path"]), row


def _read_video_paths_and_labels(video_path_label_file: str, prefix: str = "") -> Tuple[List, List, List]:
    """(frame paths per video, label list per frame per video, video labels per video), videos in first-seen order;
    a video's labels are the distinct labels of its frames."""
    image_paths, labels = defaultdict(list), defaultdict(list)
    for name, path, row in _read_frame_csv(video_path_label_file, prefix):
        image_paths[name].append(path)
        text = row["labels"].replace('"', "")
        labels[name].append([int(x) for x in text.split(",")] if text else [])
    names = list(image_paths)
    frame_labels = [labels[n] for n in names]
    return ([image_paths[n] for n in names], frame_labels,
            [list(set(itertools.chain(*per_frame))) for per_frame in frame_labels])
