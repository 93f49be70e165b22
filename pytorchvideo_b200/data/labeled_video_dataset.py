"""Labelled frame-folder video datasets: ``LabeledVideoDataset`` and the Kinetics / UCF101 builders."""
from __future__ import annotations

import gc
import logging
from typing import Any, Callable, Dict, List, Optional, Tuple, Type

import torch
import torch.utils.data

from .clip_sampling import ClipSampler
from .labeled_video_paths import LabeledVideoPaths
from .utils import GpuClipDataset, MultiProcessSampler
from .video import VideoPathHandler

logger = logging.getLogger(__name__)


class LabeledVideoDataset(GpuClipDataset, torch.utils.data.IterableDataset):
    """Iterates clips of labelled videos stored as directories of JPEG frames, decoded on the GPU.

    Videos come in ``video_sampler`` order (split across DataLoader workers by ``MultiProcessSampler``), clips in
    ``clip_sampler`` order.  A sample is {"video": float32 (C, T, H, W) on the GPU, "video_name", "video_index",
    "clip_index", "aug_index", the video's info dict (e.g. "label")}, passed through ``transform``; a transform that
    returns None skips the sample.  A video or clip that fails to load is skipped, and ``_MAX_CONSECUTIVE_FAILURES``
    failures in a row raise RuntimeError.  A path that is a video file fails to load: there is no video-file decoder.
    Frame videos have no audio, so ``decode_audio`` must be False (the default True fails every load, as in the
    reference).  ``host_only()`` yields file bytes instead (see ``GpuClipDataset``).
    """

    _MAX_CONSECUTIVE_FAILURES = 10

    def __init__(self, labeled_video_paths: List[Tuple[str, Optional[dict]]], clip_sampler: ClipSampler,
                 video_sampler: Type[torch.utils.data.Sampler] = torch.utils.data.RandomSampler,
                 transform: Optional[Callable[[dict], Any]] = None, decode_audio: bool = True,
                 decode_video: bool = True, decoder: str = "pyav") -> None:
        self._decode_audio = decode_audio
        self._decode_video = decode_video
        self._transform = transform
        self._clip_sampler = clip_sampler
        self._labeled_videos = labeled_video_paths
        self._decoder = decoder
        # a RandomSampler gets its own generator, reseeded identically in every worker (see __iter__), so that the
        # workers split one permutation
        self._video_random_generator = None
        if video_sampler == torch.utils.data.RandomSampler:
            self._video_random_generator = torch.Generator()
            self._video_sampler = video_sampler(self._labeled_videos, generator=self._video_random_generator)
        else:
            self._video_sampler = video_sampler(self._labeled_videos)
        self._video_sampler_iter = None
        # the video being sampled (video, info, index), its current clip and the end time of the last clip
        self._loaded_video_label = None
        self._loaded_clip = None
        self._last_clip_end_time = None
        self.video_path_handler = VideoPathHandler()

    @property
    def video_sampler(self):
        """The sampler of the video order (set its epoch here for a DistributedSampler)."""
        return self._video_sampler

    @property
    def num_videos(self):
        return len(self.video_sampler)

    def _release_video(self):
        self._loaded_video_label[0].close()
        self._loaded_video_label = None
        self._last_clip_end_time = None
        self._clip_sampler.reset()
        gc.collect()

    def __next__(self) -> dict:
        self._check_process()
        if not self._video_sampler_iter:
            self._video_sampler_iter = iter(MultiProcessSampler(self._video_sampler))
        for i_try in range(self._MAX_CONSECUTIVE_FAILURES):
            if self._loaded_video_label:
                video, info_dict, video_index = self._loaded_video_label
            else:
                video_index = next(self._video_sampler_iter)
                try:
                    video_path, info_dict = self._labeled_videos[video_index]
                    video = self.video_path_handler.video_from_path(video_path, decode_audio=self._decode_audio,
                                                                    decode_video=self._decode_video,
                                                                    decoder=self._decoder)
                    self._loaded_video_label = (video, info_dict, video_index)
                except Exception as e:
                    logger.debug("Failed to load video with error: {}; trial {}".format(e, i_try))
                    logger.exception("Video load exception")
                    continue

            clip_start, clip_end, clip_index, aug_index, is_last_clip = self._clip_sampler(
                self._last_clip_end_time, video.duration, info_dict)
            if isinstance(clip_start, list):
                # several clips per sample: loaded together at the first augmentation, None if any is missing
                if aug_index[0] == 0:
                    clips = []
                    for start, end in zip(clip_start, clip_end):
                        clip = self._load_clip(video, start, end)
                        if clip is None or clip["video"] is None:
                            clips = None
                            break
                        clips.append(clip)
                    self._loaded_clip = None if clips is None else {k: [c[k] for c in clips] for k in clips[0]}
                last = is_last_clip[-1]
            else:
                if aug_index == 0:         # the other augmentations of a clip reuse it
                    self._loaded_clip = self._load_clip(video, clip_start, clip_end)
                last = is_last_clip
            self._last_clip_end_time = clip_end

            missing = self._loaded_clip is None or self._loaded_clip["video"] is None
            if last or missing:
                self._release_video()
                if missing:
                    logger.debug("Failed to load clip {}; trial {}".format(video.name, i_try))
                    continue

            audio = self._loaded_clip["audio"]
            sample = {"video": self._loaded_clip["video"], "video_name": video.name, "video_index": video_index,
                      "clip_index": clip_index, "aug_index": aug_index, **info_dict,
                      **({"audio": audio} if audio is not None else {})}
            sample = self._apply_transform(sample)
            if sample is None:
                continue
            return sample
        raise RuntimeError(f"Failed to load video after {self._MAX_CONSECUTIVE_FAILURES} retries.")

    def __iter__(self):
        self._video_sampler_iter = None
        # every worker reseeds the RandomSampler generator with the seed its DataLoader iteration shares
        info = torch.utils.data.get_worker_info()
        if self._video_random_generator is not None and info is not None:
            self._video_random_generator.manual_seed(info.seed - info.id)
        return self


def labeled_video_dataset(data_path: str, clip_sampler: ClipSampler,
                          video_sampler: Type[torch.utils.data.Sampler] = torch.utils.data.RandomSampler,
                          transform: Optional[Callable[[Dict[str, Any]], Dict[str, Any]]] = None,
                          video_path_prefix: str = "", decode_audio: bool = True,
                          decoder: str = "pyav") -> LabeledVideoDataset:
    """A ``LabeledVideoDataset`` of the videos ``LabeledVideoPaths.from_path(data_path)`` lists (a csv file of
    ``<path> <label>`` lines, or a directory of class directories), each path under ``video_path_prefix``."""
    paths = LabeledVideoPaths.from_path(data_path)
    paths.path_prefix = video_path_prefix
    return LabeledVideoDataset(paths, clip_sampler, video_sampler, transform, decode_audio=decode_audio,
                               decoder=decoder)


def Kinetics(data_path: str, clip_sampler: ClipSampler,
             video_sampler: Type[torch.utils.data.Sampler] = torch.utils.data.RandomSampler,
             transform: Optional[Callable[[Dict[str, Any]], Dict[str, Any]]] = None, video_path_prefix: str = "",
             decode_audio: bool = True, decoder: str = "pyav") -> LabeledVideoDataset:
    """Kinetics-400/600/700 stored as frame folders: ``labeled_video_dataset`` with the same arguments."""
    return labeled_video_dataset(data_path, clip_sampler, video_sampler, transform, video_path_prefix, decode_audio,
                                 decoder)


def Ucf101(data_path: str, clip_sampler: ClipSampler,
           video_sampler: Type[torch.utils.data.Sampler] = torch.utils.data.RandomSampler,
           transform: Optional[Callable[[Dict[str, Any]], Dict[str, Any]]] = None, video_path_prefix: str = "",
           decode_audio: bool = True, decoder: str = "pyav") -> LabeledVideoDataset:
    """UCF101 stored as frame folders: ``labeled_video_dataset`` with the same arguments."""
    return labeled_video_dataset(data_path, clip_sampler, video_sampler, transform, video_path_prefix, decode_audio,
                                 decoder)
