"""Clip samplers: where in a video the next clip starts and ends.

The names, arguments and results are the reference's (data/clip_sampling.py), and so are the arithmetic and the
random draws: the uniform sampler works in ``Fraction`` seconds, and the random samplers draw their start from
Python's ``random.uniform``, so a run seeded with ``random.seed`` samples the reference's clips.
"""
import random
from abc import ABC, abstractmethod
from fractions import Fraction
from typing import Any, Dict, List, NamedTuple, Optional, Tuple, Union


class ClipInfo(NamedTuple):
    """One clip: start and end in seconds, its index in the video, its augmentation index, and whether it is the
    video's last clip."""

    clip_start_sec: Union[float, Fraction]
    clip_end_sec: Union[float, Fraction]
    clip_index: int
    aug_index: int
    is_last_clip: bool


class ClipInfoList(NamedTuple):
    """Several clips of one video, one list per ``ClipInfo`` field."""

    clip_start_sec: List[float]
    clip_end_sec: List[float]
    clip_index: List[float]
    aug_index: List[float]
    is_last_clip: List[float]


class ClipSampler(ABC):
    """Maps (end of the previous clip, video duration, annotation) to the next ``ClipInfo``."""

    def __init__(self, clip_duration: Union[float, Fraction]) -> None:
        self._clip_duration = Fraction(clip_duration)
        self._current_clip_index = 0
        self._current_aug_index = 0

    @abstractmethod
    def __call__(self, last_clip_end_time: Union[float, Fraction], video_duration: Union[float, Fraction],
                 annotation: Dict[str, Any]) -> ClipInfo:
        pass

    def reset(self) -> None:
        """Forget the state of the current video before the next one."""


def make_clip_sampler(sampling_type: str, *args) -> ClipSampler:
    """The sampler named by ``sampling_type`` ("uniform", "random", "constant_clips_per_video" or "random_multi"),
    built from ``args``."""
    samplers = {"uniform": UniformClipSampler, "random": RandomClipSampler,
                "constant_clips_per_video": ConstantClipsPerVideoSampler, "random_multi": RandomMultiClipSampler}
    if sampling_type not in samplers:
        raise NotImplementedError(f"{sampling_type} not supported")
    return samplers[sampling_type](*args)


class UniformClipSampler(ClipSampler):
    """Consecutive clips of clip_duration seconds, each starting ``stride`` seconds after the previous one.

    With backpad_last the last clip is moved back so that it ends at the video's end; without it, the clips stop
    before one would run past the end.  ``eps`` is the tolerance of those end comparisons.
    """

    def __init__(self, clip_duration: Union[float, Fraction], stride: Optional[Union[float, Fraction]] = None,
                 backpad_last: bool = False, eps: float = 1e-6):
        super().__init__(clip_duration)
        self._stride = self._clip_duration if stride is None else stride
        self._eps = eps
        self._backpad_last = backpad_last
        assert self._stride > 0, "stride must be positive"

    def _clip_start_end(self, last_clip_end_time, video_duration, backpad_last: bool) -> Tuple[Fraction, Fraction]:
        # the next clip starts stride - clip_duration after the previous clip's end (at 0 for the first clip)
        delta = self._stride - self._clip_duration
        previous_end = -delta if last_clip_end_time is None else last_clip_end_time
        start = Fraction(previous_end + delta)
        end = Fraction(start + self._clip_duration)
        if backpad_last:
            start -= max(0, end - video_duration)
            start = Fraction(max(0, start))
            end = Fraction(start + self._clip_duration)
        return start, end

    def __call__(self, last_clip_end_time: Optional[float], video_duration: float,
                 annotation: Dict[str, Any]) -> ClipInfo:
        start, end = self._clip_start_end(last_clip_end_time, video_duration, self._backpad_last)
        _, following_end = self._clip_start_end(end, video_duration, self._backpad_last)
        if self._backpad_last:       # the following clip would be this one again
            is_last = abs(following_end - end) < self._eps
        else:                        # the following clip would run past the end
            is_last = (following_end - video_duration) > self._eps
        index = self._current_clip_index
        self._current_clip_index += 1
        if is_last:
            self.reset()
        return ClipInfo(start, end, index, 0, is_last)

    def reset(self):
        self._current_clip_index = 0


class UniformClipSamplerTruncateFromStart(UniformClipSampler):
    """``UniformClipSampler`` over the first truncation_duration seconds of each video (all of it when None)."""

    def __init__(self, clip_duration: Union[float, Fraction], stride: Optional[Union[float, Fraction]] = None,
                 backpad_last: bool = False, eps: float = 1e-6, truncation_duration: float = None) -> None:
        super().__init__(clip_duration, stride, backpad_last, eps)
        self.truncation_duration = truncation_duration

    def __call__(self, last_clip_end_time: float, video_duration: float, annotation: Dict[str, Any]) -> ClipInfo:
        if self.truncation_duration is not None:
            video_duration = min(self.truncation_duration, video_duration)
        return super().__call__(last_clip_end_time, video_duration, annotation)


class RandomClipSampler(ClipSampler):
    """One clip per video at a start drawn uniformly (``random.uniform``) from [0, duration - clip_duration]."""

    def __call__(self, last_clip_end_time: float, video_duration: float, annotation: Dict[str, Any]) -> ClipInfo:
        latest_start = max(video_duration - self._clip_duration, 0)
        start = Fraction(random.uniform(0, latest_start))
        return ClipInfo(start, start + self._clip_duration, 0, 0, True)


class RandomMultiClipSampler(RandomClipSampler):
    """num_clips clips per sample, each drawn as ``RandomClipSampler`` draws one."""

    def __init__(self, clip_duration: float, num_clips: int) -> None:
        super().__init__(clip_duration)
        self._num_clips = num_clips

    def __call__(self, last_clip_end_time: Optional[float], video_duration: float,
                 annotation: Dict[str, Any]) -> ClipInfoList:
        clips = [super(RandomMultiClipSampler, self).__call__(last_clip_end_time, video_duration, annotation)
                 for _ in range(self._num_clips)]
        return ClipInfoList(*([clip[k] for clip in clips] for k in range(len(ClipInfo._fields))))


class RandomMultiClipSamplerTruncateFromStart(RandomMultiClipSampler):
    """``RandomMultiClipSampler`` over the first truncation_duration seconds of each video (all of it when None)."""

    def __init__(self, clip_duration: float, num_clips: int, truncation_duration: float = None) -> None:
        super().__init__(clip_duration, num_clips)
        self.truncation_duration = truncation_duration

    def __call__(self, last_clip_end_time: Optional[float], video_duration: float,
                 annotation: Dict[str, Any]) -> ClipInfoList:
        if self.truncation_duration is not None:
            video_duration = min(self.truncation_duration, video_duration)
        return super().__call__(last_clip_end_time, video_duration, annotation)


class ConstantClipsPerVideoSampler(ClipSampler):
    """clips_per_video clips at evenly spaced starts in [0, duration - clip_duration], each returned augs_per_clip
    times with aug_index 0 .. augs_per_clip - 1."""

    def __init__(self, clip_duration: float, clips_per_video: int, augs_per_clip: int = 1) -> None:
        super().__init__(clip_duration)
        self._clips_per_video = clips_per_video
        self._augs_per_clip = augs_per_clip

    def __call__(self, last_clip_end_time: Optional[float], video_duration: float,
                 annotation: Dict[str, Any]) -> ClipInfo:
        latest_start = Fraction(max(video_duration - self._clip_duration, 0))
        spacing = Fraction(latest_start, max(self._clips_per_video - 1, 1))
        index, aug = self._current_clip_index, self._current_aug_index
        start = spacing * index
        self._current_aug_index += 1
        if self._current_aug_index >= self._augs_per_clip:
            self._current_aug_index = 0
            self._current_clip_index += 1
        # the last clip: clips_per_video clips are done, or the next start would lie past the latest start
        is_last = (self._current_clip_index >= self._clips_per_video
                   or spacing * self._current_clip_index > latest_start)
        if is_last:
            self.reset()
        return ClipInfo(start, start + self._clip_duration, index, aug, is_last)

    def reset(self):
        self._current_clip_index = 0
        self._current_aug_index = 0
