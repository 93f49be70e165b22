"""Sampling across DataLoader workers, and the two modes of the GPU datasets."""
import itertools
import logging

import numpy as np
import torch
import torch.utils.data

logger = logging.getLogger(__name__)


class MultiProcessSampler(torch.utils.data.Sampler):
    """Splits the indices of ``sampler`` evenly across the workers of a DataLoader, in contiguous runs: worker k of n
    iterates run k of ``np.array_split(range(len(sampler)), n)``.  Outside a worker it iterates all of them."""

    def __init__(self, sampler: torch.utils.data.Sampler) -> None:
        self._sampler = sampler

    def __iter__(self):
        info = torch.utils.data.get_worker_info()
        if info is None or info.num_workers == 0:
            return iter(self._sampler)
        run = np.array_split(range(len(self._sampler)), info.num_workers)[info.id]
        if len(run) == 0:
            logger.warning(f"More data workers({info.num_workers}) than videos({len(self._sampler)}). "
                           "For optimal use of processes reduce num_workers.")
            return iter(())
        return itertools.islice(iter(self._sampler), run[0], run[-1] + 1)


class GpuClipDataset:
    """The two modes shared by the frame-video datasets.

    In the normal mode a sample's ``"video"`` is the decoded clip on the current CUDA device and the dataset's
    ``transform`` runs on it.  That needs CUDA, which a forked DataLoader worker cannot use, so the normal mode refuses
    to run in a worker.  ``host_only()`` switches to the mode ``ClipBatchLoader`` runs in its workers: ``"video"`` is a
    ``ClipFrames`` record of the clip's file bytes, nothing is decoded, and ``transform`` is skipped.
    """

    _host_only = False
    _host_keep = None

    def host_only(self, keep=None):
        """Yield file bytes instead of decoded clips.  ``keep`` maps a clip's frame count to the positions to read
        (default: all).  Returns the dataset."""
        self._host_only, self._host_keep = True, keep
        return self

    def _check_process(self):
        if not self._host_only and torch.utils.data.get_worker_info() is not None:
            raise RuntimeError("%s decodes on the GPU, which a DataLoader worker process cannot use; iterate it "
                               "with pytorchvideo_b200.data.ClipBatchLoader, whose workers only read files"
                               % type(self).__name__)

    def _load_clip(self, video, start_sec, end_sec, frame_filter=None):
        """get_clip in the normal mode; in the host-only mode the same clip as a ClipFrames record."""
        if not self._host_only:
            return video.get_clip(start_sec, end_sec, frame_filter)
        frames = video.get_clip_frames(start_sec, end_sec, frame_filter, self._host_keep)
        return None if frames is None else {"video": frames, "frame_indices": frames.frame_indices, "audio": None}

    def _apply_transform(self, sample):
        if self._transform is None or self._host_only:
            return sample
        return self._transform(sample)
