"""Test-time multi-view inference: K temporal clips x 3 spatial crops of one video, ensembled on device.

Reference pipeline (docs/source/model_zoo.md:63 "3 spatial x 10 temporal views"; data/clip_sampling.py:343-410
ConstantClipsPerVideoSampler; transforms/transforms.py:153-174 UniformCropVideo with
transforms/functional.py:302-347 uniform_crop; pytorchvideo_trainer module/video_classification.py:290-311
_ensemble_at_video_level): every view is decoded, transformed, pushed through the model on its own and the
per-clip predictions are accumulated per video id on the host side of the training loop.

Here the decoded uint8 video stays on the GPU and ALL views come out of ONE launch of the fused transform
kernel (the video is a batch with clip stride 0; each view has its own first frame and crop window), go through
the model as one batch of K*3 clips, and one small kernel reduces the [K*3, classes] predictions.
"""
import ctypes as C
from fractions import Fraction

import torch

from . import _lib as L
from .transforms import functional as Fv


def clip_start_frames(n_frames, clip_frames, clips_per_video):
    """ConstantClipsPerVideoSampler (clip_sampling.py:375-379) in frame units: clip i starts at
    i * max(n_frames - clip_frames, 0) / max(clips_per_video - 1, 1), rounded down to a frame."""
    last = Fraction(max(n_frames - clip_frames, 0))
    step = last / max(clips_per_video - 1, 1)
    return [int(step * i) for i in range(clips_per_video)]


def view_reduce(preds, n_views, mode="sum"):
    """[n_videos * n_views, K] f32 CUDA predictions -> [n_videos, K]; mode: "sum" | "mean" | "max"
    (video_classification.py:303-311; "mean" = the sum divided by the clip count of :279-282).

    "sum" and "max" are the reference's per-video accumulators: it starts each video from zeros and adds or
    torch.max-es the views in order, so "max" is max(0, max_i p_i) and a NaN in any view propagates.  At the end of
    the test epoch the reference divides either accumulator by the clip count (:279-282); for "max" that division is
    left to the caller."""
    if preds.device.type != "cuda" or preds.dtype != torch.float32 or preds.dim() != 2 or not preds.is_contiguous():
        raise RuntimeError("view_reduce expects a contiguous f32 CUDA tensor [n_videos * n_views, classes]")
    if preds.shape[0] % n_views:
        raise RuntimeError("%d rows are not a multiple of %d views" % (preds.shape[0], n_views))
    n_videos = preds.shape[0] // n_views
    out = torch.empty((n_videos, preds.shape[1]), dtype=torch.float32, device=preds.device)
    code = {"sum": 0, "mean": 1, "max": 2}[mode]
    L.check(L.load().pv_view_reduce(preds.data_ptr(), out.data_ptr(), n_videos, n_views, preds.shape[1], code,
                                    torch.cuda.current_stream(preds.device).cuda_stream), "pv_view_reduce")
    return out


class MultiViewEnsemble(torch.nn.Module):
    """``forward(video_u8)``: (C, T, H, W) uint8 CUDA video -> [classes] ensembled prediction.

    model          : a pytorchvideo_b200 model (SlowFast models get [slow, fast] from the same transform pass)
    clip_frames    : frames of the video covered by one temporal clip (clip_duration * fps)
    num_samples    : frames the model sees per clip (UniformTemporalSubsample inside the clip)
    clips_per_video / crops: the K x 3 views; crops are uniform_crop spatial indices 0..2
    """

    def __init__(self, model, clip_frames, num_samples, clips_per_video=10, crops=3, side_size=256, crop_size=256,
                 mean=(0.45, 0.45, 0.45), std=(0.225, 0.225, 0.225), slowfast_alpha=None, ensemble="sum",
                 out_dtype=torch.float16):
        super().__init__()
        assert crops in (1, 3) and ensemble in ("sum", "mean", "max")
        self.model = model
        self.clip_frames, self.num_samples = int(clip_frames), int(num_samples)
        self.clips_per_video, self.crops = int(clips_per_video), int(crops)
        self.side_size, self.crop_size = int(side_size), int(crop_size)
        self.mean, self.std = mean, std
        self.slowfast_alpha, self.ensemble, self.out_dtype = slowfast_alpha, ensemble, out_dtype

    def views(self, shape):
        """Per view: (resize_hw, crop window, flip, first frame), temporal clips outermost like the sampler."""
        _, T, H, W = shape
        hw = Fv.short_side_size(H, W, self.side_size)
        spatial = (1,) if self.crops == 1 else (0, 1, 2)
        out = []
        for start in clip_start_frames(T, self.clip_frames, self.clips_per_video):
            for s in spatial:
                out.append((hw, Fv.uniform_crop_window(hw[0], hw[1], self.crop_size, s), False, start))
        return hw, out

    def make_views(self, video):
        if video.dim() != 4 or video.device.type != "cuda":
            raise RuntimeError("expected a (C, T, H, W) CUDA video")
        if video.shape[1] < self.clip_frames:
            raise RuntimeError("video shorter (%d frames) than one clip (%d)" % (video.shape[1], self.clip_frames))
        hw, views = self.views(video.shape)
        idx = Fv.temporal_indices(self.clip_frames, self.num_samples)      # inside a clip
        batch = video.unsqueeze(0).expand(len(views), -1, -1, -1, -1)      # clip stride 0: every view reads the same frames
        return Fv.clip_transform_batch(batch, frame_idx=idx, resize_hw=hw, window=views[0][1], mean=self.mean, std=self.std,
                                       div255=video.dtype == torch.uint8, out_dtype=self.out_dtype, geom=views,
                                       slow_alpha=self.slowfast_alpha)

    def forward(self, video):
        x = self.make_views(video)
        preds = self.model(x).float().contiguous()
        return view_reduce(preds, preds.shape[0], self.ensemble)[0]
