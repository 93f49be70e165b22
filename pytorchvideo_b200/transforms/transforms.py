"""nn.Module wrappers with the reference's names (transforms/transforms.py) plus the fused chain.

``FusedClipTransform`` is the product: UniformTemporalSubsample -> /255 -> Normalize ->
ShortSideScale -> crop as ONE kernel launch reading uint8 frames (CTHW or the decoder's THWC
view) and writing the f16/f32 network input.  The single-op modules run the same kernel with
identity settings so that a torchvision ``Compose`` of them still works (one launch per op).
"""
import numpy as np
import torch
import torch.nn as nn

from .. import _lib as L
from . import functional as Fv
from .augment import AugMix, RandAugment  # noqa: F401


class ApplyTransformToKey:
    def __init__(self, key, transform):
        self._key = key
        self._transform = transform

    def __call__(self, x):
        x[self._key] = self._transform(x[self._key])
        return x


class UniformTemporalSubsample(nn.Module):
    def __init__(self, num_samples, temporal_dim=-3):
        super().__init__()
        self._num_samples = num_samples
        self._temporal_dim = temporal_dim

    def forward(self, x):
        return Fv.uniform_temporal_subsample(x, self._num_samples, self._temporal_dim)


class ShortSideScale(nn.Module):
    def __init__(self, size, interpolation="bilinear", backend="pytorch"):
        super().__init__()
        self._size, self._interpolation, self._backend = size, interpolation, backend

    def forward(self, x):
        return Fv.short_side_scale(x, self._size, self._interpolation, self._backend)


class RandomShortSideScale(nn.Module):
    def __init__(self, min_size, max_size, interpolation="bilinear", backend="pytorch"):
        super().__init__()
        self._min_size, self._max_size = min_size, max_size
        self._interpolation, self._backend = interpolation, backend

    def forward(self, x):
        size = torch.randint(self._min_size, self._max_size + 1, (1,)).item()
        return Fv.short_side_scale(x, size, self._interpolation, self._backend)


class Normalize(nn.Module):
    """(x - mean[c]) / std[c] on a CTHW clip (reference transforms.py:177-195)."""

    def __init__(self, mean, std, inplace=False):
        super().__init__()
        self.mean, self.std, self.inplace = list(mean), list(std), inplace

    def forward(self, x):
        if not x.is_floating_point():
            raise TypeError("Input tensor should be a float tensor. Got %s." % x.dtype)
        return Fv.clip_transform(x, mean=self.mean, std=self.std, out_dtype=x.dtype)


class Div255(nn.Module):
    def forward(self, x):
        return Fv.div_255(x)


class ConvertUint8ToFloat(nn.Module):
    def forward(self, x):
        assert x.dtype == torch.uint8, "image must have dtype torch.uint8"
        return Fv.clip_transform(x, div255=True)


class CenterCropVideo(nn.Module):
    """torchvision CenterCrop semantics on the last two dims (a view, no kernel)."""

    def __init__(self, size):
        super().__init__()
        self.size = size

    def forward(self, x):
        top, left, h, w = Fv.center_crop_window(x.shape[-2], x.shape[-1], self.size)
        return x[..., top:top + h, left:left + w]


class RandomCropVideo(nn.Module):
    """torchvision RandomCrop semantics (offsets from torch's global RNG on the host)."""

    def __init__(self, size):
        super().__init__()
        self.size = size

    def forward(self, x):
        top, left, h, w = Fv.random_crop_window(x.shape[-2], x.shape[-1], self.size)
        return x[..., top:top + h, left:left + w]


class UniformCropVideo(nn.Module):
    def __init__(self, size, video_key="video", aug_index_key="aug_index"):
        super().__init__()
        self._size, self._video_key, self._aug_index_key = size, video_key, aug_index_key

    def __call__(self, x):
        x[self._video_key] = Fv.uniform_crop(x[self._video_key], self._size, x[self._aug_index_key])
        return x


class RandomResizedCrop(nn.Module):
    """Reference RandomResizedCrop on float32 (C, T, H, W) clips, or (B, C, T, H, W) with one draw per clip."""

    def __init__(self, target_height, target_width, scale, aspect_ratio, shift=False, log_uniform_ratio=True,
                 interpolation="bilinear", num_tries=10):
        super().__init__()
        self._args = (target_height, target_width, scale, aspect_ratio, shift, log_uniform_ratio, interpolation,
                      num_tries)

    def forward(self, x):
        return Fv.random_resized_crop(x, *self._args)


class Permute(nn.Module):
    """x.permute(*dims): a view, which the augmentation and transform kernels read without a copy."""

    def __init__(self, dims):
        super().__init__()
        if sorted(dims) != list(range(len(dims))):
            raise ValueError("dims must contain every dimension (0, 1, 2, ...) once")
        self._dims = tuple(dims)

    def forward(self, x):
        return x.permute(*self._dims)


_RRC_KEYS = ("target_height", "target_width", "scale", "aspect_ratio", "shift", "log_uniform_ratio", "interpolation",
             "num_tries")


class FusedClipTransform(nn.Module):
    """One-kernel eval/train chain.  crop: None | ("center", size) | ("random", size) |
    ("uniform", size, spatial_idx).  Input: uint8 (or float) CUDA clip (C, T, H, W).

    random_resized_crop: dict of RandomResizedCrop's arguments (target_height, target_width, scale, aspect_ratio and
    optionally shift, log_uniform_ratio, interpolation, num_tries).  It replaces short_side / crop: frame selection,
    /255, normalisation, the random resized crop and the flip run as one launch; a batch draws per clip."""

    def __init__(self, num_samples=None, mean=None, std=None, short_side=None, crop=None, div255=True,
                 out_dtype=torch.float16, random_short_side=None, hflip_prob=0.0, slowfast_alpha=None,
                 random_resized_crop=None):
        super().__init__()
        if random_resized_crop is not None:
            unknown = set(random_resized_crop) - set(_RRC_KEYS)
            if unknown:
                raise ValueError("unknown random_resized_crop arguments %s" % sorted(unknown))
            if short_side is not None or crop is not None or random_short_side is not None or slowfast_alpha is not None:
                raise ValueError("random_resized_crop replaces short_side / random_short_side / crop and has no "
                                 "slow pathway output")
            if random_resized_crop.get("interpolation", "bilinear") != "bilinear":
                raise NotImplementedError("only bilinear RandomResizedCrop has a kernel")
        self.random_resized_crop = random_resized_crop
        self.num_samples, self.mean, self.std = num_samples, mean, std
        self.short_side, self.crop, self.div255, self.out_dtype = short_side, crop, div255, out_dtype
        self.random_short_side = random_short_side
        self.hflip_prob = float(hflip_prob)
        # emit [slow, fast] (SlowFastPackPathway, pytorchvideo_trainer datamodule/transforms.py:99-138) from the same pass
        self.slowfast_alpha = slowfast_alpha

    def plan(self, shape):
        """Host-side index/window/flip selection for an input of ``shape`` (C, T, H, W).  Random draws
        come from torch's global RNG in the order the reference's Compose makes them:
        RandomShortSideScale (randint), RandomCrop (randint i, randint j), RandomHorizontalFlip (rand)."""
        _, T, H, W = shape
        idx = None if self.num_samples is None else Fv.temporal_indices(T, self.num_samples)
        side = self.short_side
        if self.random_short_side is not None:
            lo, hi = self.random_short_side
            side = torch.randint(lo, hi + 1, (1,)).item()
        hw = None if side is None else Fv.short_side_size(H, W, side)
        nh, nw = (H, W) if hw is None else hw
        win = None
        if self.crop is not None:
            kind = self.crop[0]
            if kind == "center":
                win = Fv.center_crop_window(nh, nw, self.crop[1])
            elif kind == "random":
                win = Fv.random_crop_window(nh, nw, self.crop[1])
            elif kind == "uniform":
                win = Fv.uniform_crop_window(nh, nw, self.crop[1], self.crop[2])
            else:
                raise ValueError("unknown crop kind %r" % (kind,))
        flip = False
        if self.hflip_prob > 0.0:        # torchvision RandomHorizontalFlip.forward: torch.rand(1) < p
            flip = bool(torch.rand(1) < self.hflip_prob)
        return idx, hw, win, flip

    def _forward_rrc(self, x):
        rrc = dict(self.random_resized_crop)
        clips = x.unsqueeze(0) if x.dim() == 4 else x
        _, _, T, H, W = clips.shape
        idx = None if self.num_samples is None else Fv.temporal_indices(T, self.num_samples)
        n_t = T if idx is None else int(idx.numel())
        boxes, flips = [], []
        for _ in range(clips.shape[0]):      # per clip: the crop's draws, then the flip's
            boxes.append(Fv.random_resized_crop_boxes(n_t, H, W, rrc["scale"], rrc["aspect_ratio"],
                                                      rrc.get("shift", False), rrc.get("log_uniform_ratio", True),
                                                      rrc.get("num_tries", 10)))
            flips.append(bool(torch.rand(1) < self.hflip_prob) if self.hflip_prob > 0.0 else False)
        out = Fv.clip_transform_rrc(clips, boxes, (rrc["target_height"], rrc["target_width"]), frame_idx=idx,
                                    flips=flips, mean=self.mean, std=self.std, div255=self.div255,
                                    out_dtype=self.out_dtype)
        return out[0] if x.dim() == 4 else out

    def forward(self, x, out=None):
        """x: one clip (C, T, H, W) or a batch (B, C, T, H, W) - ONE launch either way (a batch in train mode
        draws short side / crop / flip per clip, in clip order).  Returns the clip(s), or [slow, fast] when
        ``slowfast_alpha`` is set."""
        if self.random_resized_crop is not None:
            if out is not None:
                raise ValueError("out= is not supported with random_resized_crop")
            return self._forward_rrc(x)
        if x.dim() == 5 and self._is_random():
            plans = [self.plan(x.shape[1:]) for _ in range(x.shape[0])]
            idx, hw, win, _ = plans[0]
            geom = [(p[1], p[2], p[3]) for p in plans]
            return Fv.clip_transform_batch(x, frame_idx=idx, resize_hw=hw, window=win, mean=self.mean, std=self.std,
                                           div255=self.div255, out_dtype=self.out_dtype, geom=geom,
                                           slow_alpha=self.slowfast_alpha, out=out)
        idx, hw, win, flip = self.plan(x.shape[-4:])
        return Fv.clip_transform_batch(x, frame_idx=idx, resize_hw=hw, window=win, mean=self.mean, std=self.std,
                                       div255=self.div255, out_dtype=self.out_dtype, hflip=flip,
                                       slow_alpha=self.slowfast_alpha, out=out)

    def _is_random(self):
        return self.random_short_side is not None or self.hflip_prob > 0.0 or (self.crop is not None and self.crop[0] == "random")


class FusedDetectionTransform(nn.Module):
    """The detection input chain on a batch of clips with ragged box lists: ONE pv_clip_transform_batch launch for the
    clips and ONE pv_clip_boxes_transform launch for the boxes and the RoI rows.

    Per clip, the output is what these reference calls give, in this order (transforms/functional.py, and the
    ``ava_inference_transform`` of the detection tutorial): uniform_temporal_subsample, /255, clip_boxes_to_image
    (source frame), [random_]short_side_scale_with_boxes, random_crop_with_boxes or uniform_crop_with_boxes
    (``crop``), horizontal_flip_with_boxes (``hflip_prob`` > 0), normalize, clip_boxes_to_image (output frame) and
    the slow / fast split.  With ``short_side`` and no crop this is ``ava_inference_transform``.

    crop: None | ("random", size) | ("uniform", size, spatial_idx).  The draws are the reference functions' own, per
    clip in clip order: torch.randint (random short side), np.random.randint for y then x (random crop, each only when
    that side is longer than the crop), np.random.uniform (flip), so a batch reproduces B sequential reference calls
    under the same torch and numpy seeds."""

    def __init__(self, num_samples, mean, std, short_side=None, random_short_side=None, crop=None, hflip_prob=0.0,
                 slowfast_alpha=None, div255=True, out_dtype=torch.float16):
        super().__init__()
        if short_side is not None and random_short_side is not None:
            raise ValueError("give short_side or random_short_side, not both")
        if crop is not None and not ((crop[0] == "random" and len(crop) == 2) or (crop[0] == "uniform" and len(crop) == 3)):
            raise ValueError("crop must be None, ('random', size) or ('uniform', size, spatial_idx) (got %r)" % (crop,))
        if crop is not None and crop[0] == "uniform" and crop[2] not in (0, 1, 2):
            raise ValueError("spatial_idx must be 0, 1 or 2")
        self.num_samples, self.mean, self.std = num_samples, mean, std
        self.short_side, self.random_short_side, self.crop = short_side, random_short_side, crop
        self.hflip_prob, self.slowfast_alpha = float(hflip_prob), slowfast_alpha
        self.div255, self.out_dtype = div255, out_dtype

    def plan(self, shape):
        """One clip's host draws for an input of ``shape`` (C, T, H, W): ((new_h, new_w), (top, left, out_h, out_w),
        flip)."""
        _, _, H, W = shape
        side = self.short_side
        if self.random_short_side is not None:
            lo, hi = self.random_short_side
            side = torch.randint(lo, hi + 1, (1,)).item()
        nh, nw = (H, W) if side is None else Fv.short_side_size(H, W, side)
        top, left, oh, ow = 0, 0, nh, nw
        if self.crop is not None and self.crop[0] == "random":
            size = self.crop[1]
            # A frame that already is size x size draws nothing and is not cropped.  Its boxes still take the crop's
            # clip at offset 0: clip, flip and the final clip give the boxes that flip and the final clip alone give.
            top, left = Fv.random_crop_offsets(nh, nw, size) or (0, 0)
            oh, ow = min(size, nh - top), min(size, nw - left)
        elif self.crop is not None:
            top, left, oh, ow = Fv.uniform_crop_window(nh, nw, self.crop[1], self.crop[2])
            if top < 0 or left < 0:
                raise RuntimeError("crop size %d larger than the %dx%d frame" % (self.crop[1], nh, nw))
        flip = bool(np.random.uniform() < self.hflip_prob) if self.hflip_prob > 0.0 else False
        return (nh, nw), (top, left, oh, ow), flip

    def box_steps(self):
        """The mask of _lib.BOX_* steps this chain runs on the boxes."""
        steps = L.BOX_CLIP_SRC | L.BOX_CLIP_OUT
        if self.short_side is not None or self.random_short_side is not None:
            steps |= L.BOX_SCALE
        if self.crop is not None:
            steps |= L.BOX_CROP | L.BOX_CLIP_CROP
        if self.hflip_prob > 0.0:
            steps |= L.BOX_FLIP
        return steps

    def _boxes(self, boxes, B, dev):
        """The box lists as one contiguous (K, 4) device tensor and the host offsets of each clip's rows."""
        if torch.is_tensor(boxes) or isinstance(boxes, np.ndarray):
            if B != 1:
                raise RuntimeError("a batch of %d clips needs a list of %d box arrays" % (B, B))
            boxes = [boxes]
        if not isinstance(boxes, (list, tuple)) or len(boxes) != B:
            raise RuntimeError("expected one (K, 4) box array per clip (%d clips)" % B)
        rows = [torch.from_numpy(b) if isinstance(b, np.ndarray) else b for b in boxes]
        for b in rows:
            if not torch.is_tensor(b) or b.dim() != 2 or b.shape[1] != 4:
                raise RuntimeError("every box array must be (K, 4) (x1, y1, x2, y2) rows")
        dtypes = set(b.dtype for b in rows)
        if len(dtypes) != 1 or rows[0].dtype not in Fv._BOX_DT:
            raise RuntimeError("boxes must all be float32 or all float64 (got %s)" % sorted(str(d) for d in dtypes))
        start = [0]
        for b in rows:
            start.append(start[-1] + int(b.shape[0]))
        if all(b.device.type == "cpu" for b in rows):
            flat = torch.cat(rows, 0).to(dev) if start[-1] else torch.empty((0, 4), dtype=rows[0].dtype, device=dev)
        else:
            flat = torch.empty((start[-1], 4), dtype=rows[0].dtype, device=dev)
            for b, s, e in zip(rows, start[:-1], start[1:]):
                flat[s:e].copy_(b)
        return flat.contiguous(), start

    def forward(self, clips, boxes):
        """clips: (C, T, H, W) or (B, C, T, H, W) uint8 / float32 CUDA clip(s), CTHW or the decoder's THWC-strided
        layout; boxes: a list of B (K_b, 4) arrays in source pixels (or one array for one clip).  Returns (inputs,
        rois): the clip batch, or [slow, fast], and the fp32 (sum K_b, 5) (clip, x1, y1, x2, y2) RoI rows."""
        if not torch.is_tensor(clips) or clips.dim() not in (4, 5):
            raise RuntimeError("expected a (C, T, H, W) or (B, C, T, H, W) clip tensor")
        if clips.device.type != "cuda":
            raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")
        x = clips.unsqueeze(0) if clips.dim() == 4 else clips
        B, _, T, H, W = x.shape
        dev = x.device
        flat, start = self._boxes(boxes, B, dev)
        plans = [self.plan(x.shape[1:]) for _ in range(B)]
        (oh, ow) = plans[0][1][2:]
        if any(p[1][2:] != (oh, ow) for p in plans):
            raise RuntimeError("the clips of a batch come out at different sizes (random short side without a crop?)")
        idx = Fv.temporal_indices(T, self.num_samples)
        geom = [(p[0], p[1], p[2]) for p in plans]
        inputs = Fv.clip_transform_batch(x, frame_idx=idx, resize_hw=plans[0][0], window=plans[0][1], mean=self.mean,
                                         std=self.std, div255=self.div255, out_dtype=self.out_dtype, geom=geom,
                                         slow_alpha=self.slowfast_alpha)
        if clips.dim() == 4:
            inputs = [t[0] for t in inputs] if self.slowfast_alpha is not None else inputs[0]
        steps = self.box_steps()
        if start[-1] == 0:
            return inputs, torch.empty((0, 5), dtype=torch.float32, device=dev)
        table = []
        for (nh, nw), (top, left, _, _), flip in plans:
            table += [nh, nw, top, left, 1 if flip else 0, 0]
        table = torch.tensor(table + start, dtype=torch.int32).to(dev)      # one copy: geometry, then offsets
        _, rois = Fv.clip_boxes_transform(flat, steps, in_hw=(H, W), out_hw=(oh, ow), n_clips=B,
                                          box_start=table[6 * B:], geom=table[:6 * B], rois=True)
        rois._pv_keepalive = (flat, table)
        return inputs, rois


class SlowFastPackPathway(nn.Module):
    """frames (C, T, H, W) or (B, C, T, H, W) -> [slow, fast]; slow = frames at linspace(0, T-1, T//alpha).long()
    (pytorchvideo_trainer/datamodule/transforms.py:99-138).  One gather launch; inside a FusedClipTransform the
    same list comes out of the transform kernel itself (``slowfast_alpha``)."""

    def __init__(self, alpha=4):
        super().__init__()
        self.alpha = alpha

    def forward(self, frames):
        out = Fv.clip_transform_batch(frames, out_dtype=frames.dtype, slow_alpha=self.alpha)
        return [out[0], frames]


class RemoveKey:
    """transforms.py:34-47: drops ``key`` from a dict sample."""

    def __init__(self, key):
        self._key = key

    def __call__(self, x):
        if self._key in x:
            del x[self._key]
        return x


class _Chain:
    """Minimal torchvision ``Compose`` (dict-level steps around the fused clip transform)."""

    def __init__(self, steps):
        self.transforms = list(steps)

    def __call__(self, x):
        for t in self.transforms:
            x = t(x)
        return x


def create_video_transform(mode, video_key=None, remove_key=None, num_samples=8, convert_to_float=True,
                           video_mean=(0.45, 0.45, 0.45), video_std=(0.225, 0.225, 0.225), min_size=256,
                           max_size=320, crop_size=224, horizontal_flip_prob=0.5, aug_type="default",
                           aug_paras=None, random_resized_crop_paras=None, out_dtype=torch.float16):
    """Fused equivalent of the reference factory's default chains (transforms_factory.py:109-284), same
    signature and argument checks:
      train = subsample, /255, normalize, RandomShortSideScale(min,max), RandomCrop, RandomHorizontalFlip(p)
      val   = subsample, /255, normalize, ShortSideScale(min_size), CenterCrop
    as ONE kernel launch.  RandAugment / AugMix (aug_type) and RandomResizedCrop have no B200 kernel:
    asking for them raises NotImplementedError instead of silently changing the augmentation."""
    if mode not in ("train", "val"):
        raise NotImplementedError("mode must be 'train' or 'val'")
    if isinstance(crop_size, int):
        assert crop_size <= min_size, "crop_size must be less than or equal to min_size"
    elif isinstance(crop_size, tuple):
        assert max(crop_size) <= min_size, "the height and width in crop_size must be less than or equal to min_size"
    else:
        raise TypeError
    if video_key is None:
        assert remove_key is None, "remove_key should be None if video_key is None"
    if aug_type == "default":
        assert aug_paras is None, "aug_paras should be None for ``default`` aug_type"
    elif aug_type in ("randaug", "augmix"):
        if mode == "train":
            raise NotImplementedError("aug_type=%r has no B200 kernel (only the 'default' chain is fused)" % aug_type)
    else:
        raise NotImplementedError
    if random_resized_crop_paras is not None and mode == "train":
        raise NotImplementedError("RandomResizedCrop has no B200 kernel (use RandomShortSideScale + RandomCrop)")
    if mode == "val":
        tr = FusedClipTransform(num_samples, video_mean, video_std, short_side=min_size,
                                crop=("center", crop_size), div255=convert_to_float, out_dtype=out_dtype)
    else:
        tr = FusedClipTransform(num_samples, video_mean, video_std, crop=("random", crop_size),
                                div255=convert_to_float, out_dtype=out_dtype,
                                random_short_side=(min_size, max_size), hflip_prob=horizontal_flip_prob)
    if video_key is None:
        return tr
    return _Chain([ApplyTransformToKey(key=video_key, transform=tr)] +
                  ([] if remove_key is None else [RemoveKey(k) for k in remove_key]))
