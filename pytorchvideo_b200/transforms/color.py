"""The contrastive-learning view augmentations of the trainer's SimCLR / BYOL recipes on the GPU
(pytorchvideo_trainer/datamodule/transforms.py: ColorJitterVideoSSl, GaussianBlur, RepeatandConverttoList,
ApplyTransformToKeyOnList; conf/datamodule/transforms/kinetics_contrastive.yaml).

The reference runs ColorJitterVideoSSl in PIL on the CPU: the clip becomes one tall (T*H, W) RGB image, which goes
through torchvision's ColorJitter (in a random order), RandomGrayscale and Pillow's GaussianBlur.  Here the host makes
the reference's random draws with its own calls in its order, encodes each view as one ``pv_cj_view`` and the whole
batch runs in three launches (pv_colorjitter_stats / _apply / _vblur) in Pillow's integer and float arithmetic, so the
bytes are the reference's.  ``FusedContrastiveTransform`` adds the recipe's Normalize, RandomResizedCrop and
RandomHorizontalFlip through pv_clip_transform_rrc.
"""
import ctypes as C
import numbers
import random

import numpy as np
import torch

from .. import _lib as L
from . import functional as Fv


def _check_input(value, name, center=1, bound=(0, float("inf")), clip_first_on_zero=True):
    """torchvision ColorJitter._check_input: the (min, max) factor range, or None when the op does nothing."""
    if isinstance(value, numbers.Number):
        if value < 0:
            raise ValueError(f"If {name} is a single number, it must be non negative.")
        value = [center - float(value), center + float(value)]
        if clip_first_on_zero:
            value[0] = max(value[0], 0.0)
    elif isinstance(value, (tuple, list)) and len(value) == 2:
        value = [float(value[0]), float(value[1])]
    else:
        raise TypeError(f"{name} should be a single number or a list/tuple with length 2.")
    if not bound[0] <= value[0] <= value[1] <= bound[1]:
        raise ValueError(f"{name} values should be between {bound}, but got {value}.")
    if value[0] == value[1] == center:
        return None
    return tuple(value)


def box_blur_params(sigma, passes=3):
    """(integer radius, ww, fw) of Pillow's GaussianBlur(radius=sigma), or None when it leaves the image as it is.

    Pillow blurs with `passes` extended box filters of variance sigma**2 / passes: a fractional box radius computed in
    C float with some double steps, then 2**24 / (2 * radius + 1) as the window weight and the rest split over the two
    pixels just outside the window."""
    f32 = np.float32
    if float(sigma) == 0.0:
        return None
    s = f32(sigma)
    sigma2 = f32(f32(s * s) / f32(passes))
    length = f32(np.sqrt(12.0 * np.float64(sigma2) + 1.0))
    lo = f32(np.floor((np.float64(length) - 1.0) / 2.0))
    a = f32(f32(f32(2) * lo + f32(1)) * f32(lo * f32(lo + f32(1)) - f32(3) * sigma2))
    a = f32(a / f32(f32(6) * f32(sigma2 - f32(lo + f32(1)) * f32(lo + f32(1)))))
    radius = f32(lo + a)
    if radius == 0:
        return None
    r = int(radius)
    ww = int(f32(f32(1 << 24) / f32(radius * f32(2) + f32(1))))
    return r, ww, ((1 << 24) - (2 * r + 1) * ww) // 2


class ViewDraw:
    """One view's ColorJitterVideoSSl draws.  order: the applied op ids (0 brightness, 1 contrast, 2 saturation,
    3 hue) in the drawn permutation (empty when the jitter was skipped); factors: the drawn (b, c, s, h), None for an
    op with nothing to draw; sigma: the blur's sigma, None when the blur was skipped."""

    __slots__ = ("jitter", "perm", "factors", "order", "gray", "sigma")

    def __init__(self, jitter, perm, factors, gray, sigma):
        self.jitter, self.perm, self.factors, self.gray, self.sigma = jitter, perm, factors, gray, sigma
        self.order = [i for i in perm if factors[i] is not None] if jitter else []

    def as_dict(self):
        return {"jitter": self.jitter, "perm": list(self.perm), "factors": list(self.factors), "gray": self.gray,
                "sigma": self.sigma}


def _hue_shift(hue_factor):
    """torchvision adjust_hue's byte offset: np.int32(hue_factor * 255).astype(np.uint8)."""
    return int(np.int32(hue_factor * 255).astype(np.uint8))


def _encode(views, clips):
    """The device table: one pv_cj_view per (draw, source clip)."""
    arr = (L.CjView * len(views))()
    for e, v, clip in zip(arr, views, clips):
        e.clip, e.n_ops = int(clip), len(v.order)
        for i, op in enumerate(v.order):
            e.ops[i] = op
        for i in range(3):
            e.factor[i] = v.factors[i] if v.factors[i] is not None else 1.0
        e.hue_shift = _hue_shift(v.factors[3]) if v.factors[3] is not None else 0
        e.gray = 1 if v.gray else 0
        blur = None if v.sigma is None else box_blur_params(v.sigma)
        e.blur_r, e.blur_ww, e.blur_fw = (-1, 0, 0) if blur is None else blur
    return arr


STAGES = ("stats", "apply", "vblur")


def plan_views(x, views, clips, frame_idx=None, src_scale=0):
    """Descriptor, device tables and output of color_jitter_views, without launching anything."""
    B, Cc, T, H, W = x.shape
    if Cc != 3:
        raise RuntimeError("ColorJitterVideoSSl needs 3-channel clips (got %d)" % Cc)
    if x.dtype not in (torch.uint8, torch.float32):
        raise RuntimeError("ColorJitterVideoSSl reads uint8 or float32 clips (got %s)" % x.dtype)
    idx = torch.arange(T) if frame_idx is None else torch.as_tensor(frame_idx).long().cpu()
    if idx.numel() == 0 or int(idx.min()) < 0 or int(idx.max()) >= T:
        raise RuntimeError("frame index out of range")
    if any(not 0 <= int(c) < B for c in clips):
        raise RuntimeError("view source clip out of range")
    n_t, n = int(idx.numel()), len(views)
    dev = x.device
    d = L.ColorJitterDesc()
    d.n_views, d.n_t, d.H, d.W = n, n_t, H, W
    d.s_clip, d.sc, d.st, d.sh, d.sw = (x.stride(i) for i in range(5))
    d.src_dtype = L.PV_U8 if x.dtype == torch.uint8 else L.PV_F32
    d.src_scale = int(src_scale)
    table = torch.frombuffer(bytearray(bytes(_encode(views, clips))), dtype=torch.uint8)
    views_d = table.pin_memory().to(dev, non_blocking=True)     # pinned: the copy does not wait for the stream
    return {"desc": d, "x": x, "views": views_d, "idx": Fv._dev_i32(idx.tolist(), dev),
            "sums": torch.empty(n, dtype=torch.int64, device=dev),
            "out": torch.empty((n, 3, n_t, H, W), dtype=torch.uint8, device=dev)}


def launch_stage(p, stage):
    """One of the three launches (STAGES) of a plan_views plan, on the current stream."""
    lib = L.load()
    d, x, out = p["desc"], p["x"], p["out"]
    stream = torch.cuda.current_stream(x.device).cuda_stream
    if stage == "stats":
        L.check(lib.pv_colorjitter_stats(C.byref(d), x.data_ptr(), p["idx"].data_ptr(), p["views"].data_ptr(),
                                         p["sums"].data_ptr(), stream), "pv_colorjitter_stats")
    elif stage == "apply":
        L.check(lib.pv_colorjitter_apply(C.byref(d), x.data_ptr(), p["idx"].data_ptr(), p["views"].data_ptr(),
                                         p["sums"].data_ptr(), out.data_ptr(), stream), "pv_colorjitter_apply")
    else:
        L.check(lib.pv_colorjitter_vblur(C.byref(d), p["views"].data_ptr(), out.data_ptr(), stream),
                "pv_colorjitter_vblur")


def color_jitter_views(x, views, clips, frame_idx=None, src_scale=0):
    """Run ``views`` (ViewDraw list) on the (B, 3, T, H, W) CUDA clips ``x`` (uint8, or float32 in [0, 1] with
    src_scale 0 / 0..255 with src_scale 1; any strides).  View k reads the frames ``frame_idx`` of clip ``clips[k]``.
    Returns the contiguous uint8 (len(views), 3, n_t, H, W) views."""
    p = plan_views(x, views, clips, frame_idx, src_scale)
    for stage in STAGES:
        launch_stage(p, stage)
    out = p["out"]
    out._pv_keepalive = (p["views"], p["idx"], p["sums"])     # device tables of the asynchronous launches
    return out


def _check_batch(x, what):
    if not torch.is_tensor(x) or x.dim() not in (4, 5):
        raise RuntimeError("%s expects a (C, T, H, W) clip or a (B, C, T, H, W) batch" % what)
    if x.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")
    return x.unsqueeze(0) if x.dim() == 4 else x


class ColorJitterVideoSSl:
    """Random colour jitter, grayscale and Gaussian blur of a clip (the trainer's ColorJitterVideoSSl), on the GPU.

    Input: a float32 CUDA clip (C, T, H, W) in [0, 1] (after Div255), or a batch (B, C, T, H, W) with one draw per clip
    in clip order.  Output: float32 of the same shape, the values u / 255 that the reference's ToTensor gives.  The draws
    are the reference's own calls under torch's and Python's global RNGs: RandomApply (torch.rand), ColorJitter's
    torch.randperm and torch.empty(1).uniform_ per op, RandomGrayscale (torch.rand), the blur's RandomApply
    (torch.rand) and random.uniform for its sigma."""

    def __init__(self, bri_con_sat, hue, p_color_jitter, p_convert_gray, p_gaussian_blur=0.5,
                 gaussian_blur_sigma=(0.1, 2.0)):
        self.brightness = _check_input(bri_con_sat[0], "brightness")
        self.contrast = _check_input(bri_con_sat[1], "contrast")
        self.saturation = _check_input(bri_con_sat[2], "saturation")
        self.hue = _check_input(hue, "hue", center=0, bound=(-0.5, 0.5), clip_first_on_zero=False)
        self.p_color_jitter, self.p_convert_gray, self.p_gaussian_blur = p_color_jitter, p_convert_gray, p_gaussian_blur
        self.sigma = gaussian_blur_sigma

    def sample(self):
        """One view's draws (ViewDraw), in the reference's order."""
        jitter, perm, factors = False, [0, 1, 2, 3], [None] * 4
        if not self.p_color_jitter < torch.rand(1):          # RandomApply: skipped when p < rand
            jitter = True
            perm = [int(i) for i in torch.randperm(4)]
            factors = [None if rng is None else float(torch.empty(1).uniform_(rng[0], rng[1]))
                       for rng in (self.brightness, self.contrast, self.saturation, self.hue)]
        gray = bool(torch.rand(1) < self.p_convert_gray)
        sigma = None
        if not self.p_gaussian_blur < torch.rand(1):
            sigma = self.sigma[0]
            if len(self.sigma) == 2:
                sigma = random.uniform(self.sigma[0], self.sigma[1])
        return ViewDraw(jitter, perm, factors, gray, sigma)

    def __call__(self, frames):
        x = _check_batch(frames, "ColorJitterVideoSSl")
        if x.dtype != torch.float32:
            raise RuntimeError("ColorJitterVideoSSl takes float32 clips in [0, 1] (got %s)" % x.dtype)
        B = x.shape[0]
        views = [self.sample() for _ in range(B)]
        u8 = color_jitter_views(x, views, list(range(B)))
        out = Fv.clip_transform_batch(u8, div255=True, out_dtype=torch.float32)     # ToTensor: u / 255 in fp32
        out._pv_keepalive = (u8, getattr(out, "_pv_keepalive", None))
        return out[0] if frames.dim() == 4 else out


class RepeatandConverttoList:
    """Replaces every value of a dict sample with a list of ``repeat_num`` references to it (the trainer's
    RepeatandConverttoList): the views of a contrastive recipe start from the same clip."""

    def __init__(self, repeat_num):
        self.repeat_num = repeat_num

    def __call__(self, sample_dict):
        for k, v in sample_dict.items():
            sample_dict[k] = self.repeat_num * [v]
        return sample_dict


class ApplyTransformToKeyOnList:
    """Applies ``transform`` to every element of the list under ``key`` (the trainer's ApplyTransformToKeyOnList)."""

    def __init__(self, key, transform):
        self._key = key
        self._transform = transform

    def __call__(self, x):
        x[self._key] = [self._transform(a) for a in x[self._key]]
        return x


class FusedContrastiveTransform:
    """The contrastive train chain of the trainer's SimCLR / BYOL recipes for a batch of clips, per view:
    UniformTemporalSubsample(num_samples) -> Div255 -> ColorJitterVideoSSl -> Normalize(mean, std) ->
    RandomResizedCrop(target_height, target_width, scale, aspect_ratio, ...) -> RandomHorizontalFlip(hflip_prob).

    Input: (B, C, T, H, W) uint8 or float32 0..255 CUDA clips, CTHW or the decoder's THWC-strided view.  Output: a list
    of ``num_views`` (B, 3, num_samples, target_height, target_width) tensors of ``out_dtype``, as SimCLR.forward(x1, x2)
    and BYOL.forward(x1, x2) take them.  The draws are those of B sequential reference calls (clip-major, then view):
    ColorJitterVideoSSl's, then RandomResizedCrop's, then the flip's torch.rand.  Four launches per batch whatever B and
    num_views: the three colour kernels and one pv_clip_transform_rrc."""

    def __init__(self, num_samples, mean, std, bri_con_sat, hue, p_color_jitter, p_convert_gray, target_height,
                 target_width, scale, aspect_ratio, p_gaussian_blur=0.5, gaussian_blur_sigma=(0.1, 2.0),
                 shift=False, log_uniform_ratio=True, interpolation="bilinear", num_tries=10, hflip_prob=0.5,
                 num_views=2, out_dtype=torch.float16):
        if interpolation != "bilinear":
            raise NotImplementedError("only bilinear RandomResizedCrop has a kernel (got %r)" % (interpolation,))
        if num_views < 1:
            raise ValueError("num_views must be at least 1")
        self.num_samples, self.mean, self.std = num_samples, mean, std
        self.jitter = ColorJitterVideoSSl(bri_con_sat, hue, p_color_jitter, p_convert_gray, p_gaussian_blur,
                                          gaussian_blur_sigma)
        self.target_hw = (int(target_height), int(target_width))
        self.rrc = (scale, aspect_ratio, shift, log_uniform_ratio, num_tries)
        self.hflip_prob, self.num_views, self.out_dtype = float(hflip_prob), int(num_views), out_dtype

    def sample(self, n_t, H, W):
        """One view's draws: (ViewDraw, per-frame crop boxes, flip)."""
        view = self.jitter.sample()
        scale, ratio, shift, log_uniform, tries = self.rrc
        boxes = Fv.random_resized_crop_boxes(n_t, H, W, scale, ratio, shift, log_uniform, tries)
        flip = bool(torch.rand(1) < self.hflip_prob)
        return view, boxes, flip

    def __call__(self, clips):
        x = _check_batch(clips, "FusedContrastiveTransform")
        if x.dtype not in (torch.uint8, torch.float32):
            raise RuntimeError("FusedContrastiveTransform reads uint8 or float32 0..255 clips (got %s)" % x.dtype)
        B, _, T, H, W = x.shape
        idx = Fv.temporal_indices(T, self.num_samples)
        n_t, V = int(idx.numel()), self.num_views
        draws = [[self.sample(n_t, H, W) for _ in range(V)] for _ in range(B)]
        # stored view-major (view v of clip b at v * B + b) so that each view's batch is one contiguous slice
        order = [(b, v) for v in range(V) for b in range(B)]
        u8 = color_jitter_views(x, [draws[b][v][0] for b, v in order], [b for b, _ in order], frame_idx=idx,
                                src_scale=1)
        out = Fv.clip_transform_rrc(u8, [draws[b][v][1] for b, v in order], self.target_hw,
                                    flips=[draws[b][v][2] for b, v in order], mean=self.mean, std=self.std,
                                    div255=True, out_dtype=self.out_dtype)
        out._pv_keepalive = (u8, out._pv_keepalive)
        return [out[v * B:(v + 1) * B] for v in range(V)]
