"""ORACLE (test infrastructure only): numpy restatement of the reference's clip transform chain.

Integer/index work is bit-exact by construction and pinned against the reference's known-answer
tests (tests/test_transforms.py:85-102, :199-226, :334-346 of the reference; see
tests/test_oracle_pinning.py) and against golden vectors produced by the reference itself
(oracle/gen_golden.py).  Floating point follows the reference op order in fp32.
"""
import math

import numpy as np


def linspace_indices(t, num_samples):
    """transforms/functional.py:36-40: clamp(torch.linspace(0, t-1, n), 0, t-1).long().

    torch.linspace (ATen CPU, float32) evaluates symmetrically: element i < n//2 is
    start + step*i, the others end - step*(n-1-i), the latter as ONE fused multiply-add.  With
    that detail this restatement agrees with torch.linspace on all (t<=300, n<=128) cases
    (a naive i*(t-1)/(n-1) does not - SURVEY section 7, hard part 4)."""
    assert num_samples > 0 and t > 0
    start, end = np.float32(0), np.float32(t - 1)
    if num_samples == 1:
        vals = np.array([start], np.float32)
    else:
        step = np.float32((end - start) / np.float32(num_samples - 1))
        i = np.arange(num_samples)
        lo = (np.float64(step) * i).astype(np.float32)                 # start == 0
        hi = (np.float64(end) - np.float64(step) * (num_samples - 1 - i)).astype(np.float32)  # fma
        vals = np.where(i < num_samples // 2, lo, hi)
    return np.clip(vals, 0, t - 1).astype(np.int64)


def uniform_temporal_subsample(x, num_samples, temporal_dim=-3):
    """functional.py:19-41 (index_select along the temporal dim)."""
    idx = linspace_indices(x.shape[temporal_dim], num_samples)
    return np.take(x, idx, axis=temporal_dim)


def uniform_temporal_subsample_repeated(frames, frame_ratios, temporal_dim=-3):
    """functional.py:134-160."""
    t = frames.shape[temporal_dim]
    return [uniform_temporal_subsample(frames, t // r, temporal_dim) for r in frame_ratios]


def short_side_size(h, w, size):
    """functional.py:118-123."""
    if w < h:
        return int(math.floor((float(h) / w) * size)), size
    return size, int(math.floor((float(w) / h) * size))


def bilinear_table(in_size, out_size):
    """ATen upsample_bilinear2d (align_corners=False, no antialias) source indices and weights:
    scale = in/out (fp32); src = fma(scale, dst+0.5, -0.5) clamped at 0; i0 = min(floor(src),
    in-1); i1 = i0 + (i0 < in-1); lambda1 = clamp(src - i0, 0, 1); identity when sizes match.
    Returns (i0, i1, lambda1) with dtypes (int32, int32, float32)."""
    if in_size == out_size:
        i = np.arange(out_size, dtype=np.int32)
        return i, i.copy(), np.zeros(out_size, np.float32)
    scale = np.float32(in_size) / np.float32(out_size)
    d = np.arange(out_size, dtype=np.float32) + np.float32(0.5)
    # fma(scale, d, -0.5) with one rounding; astype, not np.float64(d), which turns a one-element array (out_size 1)
    # into a scalar
    src = (np.float64(scale) * d.astype(np.float64) - 0.5).astype(np.float32)
    src = np.maximum(src, np.float32(0))
    i0 = np.minimum(np.floor(src).astype(np.int64), in_size - 1)
    l1 = np.clip(src - i0.astype(np.float32), np.float32(0), np.float32(1)).astype(np.float32)
    i1 = i0 + (i0 < in_size - 1)
    return i0.astype(np.int32), i1.astype(np.int32), l1


def bilinear_resize(x, out_h, out_w):
    """F.interpolate(x, size=(out_h,out_w), mode='bilinear', align_corners=False) on (...,H,W) fp32:
    l_h0*(l_w0*v00 + l_w1*v01) + l_h1*(l_w0*v10 + l_w1*v11)."""
    x = np.asarray(x, np.float32)
    y0, y1, ly = bilinear_table(x.shape[-2], out_h)
    x0, x1, lx = bilinear_table(x.shape[-1], out_w)
    ly1 = ly[:, None]
    ly0 = np.float32(1) - ly1
    lx1 = lx[None, :]
    lx0 = np.float32(1) - lx1
    r0, r1 = x[..., y0, :], x[..., y1, :]
    top = lx0 * r0[..., x0] + lx1 * r0[..., x1]
    bot = lx0 * r1[..., x0] + lx1 * r1[..., x1]
    return (ly0 * top + ly1 * bot).astype(np.float32)


def short_side_scale(x, size):
    """functional.py:92-131 (pytorch backend, bilinear)."""
    assert x.ndim == 4 and x.dtype == np.float32
    new_h, new_w = short_side_size(x.shape[2], x.shape[3], size)
    return bilinear_resize(x, new_h, new_w)


def div_255(x):
    """functional.py:604-615: x / 255.0 (fp32)."""
    return (np.asarray(x, np.float32) / np.float32(255.0)).astype(np.float32)


def normalize(x, mean, std):
    """transforms.py:177-195 -> torchvision Normalize: (x - mean[c]) / std[c] per channel of CTHW."""
    mean = np.asarray(mean, np.float32).reshape(-1, 1, 1, 1)
    std = np.asarray(std, np.float32).reshape(-1, 1, 1, 1)
    return ((np.asarray(x, np.float32) - mean) / std).astype(np.float32)


def center_crop_window(h, w, size):
    """torchvision CenterCrop window for an (h, w) image and a square/int size."""
    th, tw = (size, size) if isinstance(size, int) else size
    top = int(round((h - th) / 2.0))
    left = int(round((w - tw) / 2.0))
    return top, left, th, tw


def uniform_crop_window(h, w, size, spatial_idx):
    """functional.py:302-325 (_uniform_crop_helper offsets)."""
    assert spatial_idx in (0, 1, 2)
    y = int(math.ceil((h - size) / 2))
    x = int(math.ceil((w - size) / 2))
    if h > w:
        if spatial_idx == 0:
            y = 0
        elif spatial_idx == 2:
            y = h - size
    else:
        if spatial_idx == 0:
            x = 0
        elif spatial_idx == 2:
            x = w - size
    return y, x, size, size


def val_chain(clip_u8, num_samples, mean, std, side, crop):
    """The canonical eval chain in the reference's order (transforms_factory.py:229-261):
    UniformTemporalSubsample -> /255 -> Normalize -> ShortSideScale -> CenterCrop.  CTHW in."""
    x = uniform_temporal_subsample(clip_u8, num_samples)
    x = div_255(x)
    x = normalize(x, mean, std)
    x = short_side_scale(x, side)
    if crop is not None:
        top, left, th, tw = center_crop_window(x.shape[2], x.shape[3], crop)
        x = x[:, :, top:top + th, left:left + tw]
    return x


def random_crop_window(h, w, size, i, j):
    """torchvision RandomCrop.get_params (transforms_factory.py:251 uses torchvision's class): the window is
    (i, j, th, tw) with i ~ randint(0, h-th+1), j ~ randint(0, w-tw+1) drawn by the caller from torch's global
    RNG in that order; no draw at all when the image already has the crop size."""
    th, tw = (size, size) if isinstance(size, int) else size
    if h < th or w < tw:
        raise ValueError("Required crop size %s is larger than input image size %s" % ((th, tw), (h, w)))
    if w == tw and h == th:
        return 0, 0, h, w
    return int(i), int(j), th, tw


def train_chain(clip_u8, num_samples, mean, std, side, crop, i, j, flip):
    """The default train chain in the reference's order (transforms_factory.py:229-258, aug_type "default",
    no RandomResizedCrop): UniformTemporalSubsample -> /255 -> Normalize -> RandomShortSideScale(side drawn by
    the caller: torch.randint(min, max+1, (1,)), transforms.py:148) -> RandomCrop(i, j) ->
    RandomHorizontalFlip (flip = torch.rand(1) < p, torchvision).  CTHW in."""
    x = uniform_temporal_subsample(clip_u8, num_samples)
    x = div_255(x)
    x = normalize(x, mean, std)
    x = short_side_scale(x, side)
    top, left, th, tw = random_crop_window(x.shape[2], x.shape[3], crop, i, j)
    x = x[:, :, top:top + th, left:left + tw]
    if flip:
        x = x[..., ::-1]
    return np.ascontiguousarray(x)
