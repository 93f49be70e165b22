"""MixUp, CutMix and MixVideo for batches of clips on the GPU (reference transforms/mix.py).

Clip b is mixed with clip B-1-b, in place: the call mutates ``x_video`` (and ``x_audio``) and returns the same tensor
objects, as the reference does.  The host draws every random number from torch's global RNG with the reference's calls
in the reference's order (the Beta draw, then the box centre, then the audio box centre; MixVideo's branch draw first),
so under one seed the same lambda and box are picked.  What reaches the GPU is one in-place launch per tensor (none for
an empty CutMix box) and one launch for the (B, num_classes) float32 soft labels.

One difference from the reference: index labels are range-checked before the video is touched, so a call that raises
for a bad label leaves the batch unchanged (the reference mixes the video first and then asserts).  The check reads one
flag back from the device, the same single host sync as the reference's ``torch.max(targets).item()``.
"""
import ctypes as C

import torch
import torch.nn as nn

from .. import _lib as L

_DTYPES = {torch.float32: L.PV_F32, torch.float16: L.PV_F16, torch.uint8: L.PV_U8}
MODE_MIX, MODE_ONE_HOT_F32, MODE_ONE_HOT_I64 = 0, 1, 2


# ---- argument checks and descriptors --------------------------------------------------------------------------------
def _overlaps(x):
    """Whether two elements of ``x`` may share memory (an ``expand``ed batch, for one).  Conservative: every dim,
    ordered by stride, must step past all the memory spanned by the dims inside it."""
    reach = 0
    for stride, size in sorted((s, n) for n, s in zip(x.shape, x.stride()) if n > 1):
        if stride <= reach:
            return True
        reach += (size - 1) * stride
    return False


def _check_batch(x, what, dtypes):
    if not torch.is_tensor(x):
        raise RuntimeError("%s expects a tensor" % what)
    if x.dim() < 2 or x.dim() > 5:
        raise RuntimeError("%s takes (B, ...) batches of 2 to 5 dims (got %d)" % (what, x.dim()))
    if x.dtype not in dtypes:
        raise RuntimeError("%s takes %s batches (got %s)" % (what, " or ".join(str(d) for d in dtypes), x.dtype))
    if _overlaps(x):
        raise RuntimeError("%s works in place: the batch must not have elements that share memory" % what)
    if x.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")


def _mix_desc(x):
    d = L.MixDesc()
    d.B, d.dtype = x.shape[0], _DTYPES[x.dtype]
    dims = [(1, 0)] * (5 - x.dim()) + list(zip(x.shape[1:], x.stride()[1:]))
    for i, (n, s) in enumerate(dims):
        d.size[i], d.stride[i] = n, s
    d.s_batch = x.stride(0)
    return d


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def _check_labels(labels, B, one_hot, dev):
    if not torch.is_tensor(labels):
        raise RuntimeError("labels must be a tensor")
    if one_hot:
        if labels.dtype != torch.float32 or labels.dim() != 2 or labels.shape[0] != B:
            raise RuntimeError("one_hot labels must be float32 (B, K) = (%d, K) (got %s %s)"
                               % (B, labels.dtype, tuple(labels.shape)))
    elif labels.dtype != torch.int64 or labels.dim() != 1 or labels.shape[0] != B:
        raise RuntimeError("labels must be int64 class indices of shape (%d,) (got %s %s)"
                           % (B, labels.dtype, tuple(labels.shape)))
    if labels.device != dev:
        raise RuntimeError("labels must be on the video's device %s (got %s)" % (dev, labels.device))


def _labels(labels, num_classes, label_smoothing, one_hot, lam, oml, mode=MODE_MIX):
    """Launch pv_mix_labels and check the indices: (B, K) float32 mixed labels (int64 one-hot rows in
    MODE_ONE_HOT_I64).  ``lam`` / ``oml`` are rounded to float32 here, as ATen rounds a scalar factor."""
    B = labels.shape[0]
    d = L.MixLabelDesc()
    d.B, d.one_hot, d.mode, d.lam, d.oml = B, int(one_hot), mode, float(lam), float(oml)
    if one_hot:
        d.K = labels.shape[1]
        d.s_row, d.s_col = labels.stride(0), labels.stride(1)
    else:
        assert 0 <= label_smoothing < 1.0, "Label smooth value needs to be between 0 and 1."
        d.K = num_classes
        off = label_smoothing / num_classes             # convert_to_one_hot's values, in double
        d.on, d.off = 1.0 - label_smoothing + off, off
        d.s_row, d.s_col = labels.stride(0), 0
    dev = labels.device
    out = torch.empty((B, d.K), dtype=torch.int64 if mode == MODE_ONE_HOT_I64 else torch.float32, device=dev)
    flag = None if one_hot else torch.empty(1, dtype=torch.int32, device=dev)
    L.check(L.load().pv_mix_labels(C.byref(d), labels.data_ptr(), out.data_ptr(),
                                   None if flag is None else flag.data_ptr(), _stream(dev)), "pv_mix_labels")
    if flag is not None:
        bad = int(flag.item())
        if bad & 1:
            raise AssertionError("Class Index must be less than number of classes")
        if bad & 2:
            raise RuntimeError("class indices must not be negative")
    return out


def mixup_(x, lam, oml):
    """x[b] = x[b]*lam + x[B-1-b]*oml for every clip at once, in place (float32 or float16, any strides)."""
    L.check(L.load().pv_mixup(C.byref(_mix_desc(x)), x.data_ptr(), float(lam), float(oml), _stream(x.device)),
            "pv_mixup")
    return x


def cutmix_(x, box):
    """Swap the (yl, yh, xl, xh) box of clips b and B-1-b across every C and T, in place."""
    yl, yh, xl, xh = box
    L.check(L.load().pv_cutmix(C.byref(_mix_desc(x)), x.data_ptr(), yl, yh, xl, xh, _stream(x.device)), "pv_cutmix")
    return x


def convert_to_one_hot(targets, num_class, label_smooth=0.0):
    """(B, num_class) one-hot rows of int64 class indices: int64 without smoothing, else float32 with
    ``label_smooth / num_class`` off the target and ``1 - label_smooth + label_smooth / num_class`` on it."""
    if not torch.is_tensor(targets) or targets.dtype != torch.int64 or targets.dim() != 1:
        raise RuntimeError("targets must be a 1-D int64 tensor of class indices")
    if targets.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")
    mode = MODE_ONE_HOT_I64 if label_smooth == 0.0 else MODE_ONE_HOT_F32
    return _labels(targets, num_class, label_smooth, False, 1.0, 0.0, mode)


# ---- the modules ----------------------------------------------------------------------------------------------------
class MixUp(nn.Module):
    """MixUp (https://arxiv.org/abs/1710.09412) for float32 / float16 batches (B, C, T, H, W) or (B, C, H, W), any
    strides, mixed in place.  Returns (x_video, labels) or (x_video, x_audio, labels) with ``x_audio=``."""

    def __init__(self, alpha=1.0, label_smoothing=0.0, num_classes=400, one_hot=False):
        super().__init__()
        self.mixup_beta_sampler = torch.distributions.beta.Beta(alpha, alpha)
        self.label_smoothing = label_smoothing
        self.num_classes = num_classes
        self.one_hot = one_hot

    def sample(self):
        """lambda: a float32 0-dim tensor, as the reference draws it."""
        return self.mixup_beta_sampler.sample()

    def forward(self, x_video, labels, **args):
        x_audio = args.get("x_audio", None)
        for x in (x_video,) if x_audio is None else (x_video, x_audio):
            assert x.size(0) > 1, "MixUp cannot be applied to a single instance."
            _check_batch(x, "MixUp", (torch.float32, torch.float16))
        _check_labels(labels, x_video.shape[0], self.one_hot, x_video.device)
        lam = self.sample()
        oml = 1.0 - lam                                  # float32, as the reference's 1.0 - mixup_lambda
        new_labels = _labels(labels, self.num_classes, self.label_smoothing, self.one_hot, lam, oml)
        mixup_(x_video, lam, oml)
        if x_audio is None:
            return x_video, new_labels
        mixup_(x_audio, lam, oml)
        return x_video, x_audio, new_labels


class CutMix(nn.Module):
    """CutMix (https://arxiv.org/abs/1905.04899) for uint8 / float16 / float32 batches (B, C, T, H, W) or
    (B, C, H, W), any strides: the box of clip B-1-b is pasted into clip b, in place.  Returns as MixUp."""

    def __init__(self, alpha=1.0, label_smoothing=0.0, num_classes=400, one_hot=False):
        super().__init__()
        self.one_hot = one_hot
        self.cutmix_beta_sampler = torch.distributions.beta.Beta(alpha, alpha)
        self.label_smoothing = label_smoothing
        self.num_classes = num_classes

    @staticmethod
    def rand_box(h, w, lam):
        """(yl, yh, xl, xh): a box of side int(h * sqrt(1 - lam)) by int(w * sqrt(1 - lam)) in float32 (lam is the
        float32 draw), centred on randint(h), randint(w) and clipped to the frame."""
        ratio = (1 - lam) ** 0.5
        half_h, half_w = int(h * ratio) // 2, int(w * ratio) // 2
        cy = torch.randint(h, (1,)).item()
        cx = torch.randint(w, (1,)).item()
        return (min(max(cy - half_h, 0), h), min(max(cy + half_h, 0), h),
                min(max(cx - half_w, 0), w), min(max(cx + half_w, 0), w))

    def sample(self, video_shape, audio_shape=None):
        """(lam, video box, corrected lam, audio box or None) in the reference's draw order.  The corrected lam, the
        share of the frame outside the box, is a Python float (double)."""
        lam = self.cutmix_beta_sampler.sample()
        h, w = video_shape[-2:]
        box = self.rand_box(h, w, lam)
        lam_c = 1.0 - float((box[1] - box[0]) * (box[3] - box[2])) / (h * w)
        audio_box = None if audio_shape is None else self.rand_box(audio_shape[-2], audio_shape[-1], lam)
        return lam, box, lam_c, audio_box

    def forward(self, x_video, labels, **args):
        x_audio = args.get("x_audio", None)
        for x in (x_video,) if x_audio is None else (x_video, x_audio):
            assert x.size(0) > 1, "Cutmix cannot be applied to a single instance."
            assert x.dim() == 4 or x.dim() == 5, "Please correct input shape."
            _check_batch(x, "CutMix", (torch.uint8, torch.float16, torch.float32))
        _check_labels(labels, x_video.shape[0], self.one_hot, x_video.device)
        _, box, lam_c, audio_box = self.sample(x_video.shape, None if x_audio is None else x_audio.shape)
        new_labels = _labels(labels, self.num_classes, self.label_smoothing, self.one_hot, lam_c, 1.0 - lam_c)
        cutmix_(x_video, box)
        if x_audio is None:
            return x_video, new_labels
        cutmix_(x_audio, audio_box)
        return x_video, x_audio, new_labels


class MixVideo(nn.Module):
    """CutMix with probability ``cutmix_prob``, else MixUp (reference MixVideo).  As in the reference, the CutMix branch
    is built without ``one_hot``, so one-hot labels work on the MixUp branch only, and ``x_audio`` is not taken."""

    def __init__(self, cutmix_prob=0.5, mixup_alpha=1.0, cutmix_alpha=1.0, label_smoothing=0.0, num_classes=400,
                 one_hot=False):
        assert 0.0 <= cutmix_prob <= 1.0, "cutmix_prob should be between 0.0 and 1.0"
        super().__init__()
        self.cutmix_prob = cutmix_prob
        self.mixup = MixUp(alpha=mixup_alpha, label_smoothing=label_smoothing, num_classes=num_classes,
                           one_hot=one_hot)
        self.cutmix = CutMix(alpha=cutmix_alpha, label_smoothing=label_smoothing, num_classes=num_classes)

    def use_cutmix(self):
        """The branch draw: torch.rand(1).item() < cutmix_prob."""
        return torch.rand(1).item() < self.cutmix_prob

    def forward(self, x_video, labels, **args):
        if args.get("x_audio", None) is not None:
            raise TypeError("MixVideo does not take x_audio (the reference hands it to MixUp / CutMix positionally, "
                            "which they do not accept); call MixUp or CutMix with x_audio= instead")
        if self.use_cutmix():
            return self.cutmix(x_video, labels)
        return self.mixup(x_video, labels)
