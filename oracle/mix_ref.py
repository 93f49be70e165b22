"""ORACLE (test infrastructure only): MixUp, CutMix and MixVideo restated on the CPU.

The formulas, for clip b and its partner B-1-b (the middle clip of an odd batch is its own partner):
  MixUp   x[b] = T(T(x[b] * lam) + T(x[B-1-b] * oml)), each product in fp32 and each result rounded to the element
          type T; lam is the float32 Beta draw and oml = float32(1 - lam).
  CutMix  x[b][..., yl:yh, xl:xh] = x[B-1-b][..., yl:yh, xl:xh] (a pure copy, any dtype).
  labels  f(f(l1 * lam) + f(l2 * oml)) in float32, l1 / l2 the one-hot rows of b and B-1-b: ls/K off the class and
          1 - ls + ls/K on it (double, then float32), or the given float32 rows with one_hot.  CutMix's lam is the
          corrected double 1 - area / (H*W); its factors are float32(lam) and float32(1.0 - lam).
The draws restate the reference's: Beta(alpha, alpha).sample(); for CutMix then randint(H), randint(W) for the box
centre and, with audio, the audio box's centre; MixVideo first draws torch.rand(1).item() < cutmix_prob.
oracle/gen_golden_mix.py asserts these equal the reference bit for bit.
"""
import torch


def one_hot_rows(labels, num_classes, ls):
    off = ls / num_classes
    rows = torch.full((labels.shape[0], num_classes), off, dtype=torch.float32)
    rows[torch.arange(labels.shape[0]), labels] = float(torch.tensor(1.0 - ls + off, dtype=torch.float32))
    return rows


def mix_labels(labels, num_classes, lam, oml, ls=0.0, one_hot=False):
    """lam / oml must be float32 values (Python floats holding them)."""
    l1 = labels.float() if one_hot else one_hot_rows(labels, num_classes, ls)
    return l1 * lam + l1.flip(0) * oml


def mixup(x, lam, oml):
    def r(v):
        return v.to(x.dtype).float()
    a, b = x.float(), x.flip(0).float()
    return r(r(a * lam) + r(b * oml)).to(x.dtype)


def cutmix(x, box):
    yl, yh, xl, xh = box
    y = x.clone()
    B = x.shape[0]
    for p in range(B // 2):
        q = B - 1 - p
        y[p, ..., yl:yh, xl:xh] = x[q, ..., yl:yh, xl:xh]
        y[q, ..., yl:yh, xl:xh] = x[p, ..., yl:yh, xl:xh]
    return y


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def draw_box(h, w, lam):
    side = (1 - lam) ** 0.5                                 # float32, from the float32 lam
    ch, cw = int(h * side), int(w * side)
    cy, cx = int(torch.randint(h, (1,))), int(torch.randint(w, (1,)))
    clamp = lambda v, hi: max(0, min(v, hi))                # noqa: E731
    return clamp(cy - ch // 2, h), clamp(cy + ch // 2, h), clamp(cx - cw // 2, w), clamp(cx + cw // 2, w)


def mixup_call(x, labels, alpha=1.0, ls=0.0, num_classes=400, one_hot=False, audio=None):
    """(video, audio or None, labels, draws) of one MixUp call on torch's global RNG."""
    lam = torch.distributions.beta.Beta(alpha, alpha).sample()
    lf, of = float(lam), float(1.0 - lam)
    out = mixup(x, lf, of)
    aout = None if audio is None else mixup(audio, lf, of)
    return out, aout, mix_labels(labels, num_classes, lf, of, ls, one_hot), {"lam": lf}


def cutmix_call(x, labels, alpha=1.0, ls=0.0, num_classes=400, one_hot=False, audio=None):
    lam = torch.distributions.beta.Beta(alpha, alpha).sample()
    H, W = x.shape[-2:]
    box = draw_box(H, W, lam)
    lam_c = 1.0 - float((box[1] - box[0]) * (box[3] - box[2])) / (H * W)
    abox = None if audio is None else draw_box(audio.shape[-2], audio.shape[-1], lam)
    out = cutmix(x, box)
    aout = None if audio is None else cutmix(audio, abox)
    lab = mix_labels(labels, num_classes, _f32(lam_c), _f32(1.0 - lam_c), ls, one_hot)
    return out, aout, lab, {"lam": float(lam), "box": box, "lam_c": lam_c, "audio_box": abox}


def mixvideo_call(x, labels, cutmix_prob=0.5, mixup_alpha=1.0, cutmix_alpha=1.0, ls=0.0, num_classes=400,
                  one_hot=False):
    if torch.rand(1).item() < cutmix_prob:
        out, _, lab, draws = cutmix_call(x, labels, cutmix_alpha, ls, num_classes)
        return out, lab, dict(draws, branch="cutmix")
    out, _, lab, draws = mixup_call(x, labels, mixup_alpha, ls, num_classes, one_hot)
    return out, lab, dict(draws, branch="mixup")
