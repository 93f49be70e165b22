"""ORACLE (test infrastructure only): the video augmentation ops restated on torchvision's functional API, on the CPU.

Each op takes a (T, C, H, W) uint8 or float32 CPU tensor and an already drawn argument (the draws themselves are the
product's host code, pinned against the reference's recorded draws by the goldens).  oracle/gen_golden_augment.py
asserts these functions equal the reference bit for bit.  For the ops whose uint8 result ends in a cast of a float
sum with no fixed order (AdjustContrast, AdjustSharpness, the warps), ``pre_cast64`` gives the float64 value before
each cast, so a test can tell a rounding-boundary pixel from a wrong one.
"""
import torch
import torch.nn.functional as F
import torchvision.transforms.functional as TF
from torchvision.transforms import InterpolationMode
from torchvision.transforms import _functional_tensor as TFT

FILL = (0.5, 0.5, 0.5)
TIER2_OPS = ("AdjustContrast", "AdjustSharpness", "Rotate", "ShearX", "ShearY", "TranslateX", "TranslateY")


def _via_u8(video, fn):
    """The reference's float path of Equalize / Posterize: (x * 255).to(uint8), the uint8 op, / 255."""
    return (fn((video * 255).to(torch.uint8)) / 255).to(video.dtype)


def warp_matrix(name, arg, h, w):
    if name == "ShearX":
        return [1, arg, h * arg / 2, 0, 1, 0]
    if name == "ShearY":
        return [1, 0, 0, arg, 1, w * arg / 2]
    if name == "TranslateX":
        return [1, 0, arg * w, 0, 1, 0]
    if name == "TranslateY":
        return [1, 0, 0, 0, 1, arg * h]
    raise ValueError(name)


def apply_op(video, name, arg=None, fill=FILL):
    u8 = video.dtype == torch.uint8
    if name == "AdjustBrightness":
        return TF.adjust_brightness(video, arg)
    if name == "AdjustContrast":
        return TF.adjust_contrast(video, arg)
    if name == "AdjustSaturation":
        return TF.adjust_saturation(video, arg)
    if name == "AdjustSharpness":
        return TF.adjust_sharpness(video, arg)
    if name == "AutoContrast":
        return TF.autocontrast(video)
    if name == "Equalize":
        return TF.equalize(video) if u8 else _via_u8(video, TF.equalize)
    if name == "Invert":
        return TF.invert(video)
    if name == "Posterize":
        if arg >= 8:
            return video
        return TF.posterize(video, arg) if u8 else _via_u8(video, lambda v: TF.posterize(v, arg))
    if name == "Solarize":
        return TF.solarize(video, int(arg * 255.0) if u8 else arg)
    if name == "Rotate":
        return TF.rotate(video, arg, fill=list(fill), interpolation=InterpolationMode.BILINEAR)
    h, w = video.shape[-2:]
    return TFT.affine(video, warp_matrix(name, arg, h, w), interpolation="bilinear", fill=list(fill))


def apply_chain(video, ops, fill=FILL):
    for op in ops:
        if op is not None:
            video = apply_op(video, op[0], op[1], fill)
    return video


def mix_chains(video, weights, m, chain_outputs):
    """AugMix's mix of already augmented chains: mixed = sum_k w_k * chain_k (fp32, chain order), then
    m * video + (1 - m) * mixed (uint8: truncated)."""
    mixed = torch.zeros(video.shape, dtype=torch.float32)
    for w, out in zip(weights, chain_outputs):
        mixed += w * out
    out = m * video + (1 - m) * mixed
    return out.type(torch.uint8) if video.dtype == torch.uint8 else out


def augmix(video, weights, m, chains, fill=FILL):
    """mix_chains over chain_k(video), each chain applied in order."""
    return mix_chains(video, weights, m, [apply_chain(video, ops, fill) for ops in chains])


def random_resized_crop(frames, boxes, target_h, target_w):
    """(C, T, H, W) float32: frame t's window boxes[t] = (top, left, h, w) resized bilinearly to target_h x target_w."""
    out = torch.zeros((frames.shape[0], frames.shape[1], target_h, target_w))
    for t, (i, j, h, w) in enumerate(boxes):
        out[:, t:t + 1] = F.interpolate(frames[:, t:t + 1, i:i + h, j:j + w], size=(target_h, target_w),
                                        mode="bilinear")
    return out


def pre_cast64(video, name, arg, fill=FILL):
    """[(float64 tensor, "round" | "trunc")]: the value before each uint8 cast of a tier-2 op on a uint8 ``video``,
    NaN where that cast does not apply."""
    x = video.double()
    if name == "AdjustContrast":
        gray = TF.rgb_to_grayscale(video).double()          # the reference's truncated uint8 grayscale
        mean = gray.mean(dim=(-3, -2, -1), keepdim=True)
        return [((arg * x + (1.0 - arg) * mean).clamp(0, 255), "trunc")]
    if name == "AdjustSharpness":
        k = torch.ones(3, 3, dtype=torch.float64)
        k[1, 1] = 5.0
        k = (k / k.sum()).expand(x.shape[-3], 1, 3, 3)
        blur = torch.full_like(x, float("nan"))
        blur[..., 1:-1, 1:-1] = F.conv2d(x, k, groups=x.shape[-3])
        ref_blur = x.clone()
        ref_blur[..., 1:-1, 1:-1] = torch.round(F.conv2d(video.float(), k.float(), groups=x.shape[-3])).double()
        return [(blur, "round"), ((arg * x + (1.0 - arg) * ref_blur).clamp(0, 255), "trunc")]
    h, w = video.shape[-2:]
    if name == "Rotate":
        matrix = TF._get_inverse_affine_matrix([0.0, 0.0], -arg, [0.0, 0.0], 1.0, [0.0, 0.0])
    else:
        matrix = warp_matrix(name, arg, h, w)
    theta = torch.tensor(matrix, dtype=torch.float64).reshape(1, 2, 3)
    grid = TFT._gen_affine_grid(theta, w=w, h=h, ow=w, oh=h)
    img = torch.cat((x, torch.ones_like(x[:, :1])), dim=1)
    img = F.grid_sample(img, grid.expand(x.shape[0], -1, -1, -1), mode="bilinear", padding_mode="zeros",
                        align_corners=False)
    mask = img[:, -1:].expand_as(x)
    fill_img = torch.tensor(fill, dtype=torch.float64).view(1, -1, 1, 1).expand_as(x)
    return [(img[:, :-1] * mask + (1.0 - mask) * fill_img, "round")]


def near_boundary(stages, eps=1e-3):
    """Pixels whose pre-cast value lies within eps of a rounding (x.5) or truncation (integer) boundary."""
    near = None
    for v, kind in stages:
        d = (v - v.floor() - 0.5).abs() if kind == "round" else (v - v.round()).abs()
        m = torch.nan_to_num(d, nan=1.0) < eps
        near = m if near is None else near | m
    return near
