"""numpy restatement of the Pillow arithmetic behind ColorJitterVideoSSl (pytorchvideo_trainer datamodule/transforms.py).

The reference turns a (C, T, H, W) clip in [0, 1] into one tall (T*H, W) RGB PIL image and runs torchvision's PIL
ColorJitter (ImageEnhance Brightness / Contrast / Color blends, HSV hue shift), RandomGrayscale and ImageFilter.GaussianBlur
on it.  Every function here reproduces the C code of Pillow's Convert.c, Blend.c and BoxBlur.c operation by operation,
with its float32 / float64 types, so the results are Pillow's bytes (tests/test_gpu_color.py pins them against Pillow).
Images are uint8 arrays of shape (..., 3) (HWC), as np.asarray(PIL image) gives them.
"""
import numpy as np

F32, F64 = np.float32, np.float64


def to_bytes(x):
    """ToPILImage of a float tensor in [0, 1]: (x * 255).astype(uint8), a truncation, in float32."""
    return (np.asarray(x, F32) * F32(255)).astype(np.uint8)


def rgb_to_l(img):
    """convert("L"): (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16 (ITU-R 601-2 luma in 16-bit fixed point)."""
    i = img.astype(np.int64)
    return ((i[..., 0] * 19595 + i[..., 1] * 38470 + i[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def gray3(img):
    """RandomGrayscale(num_output_channels=3): convert("L") replicated to three channels."""
    g = rgb_to_l(img)
    return np.stack([g, g, g], -1)


def blend(deg, img, factor):
    """Image.blend(deg, img, factor): float32 deg + alpha * (img - deg), clipped to [0, 255], truncated.  Pillow takes
    alpha as a C float and interpolates without the clip for alpha in [0, 1], where the result cannot leave the range."""
    a = F32(factor)
    d = np.asarray(deg).astype(F32)
    v = d + a * (np.asarray(img).astype(F32) - d)
    return np.clip(v, F32(0), F32(255)).astype(np.uint8)


def brightness(img, factor):
    return blend(np.zeros_like(img), img, factor)


def saturation(img, factor):
    return blend(gray3(img), img, factor)


def contrast_mean(img):
    """int(ImageStat.Stat(img.convert("L")).mean[0] + 0.5): the integer luma sum over the whole image, divided in
    float64."""
    s = int(rgb_to_l(img).astype(np.int64).sum())
    n = int(np.prod(img.shape[:-1]))
    return int(s / n + 0.5)


def contrast(img, factor, mean=None):
    m = contrast_mean(img) if mean is None else mean
    return blend(np.full_like(img, m), img, factor)


def _clip8(v):
    return np.clip(v, 0, 255).astype(np.uint8)


def rgb_to_hsv(img):
    """convert("HSV") (Convert.c rgb2hsv_row): float32 ratios, float64 where the C code mixes in double constants."""
    r, g, b = (img[..., c].astype(np.int64) for c in range(3))
    maxc = np.maximum(r, np.maximum(g, b))
    minc = np.minimum(r, np.minimum(g, b))
    grey = maxc == minc
    safe = np.where(grey, 1, maxc - minc)
    cr = safe.astype(F32)
    s = (cr / np.where(grey, 1, maxc).astype(F32)).astype(F32)
    rc = ((maxc - r).astype(F32) / cr).astype(F32)
    gc = ((maxc - g).astype(F32) / cr).astype(F32)
    bc = ((maxc - b).astype(F32) / cr).astype(F32)
    h = np.where(r == maxc, (bc - gc).astype(F64),
                 np.where(g == maxc, F64(2.0) + rc.astype(F64) - bc.astype(F64),
                          F64(4.0) + gc.astype(F64) - rc.astype(F64))).astype(F32)
    h = np.fmod(h.astype(F64) / 6.0 + 1.0, 1.0).astype(F32)
    uh = _clip8(np.trunc(h.astype(F64) * 255.0).astype(np.int64))
    us = _clip8(np.trunc(s.astype(F64) * 255.0).astype(np.int64))
    uh = np.where(grey, 0, uh).astype(np.uint8)
    us = np.where(grey, 0, us).astype(np.uint8)
    return np.stack([uh, us, maxc.astype(np.uint8)], -1)


def hsv_to_rgb(hsv):
    """convert("RGB") of an HSV image (Convert.c hsv2rgb)."""
    h, s, v = (hsv[..., c].astype(np.int64) for c in range(3))
    hd = h.astype(F32).astype(F64) * 6.0 / 255.0
    i = np.floor(hd).astype(np.int64)
    f = (hd - i.astype(F32).astype(F64)).astype(F32)
    fs = (s.astype(F32).astype(F64) / 255.0).astype(F32)
    vd = v.astype(F32).astype(F64)
    p = _clip8(np.round(vd * (1.0 - fs.astype(F64))).astype(np.int64))
    q = _clip8(np.round(vd * (1.0 - (fs * f).astype(F32).astype(F64))).astype(np.int64))
    t = _clip8(np.round(vd * (1.0 - fs.astype(F64) * (1.0 - f.astype(F64)))).astype(np.int64))
    vv = v.astype(np.uint8)
    sel = i % 6
    out_r = np.choose(sel, [vv, q, p, p, t, vv])
    out_g = np.choose(sel, [t, vv, vv, q, p, p])
    out_b = np.choose(sel, [p, p, t, vv, vv, q])
    out = np.stack([out_r, out_g, out_b], -1)
    return np.where((s == 0)[..., None], np.stack([vv, vv, vv], -1), out).astype(np.uint8)


def hue_shift(hue_factor):
    """torchvision adjust_hue's byte offset: np.int32(hue_factor * 255).astype(np.uint8)."""
    return int(np.int32(hue_factor * 255).astype(np.uint8))


def hue(img, hue_factor):
    hsv = rgb_to_hsv(img)
    hsv[..., 0] = (hsv[..., 0].astype(np.int64) + hue_shift(hue_factor)) & 0xFF
    return hsv_to_rgb(hsv)


# ---- GaussianBlur (BoxBlur.c) --------------------------------------------------------------------------------------
def box_radius(sigma, passes=3):
    """_gaussian_blur_radius: the extended box radius whose `passes` box blurs have variance sigma**2 (float32, with
    the float64 steps of the C code).  Pillow receives sigma as a C float."""
    sigma = F32(sigma)
    sigma2 = F32(F32(sigma * sigma) / F32(passes))
    L = F32(np.sqrt(12.0 * F64(sigma2) + 1.0))
    l = F32(np.floor((F64(L) - 1.0) / 2.0))
    a = F32(F32(F32(2) * l + F32(1)) * F32(l * F32(l + F32(1)) - F32(3) * sigma2))
    a = F32(a / F32(F32(6) * F32(sigma2 - F32(l + F32(1)) * F32(l + F32(1)))))
    return F32(l + a)


def box_weights(radius):
    """(integer radius, ww, fw) of ImagingHorizontalBoxBlur: 2**24 / (2 * radius + 1) in float32, truncated, and the
    weight of the two partial pixels."""
    radius = F32(radius)
    r = int(radius)
    ww = int(F32(F32(1 << 24) / F32(radius * F32(2) + F32(1))))
    fw = ((1 << 24) - (2 * r + 1) * ww) // 2
    return r, ww, fw


def box_pass(a, r, ww, fw, axis):
    """One box pass along ``axis`` with edge pixels repeated: (sum of the 2r+1 window) * ww + (the two pixels just
    outside it) * fw, in 32-bit fixed point, rounded to a byte."""
    a = np.moveaxis(np.asarray(a, np.int64), axis, -1)
    n = a.shape[-1]
    x = np.arange(n)
    acc = np.zeros(a.shape, np.int64)
    for k in range(-r, r + 1):
        acc += a[..., np.clip(x + k, 0, n - 1)]
    far = a[..., np.clip(x - r - 1, 0, n - 1)] + a[..., np.clip(x + r + 1, 0, n - 1)]
    out = ((acc * ww + far * fw + (1 << 23)) >> 24).astype(np.uint8)
    return np.moveaxis(out, -1, axis)


def gaussian_blur(img, sigma, passes=3):
    """img.filter(ImageFilter.GaussianBlur(sigma)) on an (H, W, 3) image: `passes` horizontal box passes, then
    `passes` vertical ones, each rounded to bytes."""
    if F32(sigma) == 0:
        return img.copy()
    radius = box_radius(sigma, passes)
    out = np.asarray(img, np.uint8)
    if radius == 0:
        return out.copy()
    r, ww, fw = box_weights(radius)
    for axis in (1, 0):
        for _ in range(passes):
            out = box_pass(out, r, ww, fw, axis)
    return out


# ---- one view of ColorJitterVideoSSl --------------------------------------------------------------------------------
def color_jitter_view(img, order, factors, hue_factor, gray, sigma):
    """The PIL chain on one stacked (T*H, W, 3) image.  order: op ids (0 brightness, 1 contrast, 2 saturation, 3 hue)
    in the drawn permutation, with ops whose factor is None left out; factors: (b, c, s); sigma: None = no blur."""
    for op in order:
        if op == 0:
            img = brightness(img, factors[0])
        elif op == 1:
            img = contrast(img, factors[1])
        elif op == 2:
            img = saturation(img, factors[2])
        else:
            img = hue(img, hue_factor)
    if gray:
        img = gray3(img)
    if sigma is not None:
        img = gaussian_blur(img, sigma)
    return img
