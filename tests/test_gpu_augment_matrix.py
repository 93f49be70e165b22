"""The kernels that prepare a training batch, one row per instance and edge: pv_augment.cu (RandAugment / AugMix ops
and the AugMix mix), pv_mix.cu (MixUp, CutMix, mixed labels), pv_colorjitter.cu (the contrastive views' colour jitter
and Gaussian blur) and pv_boxes.cu (detection box arithmetic).

Every GPU test calls the C ABI directly (ctypes) with a descriptor the row fills itself, asserts from the library's
launch counts which kernel instance ran, puts a sentinel after every output buffer (for the in-place kernels:
everywhere outside the addressed elements) and checks that it survives, fills source padding with a large value, and
compares:
  - bit-exact: Brightness, Saturation, AutoContrast, Equalize, Invert, Posterize, Solarize and the identity op against
    torchvision on the CPU (oracle.augment_ref.apply_op); augment_stats_kernel's min / max / table / grey sum against a
    restatement of torchvision's _scale_channel and an exact sum; the AugMix mix against oracle.augment_ref.mix_chains;
    MixUp, CutMix and the labels against oracle.mix_ref; the colour jitter against oracle.color_ref (Pillow's
    arithmetic); the boxes against numpy in the boxes' own type;
  - bounded against float64, the bound derived beside each reference from the kernel's operation count:
    AdjustContrast (3 roundings of the blend on top of the fp32 mean), AdjustSharpness (9 products and 9 sums, then the
    blend) and the five warps (the fp32 geometry restated exactly, which fixes the taps; 4 products and sums per
    accumulator, then the mask / fill blend).  A uint8 result must be the cast of a value inside the float64 value's
    bound.  These rows are also held to the tier of test_gpu_augment.py against torchvision (1e-5 absolute; uint8 off
    by one only at a cast boundary), and AdjustSharpness and the warps, whose operation order the kernel fixes, must
    equal the fp32 restatement bit for bit.
CPU tests check that the launch sites of the four files are exactly the instances the rows expect, that the rows reach
the branches they are meant to, that the fp32 restatement of each family passes its check, and that named wrong
kernels fail it.  One listed wrong kernel cannot fail: `ix >= -1` for `ix > -1` in the warp changes no output (at
ix == -1 the only inside tap has weight 0), test_warp_cutoff_is_an_early_out_only shows it; the visible neighbour
(cutting at ix >= 0, which drops the partly covered border column) is the mutation instead.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit): the largest err / tol of the float32 rows per bounded family,
and in brackets the largest share of a uint8 row's pixels that had two admissible values:
  AdjustContrast 0.666 (0.037), AdjustSharpness 0.672 (0.778, a 3 x 3 frame), the warps 0.270 (1.0: a frame shifted
  wholly outside is fill 0.5 everywhere, a tie; next 0.09).
AdjustSharpness and the warps also equalled the fp32 restatement bit for bit, and every other family matched its
reference bit for bit.  The vertical blur ran for the first time above 48 KiB of shared memory (1792 rows: strip 16,
56 KiB; 3200 rows: strip 8, 50 KiB; 24600 and 12300 rows: strip 1) and matched oracle.color_ref bit for bit, also
with the 48 KiB size launched before and after the larger ones.

The rows found one defect, fixed with them: uint8 AutoContrast computed its scale as 255 / (max - min) in one
division, where torch evaluates torchvision's `bound / tensor` as reciprocal() * bound.  The two differ in the last
bit for 46 of the 255 possible ranges, and for 33 of them some pixel (usually the frame's maximum, 254 in torchvision)
came out one higher; the single golden clip has none of these ranges.  The one-division restatement fails the 3 x 3
AutoContrast row (test_augment_check_rejects_wrong_kernels); the kernel before the fix was not run on the GPU.  The
box rows compare zeros by value: numpy leaves the sign of maximum(0.0, -0.0) to its build.

Not verified: the 2^31 offset guards (a frame of 2^31 / 3 pixels, clips over 2 GB), n_views beyond a few dozen, and
the vertical blur's upper limit of 200 KiB (a stack of 102400 rows).
"""
import ctypes
import os
import re
import zlib

import numpy as np
import pytest
import torch

from oracle import augment_ref as AO
from oracle import color_ref as CO
from oracle import mix_ref as MO
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.transforms import augment as AUG
from pytorchvideo_b200.transforms import color as CJ

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorchvideo_b200", "csrc")
f32, f64 = np.float32, np.float64
U = TS.F32_EPS
TAIL = 64
SENT = {torch.uint8: 0x5A, torch.float16: 0x5A5A, torch.float32: 0x5A5A5A5A, torch.float64: 0x5A5A5A5A5A5A5A5A,
        torch.int64: 0x5A5A5A5A5A5A5A5A}
INT = {torch.uint8: torch.uint8, torch.float16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64,
       torch.int64: torch.int64}
TDT = {"u8": torch.uint8, "f16": torch.float16, "f32": torch.float32, "f64": torch.float64}
CT = {"u8": "uint8_t", "f16": "__half", "f32": "float", "f64": "double"}


def _dev():
    return torch.device("cuda:0")


def _L():
    from pytorchvideo_b200 import _lib as L
    return L


def _code(dt):
    L = _L()
    return {"u8": L.PV_U8, "f16": L.PV_F16, "f32": L.PV_F32}[dt]


def _gen(row):
    return torch.Generator().manual_seed(zlib.crc32(repr(row).encode()))


def _rid(row):
    return "-".join(str(v) for v in row).replace(" ", "")


def _bits(t):
    return t.detach().cpu().contiguous().view(INT[t.dtype])


def _sentinel(n, dtype):
    return torch.full((n,), SENT[dtype], dtype=INT[dtype]).view(dtype)


def _assert_untouched(buf, written, what):
    b = _bits(buf).reshape(-1)
    bad = (b != _bits(_sentinel(1, buf.dtype))[0]) & ~written.reshape(-1)
    assert not bool(bad.any()), "%s: %d elements outside the output changed (first at flat %d)" % (
        what, int(bad.sum()), int(bad.nonzero()[0]))


def _launch(entry, *args):
    L = _L()
    before = TS.kernel_counts()
    L.check(getattr(L.load(), entry)(*args), entry)
    torch.cuda.synchronize()
    return TS.kernel_count_diff(before, TS.kernel_counts())


def _expect(name, launched):
    want = {name: 1} if name else {}
    assert launched == want, "expected %s, launched %s" % (want, launched)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _same_bits(got, want, what):
    """Bit equality, except that any NaN equals any NaN at the same place (arithmetic does not fix a NaN's payload)."""
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    if got.dtype.is_floating_point:
        gn, wn = torch.isnan(got), torch.isnan(want)
        assert torch.equal(gn, wn), "%s: NaN positions differ" % what
        gb, wb = _bits(got)[~gn], _bits(want)[~wn]
    else:
        gb, wb = got.reshape(-1), want.reshape(-1)
    n = int((gb != wb).sum())
    assert n == 0, "%s: %d of %d values differ (first at %d)" % (what, n, gb.numel(), int((gb != wb).nonzero()[0]))


def _strided_index(shape, strides, base=0):
    """Flat element offsets of a strided view (int64 tensor of ``shape``)."""
    idx = torch.full(tuple(shape), base, dtype=torch.int64)
    for i, (n, s) in enumerate(zip(shape, strides)):
        view = [1] * len(shape)
        view[i] = n
        idx = idx + (torch.arange(n, dtype=torch.int64) * s).view(view)
    return idx


# =====================================================================================================================
# pv_augment.cu: rows
# =====================================================================================================================
AUG_SIZES = [(1, 1), (1, 7), (9, 1), (3, 3), (15, 16), (16, 16), (17, 31), (64, 80), (224, 224)]
AUG_LAYOUTS = ("cont", "thwc", "wslice")
AUG_CLIPS = ((1, 1), (2, 1), (3, 3), (6, 3))               # (n_clips, src_div)
EXACT_OPS = [("Identity", None), ("AdjustBrightness", 1.7), ("AdjustBrightness", 0.3), ("AdjustSaturation", 1.9),
             ("AdjustSaturation", 0.25), ("AutoContrast", None), ("Equalize", None), ("Invert", None),
             ("Posterize", 0), ("Posterize", 1), ("Posterize", 7), ("Solarize", 0.5), ("Solarize", 0.3)]
WARP_OPS = [("Rotate", 30.0), ("Rotate", -17.5), ("Rotate", 90.0), ("Rotate", 0.0), ("ShearX", 0.3),
            ("ShearY", -0.21), ("TranslateX", 0.25), ("TranslateX", -0.28125), ("TranslateX", 0.28125),
            ("TranslateY", -0.45), ("TranslateY", 0.28125), ("TranslateX", 1.5)]
BOUNDED_OPS = [("AdjustContrast", 1.6), ("AdjustContrast", 0.4), ("AdjustSharpness", 1.9),
               ("AdjustSharpness", 0.2)] + WARP_OPS
STATS_OPS = ("AdjustContrast", "AutoContrast", "Equalize")


def _aug_rows():
    rows = []
    for i, (name, arg) in enumerate(EXACT_OPS + BOUNDED_OPS):
        for j, (H, W) in enumerate(AUG_SIZES):
            k = i + j
            n_clips, div = AUG_CLIPS[k % 4]
            content = {"AutoContrast": "constch", "Equalize": ("eqident", "rand")[(j // 2) % 2]}.get(name, "rand")
            rows.append((name, arg, ("u8", "f32")[k % 2], 1 if H >= 224 else 2, H, W, AUG_LAYOUTS[(k // 2) % 3],
                         n_clips, div, content))
    for k, (name, arg) in enumerate([("Equalize", None), ("AdjustContrast", 1.6), ("Rotate", 30.0),
                                     ("AdjustSharpness", 1.9)]):
        rows.append((name, arg, ("u8", "f32")[k % 2], 1, 720, 1280, AUG_LAYOUTS[k % 3], 1, 1, "rand"))
    # every frame the launch limit allows: 4369 clips of 15 one-pixel frames
    rows.append(("Invert", None, "u8", 15, 1, 1, "cont", 4369, 1, "rand"))
    rows.append(("AdjustBrightness", 1.7, "f32", 15, 1, 1, "cont", 4369, 1, "rand"))
    return rows


AUG_ROWS = _aug_rows()


def aug_instance(kernel, dt):
    return "augment_%s_kernel<%s>" % (kernel, CT[dt])


def _special_f32(g, n, thr):
    k = torch.randint(0, 256, (n,), generator=g).numpy()
    grid = (k.astype(f32) / f32(255))
    below = np.maximum(np.nextafter(grid, f32(0)), f32(0))
    v = np.concatenate([[0.0, 1.0], grid, below, [thr, np.nextafter(f32(thr), f32(0)), np.nextafter(f32(thr), f32(1))]])
    return np.clip(v, 0, 1).astype(f32)


def aug_case(row):
    """Source values [n_src, T, 3, H, W], the per-clip op records (the product's encode_op), and the (name, arg) per
    clip; clip 1 of a multi-clip row runs the identity op, so ops[clip] is indexed."""
    name, arg, dt, T, H, W, layout, n_clips, div, content = row
    g = _gen(row)
    n_src = n_clips // div
    shape = (n_src, T, 3, H, W)
    hw = H * W
    if dt == "u8":
        v = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
    else:
        v = torch.rand(shape, generator=g)
    if content == "constch":
        v[:, :, 1] = v[:, :, 1].reshape(-1)[0]
    elif content == "eqident":      # one dominant value in the last non-empty bin: step == 0 although not constant
        top = 200 if dt == "u8" else float(f32(200) / f32(255))
        keep = torch.rand(shape, generator=g) < min(0.4, 200.0 / max(hw, 1))
        low = v if dt == "u8" else v * 0.7
        v = torch.where(keep, (low.float() * (0.7 if dt == "u8" else 1.0)).to(v.dtype), torch.full_like(v, top))
    elif hw >= 9 and n_clips < 100:
        flat = v.view(n_src, T, 3, hw)
        if dt == "u8":
            thr = int(arg * 255.0) if name == "Solarize" else 128
            sp = torch.tensor([0, 255, thr, max(thr - 1, 0), min(thr + 1, 255)], dtype=torch.uint8)
        else:
            sp = torch.from_numpy(_special_f32(g, 4, arg if name == "Solarize" else 0.5))
        n = min(len(sp), hw // 2)
        pos = torch.randperm(hw, generator=g)[:n]
        flat[..., pos] = sp[:n]
    ops = [(name, arg) if (c != 1 or n_clips == 1) and name != "Identity" else None for c in range(n_clips)]
    recs = [AUG.encode_op(op, TDT[dt], H, W, AO.FILL) for op in ops]
    return dict(vals=v, ops=ops, recs=recs)


def _aug_src_buffer(vals, layout):
    n, T, C, H, W = vals.shape
    big = 0xEE if vals.dtype == torch.uint8 else 60000.0
    if layout == "thwc":
        strides = (T * H * W * 4, H * W * 4, 1, W * 4, 4)
    elif layout == "wslice":
        Wp = W + 3
        strides = (T * 3 * H * Wp + 7, 3 * H * Wp, H * Wp, Wp, 1)
    else:
        strides = (T * 3 * H * W, 3 * H * W, H * W, W, 1)
    size = 1 + sum((d - 1) * s for d, s in zip(vals.shape, strides))
    buf = torch.full((size + 16,), big, dtype=vals.dtype)
    buf.as_strided(vals.shape, strides).copy_(vals)
    return buf, strides


def _aug_desc(row, strides):
    name, arg, dt, T, H, W, layout, n_clips, div, content = row
    d = _L().AugmentDesc()
    d.n_clips, d.src_div, d.T, d.C, d.H, d.W = n_clips, div, T, 3, H, W
    d.s_clip, d.st, d.sc, d.sh, d.sw = strides
    d.dtype = _code(dt)
    return d


STATS_NP = np.dtype([("mn", "f4", 3), ("mx", "f4", 3), ("gray_sum", "f8"), ("lut", "u1", (3, 256))])


# ---- fp32 restatement of the kernels (numpy float32: one rounding per operation, in the kernels' order) ---------------
def _gray32(v, u8):
    l = (f32(0.2989) * v[0] + f32(0.587) * v[1]) + f32(0.114) * v[2]
    return np.trunc(l) if u8 else l


def _byte_of(v, u8):
    return v.astype(np.int64) if u8 else ((v * f32(255)).astype(np.int64) & 0xFF)


def _blend32(a, b, ratio, omr, u8, fma=False):
    ratio, omr = f32(ratio), f32(omr)
    b = np.asarray(b, f32)
    if fma:      # fma(ratio, a, omr * b): the product ratio * a is exact in float64
        v = (f64(ratio) * a.astype(f64) + (omr * b).astype(f64)).astype(f32)
    else:
        v = ratio * a + omr * b
    v = np.clip(v, f32(0), f32(255 if u8 else 1))
    return np.trunc(v) if u8 else v


def scale_channel_lut(hist):
    """torchvision _scale_channel's table from a 256-bin histogram; None when step == 0 (the channel is kept)."""
    hist = torch.as_tensor(hist, dtype=torch.int64)
    nonzero = hist[hist != 0]
    step = torch.div(nonzero[:-1].sum(), 255, rounding_mode="floor")
    if step == 0:
        return None
    lut = torch.div(torch.cumsum(hist, 0) + torch.div(step, 2, rounding_mode="floor"), step, rounding_mode="floor")
    return torch.nn.functional.pad(lut, [1, 0])[:-1].clamp(0, 255).numpy().astype(np.uint8)


def frame_stats(v, u8, mutation=None):
    """(mn[3], mx[3], grey sum in float64, lut[3][256]) of one float32 [3, H, W] frame, as augment_stats_kernel."""
    mn, mx = v.reshape(3, -1).min(1), v.reshape(3, -1).max(1)
    gsum = float(_gray32(v, u8).astype(f64).sum())
    lut = np.zeros((3, 256), np.uint8)
    for c in range(3):
        hist = np.bincount(_byte_of(v[c], u8).reshape(-1), minlength=256)
        t = scale_channel_lut(hist)
        if t is not None and mutation == "lut_unshifted":
            step = int(hist[hist != 0][:-1].sum()) // 255
            t = np.minimum((np.cumsum(hist) + step // 2) // step, 255).astype(np.uint8)
        lut[c] = np.arange(256) if t is None else t
    return mn.astype(f32), mx.astype(f32), gsum, lut


def affine_geometry(H, W, theta, mutation=None):
    """The warp's sampling geometry in fp32, as the kernel states it: per output pixel the top-left tap (x0, y0), the
    four weights and whether any tap can be inside."""
    t = [f32(x) for x in theta]
    bx = np.arange(W, dtype=f32)[None, :] + f32(0.5 - 0.5 * W)
    by = np.arange(H, dtype=f32)[:, None] + f32(0.5 - 0.5 * H)
    gx = (bx * t[0] + by * t[1]) + t[2]
    gy = (bx * t[3] + by * t[4]) + t[5]
    ix = (gx + f32(1)) * f32(0.5 * W) - f32(0.5)
    iy = (gy + f32(1)) * f32(0.5 * H) - f32(0.5)
    lo = {"ix_ge_m1": ix >= -1, "ix_ge_0": ix >= 0}.get(mutation, ix > -1)
    inside = lo & (ix < W) & (iy > -1) & (iy < H)
    ix, iy = np.where(inside, ix, f32(0)), np.where(inside, iy, f32(0))
    fx, fy = np.floor(ix), np.floor(iy)
    tx, ty = ix - fx, iy - fy
    ex, sy = f32(1) - tx, f32(1) - ty
    wt = [sy * ex, sy * tx, ty * ex, ty * tx]
    return fx.astype(np.int64), fy.astype(np.int64), wt, inside, tx, ty


def _taps(v, x0, y0, inside):
    """Per tap k: (values [3, H, W] with 0 outside the frame, in-frame mask [H, W])."""
    H, W = v.shape[1:]
    out = []
    for k in range(4):
        xx, yy = x0 + (k & 1), y0 + (k >> 1)
        ok = inside & (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        val = v[:, np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)]
        out.append((np.where(ok[None], val, f32(0)), ok))
    return out


def emulate_frame(v, rec, u8, mutation=None):
    """One frame through augment_apply_kernel: v float32 [3, H, W] (uint8 values as floats), rec an encode_op record.
    Returns the float32 value the kernel stores (uint8: before the final integer conversion, already integral)."""
    kind, ival, ratio, omr = int(rec[0]), int(rec[1]), f32(rec[2]), f32(rec[3])
    bound = f32(255 if u8 else 1)
    H, W = v.shape[1:]
    fma = mutation == "fma"
    if kind == 1:
        return _blend32(v, np.zeros_like(v), ratio, omr, u8, fma)
    if kind == 2:
        mean = f32(frame_stats(v, u8)[2] / f64(H * W))
        return _blend32(v, mean, ratio, omr, u8, fma)
    if kind == 3:
        return _blend32(v, _gray32(v, u8)[None], ratio, omr, u8, fma)
    if kind == 4:
        k1, k5 = f32(1) / f32(13), f32(5) / f32(13)
        b = v.copy()
        if mutation == "blur_border":
            p = np.pad(v, ((0, 0), (1, 1), (1, 1)), mode="edge")
            ys, xs = slice(0, H), slice(0, W)
        else:
            p = v
            ys, xs = slice(1, H - 1), slice(1, W - 1)
        hh, ww = (H, W) if mutation == "blur_border" else (H - 2, W - 2)
        acc = np.zeros((3, hh, ww), f32)
        for dy in range(3):
            for dx in range(3):
                acc = acc + (k5 if dy == 1 and dx == 1 else k1) * p[:, dy:dy + hh, dx:dx + ww]
        b[:, ys, xs] = np.rint(acc) if u8 else acc
        return _blend32(v, b, ratio, omr, u8, fma)
    if kind == 5:
        mn, mx, _, _ = frame_stats(v, u8)
        out = np.empty_like(v)
        for c in range(3):
            with np.errstate(divide="ignore"):
                d = mx[c] - mn[c]      # torch evaluates `bound / tensor` as tensor.reciprocal() * bound
                lo, sc = mn[c], (bound / d if mutation == "one_division" else (f32(1) / d) * bound)
            if not np.isfinite(sc):
                lo, sc = f32(0), f32(1)
            q = np.clip((v[c] - lo) * sc, f32(0), bound)
            out[c] = np.trunc(q) if u8 else q
        return out
    if kind == 6:
        lut = frame_stats(v, u8, mutation)[3]
        e = np.stack([lut[c][_byte_of(v[c], u8)] for c in range(3)]).astype(f32)
        return e if u8 else e / f32(255)
    if kind == 7:
        return bound - v
    if kind == 8:
        e = (_byte_of(v, u8) & ival).astype(f32)
        return e if u8 else e / f32(255)
    if kind == 9:
        hit = (v > f32(ival) if mutation == "solarize_gt" else v >= f32(ival)) if u8 else \
              (v > ratio if mutation == "solarize_gt" else v >= ratio)
        return np.where(hit, bound - v, v)
    if kind == 10:
        x0, y0, wt, inside, _, _ = affine_geometry(H, W, rec[4:10], mutation)
        acc, mask = np.zeros_like(v), np.zeros((H, W), f32)
        for (val, ok), w in zip(_taps(v, x0, y0, inside), wt):
            w = np.where(inside, w, f32(0))
            acc = acc + val * w[None]
            mask = mask + ok.astype(f32) * w
        fill = np.asarray(rec[10:13], f32).reshape(3, 1, 1)
        q = acc * mask[None] + (f32(1) - mask)[None] * fill
        if not u8:
            return q
        return np.trunc(q) if mutation == "warp_trunc" else np.rint(q)
    return v.copy()


def aug_emulate(row, case, mutation=None):
    name, arg, dt, T, H, W, layout, n_clips, div, content = row
    u8 = dt == "u8"
    out = np.empty((n_clips, T, 3, H, W), f32)
    src = case["vals"].numpy().astype(f32)
    for c in range(n_clips):
        for t in range(T):
            out[c, t] = emulate_frame(src[c // div, t], case["recs"][c], u8, mutation)
    return torch.from_numpy(out.astype(np.uint8) if u8 else out)


# ---- float64 references of the bounded ops: (ref, tol) before the cast, per frame ------------------------------------
def _tol(ref, absref, n_round):
    return U * np.abs(ref) + n_round * U * absref + 2.0 ** -37


def bounded_range(v, rec, u8):
    """[lo, hi] the stored value of one frame must lie in, and the float64 value / tolerance for the RATIO line:
    float: the float64 result -+ its tolerance; uint8: the casts of the ends of that interval."""
    kind, ratio, omr = int(rec[0]), f64(f32(rec[2])), f64(f32(rec[3]))
    H, W = v.shape[1:]
    x = v.astype(f64)
    top = 255.0 if u8 else 1.0
    if kind == 2:
        # mean: the float64 mean of the fp32 (uint8: truncated) grey, rounded once to fp32 by the kernel; the blend
        # rounds both products and the sum: U |omr mean| + U |ratio v| + U |omr mean| + U |result|
        mean = _gray32(v, u8).astype(f64).sum() / (H * W)
        ref = ratio * x + omr * mean
        tol = _tol(ref, np.abs(ratio * x) + 2 * abs(omr * mean), 1)
        lo, hi = np.clip(ref - tol, 0, top), np.clip(ref + tol, 0, top)
        return (np.floor(lo), np.floor(hi), ref, tol) if u8 else (lo, hi, np.clip(ref, 0, top), tol)
    if kind == 4:
        k1, k5 = f64(f32(1) / f32(13)), f64(f32(5) / f32(13))
        b = x.copy()
        eb = np.zeros_like(x)
        if H > 2 and W > 2:
            acc = np.zeros((3, H - 2, W - 2))
            for dy in range(3):
                for dx in range(3):
                    acc += (k5 if dy == 1 and dx == 1 else k1) * x[:, dy:dy + H - 2, dx:dx + W - 2]
            b[:, 1:-1, 1:-1] = acc
            eb[:, 1:-1, 1:-1] = 10 * U * acc        # 9 products and 9 sums of non-negative terms (the first sum is exact)
        cands = [np.rint(b - eb), np.rint(b + eb)] if u8 else [b - eb, b + eb]
        los, his = [], []
        for bc in cands:
            p = ratio * x + omr * bc
            t = _tol(p, np.abs(ratio * x) + np.abs(omr * bc), 1)
            los.append(np.clip(p - t, 0, top))
            his.append(np.clip(p + t, 0, top))
        lo, hi = np.minimum(*los), np.maximum(*his)
        ref = np.clip(ratio * x + omr * (np.rint(b) if u8 else b), 0, top)
        tol = np.maximum((hi - lo) / 2, 2.0 ** -37)
        return (np.floor(lo), np.floor(hi), ref, tol) if u8 else (lo, hi, ref, tol)
    assert kind == 10
    x0, y0, wt, inside, _, _ = affine_geometry(H, W, rec[4:10])
    acc, mask, mag = np.zeros_like(x), np.zeros((H, W)), np.zeros_like(x)
    for (val, ok), w in zip(_taps(v, x0, y0, inside), wt):
        w = np.where(inside, w, f32(0)).astype(f64)
        acc += val.astype(f64) * w[None]
        mag += np.abs(val.astype(f64)) * w[None]
        mask += ok * w
    fill = np.asarray(rec[10:13], f32).astype(f64).reshape(3, 1, 1)
    ref = acc * mask[None] + (1.0 - mask)[None] * fill
    # each accumulator: 4 products and 3 inexact sums (<= 4 U of its magnitude); then acc * mask, 1 - mask, its
    # product with fill, and the sum: 4 U mag mask + 4 U mask mag + U mag mask + (4 U mask + 2 U) fill + U |ref|
    tol = _tol(ref, 9 * mag * mask[None] + (4 * mask[None] + 2) * np.abs(fill), 1)
    if u8:
        return np.rint(ref - tol), np.rint(ref + tol), ref, tol
    return ref - tol, ref + tol, ref, tol


def aug_check(row, case, got):
    """Assert ``got`` [n_clips, T, 3, H, W] (torch, the row's dtype) is what the row's ops must give; returns
    (largest float32 err / tol, uint8 pixels with two admissible values, uint8 pixels) for bounded rows, else None."""
    name, arg, dt, T, H, W, layout, n_clips, div, content = row
    u8 = dt == "u8"
    vals = case["vals"]
    worst, loose, total = 0.0, 0, 0
    for c in range(n_clips):
        video, op, rec = vals[c // div], case["ops"][c], case["recs"][c]
        what = "%s clip %d" % (_rid(row), c)
        if op is None or rec[0] == 0:
            _same_bits(got[c], video, what + " identity")
            continue
        if (name, arg) in EXACT_OPS:
            if n_clips > 100 and c % 97:
                continue
            _same_bits(got[c], AO.apply_op(video, name, arg), what)
            continue
        g = got[c].numpy().astype(f64)
        for t in range(T):
            v = video[t].numpy().astype(f32)
            lo, hi, ref, tol = bounded_range(v, rec, u8)
            bad = (g[t] < lo) | (g[t] > hi)
            assert not bad.any(), "%s frame %d: %d values outside the float64 bound, first got %r allowed [%r, %r]" % (
                what, t, int(bad.sum()), g[t][bad][0], lo[bad][0], hi[bad][0])
            if u8:
                loose += int((lo != hi).sum())
                total += lo.size
            else:
                worst = max(worst, float((np.abs(g[t] - ref) / tol).max()))
        if rec[0] in (4, 10):       # the kernel fixes the whole operation order: equal to the fp32 restatement
            emu = np.stack([emulate_frame(video[t].numpy().astype(f32), rec, u8) for t in range(T)])
            _same_bits(got[c], torch.from_numpy(emu.astype(np.uint8) if u8 else emu), what + " fp32 restatement")
        if H * W <= 64 * 80:        # torchvision's own result, at the tier of test_gpu_augment.py
            want = AO.apply_op(video, name, arg)
            d = (got[c].double() - want.double()).abs()
            if u8:
                assert float(d.max()) <= 1.0, (what, float(d.max()))
                if bool((d > 0).any()):
                    near = AO.near_boundary(AO.pre_cast64(video, name, arg))
                    assert bool(near[got[c] != want].all()), what + ": differs from torchvision away from a cast boundary"
            else:
                assert float(d.max()) <= 1e-5, (what, float(d.max()))
    if (name, arg) in EXACT_OPS:
        return None
    return worst, loose, total


def stats_check(row, case, stats):
    """augment_stats_kernel's records (structured array [n_clips * T]) against exact references."""
    name, arg, dt, T, H, W, layout, n_clips, div, content = row
    u8 = dt == "u8"
    for c in range(n_clips):
        for t in range(T):
            v = case["vals"][c // div, t].numpy().astype(f32)
            mn, mx, gsum, lut = frame_stats(v, u8)
            s = stats[c * T + t]
            what = "%s clip %d frame %d" % (_rid(row), c, t)
            assert np.array_equal(s["mn"], mn) and np.array_equal(s["mx"], mx), (what, s["mn"], mn, s["mx"], mx)
            assert np.array_equal(s["lut"], lut), what + ": Equalize table differs from torchvision's"
            if u8:
                assert s["gray_sum"] == gsum, (what, s["gray_sum"], gsum)
            else:                   # a double sum of H * W fp32 values in another order
                assert abs(s["gray_sum"] - gsum) <= 2.0 ** -52 * H * W * max(gsum, 1.0), (what, s["gray_sum"], gsum)


def _ops_device(recs):
    arr = AUG._ops_array(recs)
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(_dev())


@pytest.mark.gpu
@pytest.mark.parametrize("row", AUG_ROWS, ids=[_rid(r) for r in AUG_ROWS])
def test_augment_row(row):
    name, arg, dt, T, H, W, layout, n_clips, div, content = row
    L = _L()
    case = aug_case(row)
    buf, strides = _aug_src_buffer(case["vals"], layout)
    d = _aug_desc(row, strides)
    dev = _dev()
    src = buf.to(dev)
    n_out = n_clips * T * 3 * H * W
    dst = _sentinel(n_out + TAIL, TDT[dt]).to(dev)
    ops_d = _ops_device(case["recs"])
    stats_d, ran = None, []
    if name in STATS_OPS:
        nb = n_clips * T * ctypes.sizeof(L.AugFrameStats)
        stats_d = _sentinel(nb + TAIL, torch.uint8).to(dev)
        launched = _launch("pv_augment_stats", ctypes.byref(d), src.data_ptr(), stats_d.data_ptr(), _stream())
        _expect(aug_instance("stats", dt), launched)
        ran += sorted(launched)
        sb = stats_d.cpu()
        mask = torch.zeros(sb.numel(), dtype=torch.bool)
        mask[:nb] = True
        _assert_untouched(sb, mask, "stats")
        stats_check(row, case, np.frombuffer(sb[:nb].numpy().tobytes(), dtype=STATS_NP))
    launched = _launch("pv_augment_apply", ctypes.byref(d), src.data_ptr(), ops_d.data_ptr(),
                       None if stats_d is None else stats_d.data_ptr(), dst.data_ptr(), _stream())
    _expect(aug_instance("apply", dt), launched)
    ran += sorted(launched)
    out = dst.cpu()
    mask = torch.zeros(out.numel(), dtype=torch.bool)
    mask[:n_out] = True
    _assert_untouched(out, mask, "dst")
    res = aug_check(row, case, out[:n_out].view(n_clips, T, 3, H, W))
    if res is None:
        print("RATIO augment %s 0.0000 0.0000 %s bit-exact" % (_rid(row), ran))
    else:
        print("RATIO augment %s %.4f %.6f %s" % (_rid(row), res[0], res[1] / max(res[2], 1), ran))


def test_stats_record_layout():
    assert STATS_NP.itemsize == ctypes.sizeof(_L().AugFrameStats) == 800


# ---- AugMix mix ----------------------------------------------------------------------------------------------------------
AUGMIX_ROWS = [
    # (dtype, width, m, T, H, W, layout, n_clips)
    ("u8", 1, "drawn", 2, 5, 7, "cont", 2), ("u8", 3, "drawn", 2, 17, 31, "wslice", 3), ("u8", 5, "drawn", 1, 9, 1, "thwc", 2),
    ("u8", 3, 0.0, 2, 3, 3, "cont", 1), ("u8", 3, 1.0, 2, 16, 16, "thwc", 2),
    ("f32", 1, "drawn", 2, 1, 7, "thwc", 2), ("f32", 3, "drawn", 1, 64, 80, "cont", 2), ("f32", 5, "drawn", 2, 15, 16, "wslice", 3),
    ("f32", 3, 0.0, 2, 1, 1, "wslice", 2), ("f32", 5, 1.0, 2, 17, 31, "cont", 1),
]


def augmix_case(row):
    dt, width, m, T, H, W, layout, n_clips = row
    g = _gen(row)
    shape = (n_clips, T, 3, H, W)
    if dt == "u8":
        x = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
        ch = torch.randint(0, 256, (n_clips, width) + shape[1:], generator=g, dtype=torch.uint8)
        x.view(-1)[:2] = torch.tensor([0, 255], dtype=torch.uint8)
        ch.view(-1)[:2] = torch.tensor([255, 0], dtype=torch.uint8)
    else:
        x, ch = torch.rand(shape, generator=g), torch.rand((n_clips, width) + shape[1:], generator=g)
    w = torch.rand(n_clips, width, generator=g) + 0.05
    w = (w / w.sum(1, keepdim=True)).float()
    ms = [float(torch.rand(1, generator=g)) if m == "drawn" else m for _ in range(n_clips)]
    mix = torch.tensor([[float(v) for v in w[c]] + [ms[c], 1.0 - ms[c]] for c in range(n_clips)], dtype=torch.float32)
    return dict(x=x, chains=ch, w=w, m=ms, mix=mix)


def augmix_expected(row, case):
    return torch.stack([AO.mix_chains(case["x"][c], case["w"][c], case["m"][c], list(case["chains"][c]))
                        for c in range(row[7])])


def augmix_emulate(row, case, mutation=None):
    """augment_mix_kernel in numpy float32."""
    dt, width, m, T, H, W, layout, n_clips = row
    x, ch, mix = case["x"].numpy().astype(f32), case["chains"].numpy().astype(f32), case["mix"].numpy()
    out = np.empty_like(x)
    for c in range(n_clips):
        mixed = np.zeros_like(x[c])
        for k in (range(width - 1, -1, -1) if mutation == "reverse" else range(width)):
            mixed = mixed + mix[c, k] * ch[c, k]
        out[c] = mix[c, width] * x[c] + mix[c, width + 1] * mixed
    if dt == "u8":
        return torch.from_numpy((np.rint(out) if mutation == "round" else np.trunc(out)).astype(np.uint8))
    return torch.from_numpy(out)


@pytest.mark.gpu
@pytest.mark.parametrize("row", AUGMIX_ROWS, ids=[_rid(r) for r in AUGMIX_ROWS])
def test_augment_mix_row(row):
    dt, width, m, T, H, W, layout, n_clips = row
    case = augmix_case(row)
    buf, strides = _aug_src_buffer(case["x"], layout)
    d = _aug_desc((None, None, dt, T, H, W, layout, n_clips, 1, None), strides)
    dev = _dev()
    n_out = n_clips * T * 3 * H * W
    dst = _sentinel(n_out + TAIL, TDT[dt]).to(dev)
    src, ch, mix = buf.to(dev), case["chains"].contiguous().to(dev), case["mix"].to(dev)
    launched = _launch("pv_augment_mix", ctypes.byref(d), src.data_ptr(), ch.data_ptr(), width, mix.data_ptr(),
                       dst.data_ptr(), _stream())
    _expect(aug_instance("mix", dt), launched)
    out = dst.cpu()
    mask = torch.zeros(out.numel(), dtype=torch.bool)
    mask[:n_out] = True
    _assert_untouched(out, mask, "dst")
    _same_bits(out[:n_out].view(n_clips, T, 3, H, W), augmix_expected(row, case), _rid(row))
    print("RATIO augmix %s 0.0000 0.0000 %s bit-exact" % (_rid(row), sorted(launched)))


# =====================================================================================================================
# pv_mix.cu
# =====================================================================================================================
MIX_SIZE = (3, 2, 4, 8)          # (C, T, H, W): 192 elements


def _mix_layout(kind, es):
    """(sizes, strides, batch stride, base offset in elements) of a clip layout."""
    C, T, H, W = MIX_SIZE
    n = C * T * H * W
    if kind == "dense":
        return MIX_SIZE, (T * H * W, H * W, W, 1), n, 0
    if kind == "off1":               # the base pointer one element past a 16-byte boundary
        return MIX_SIZE, (T * H * W, H * W, W, 1), n, 1
    if kind == "sbatch":             # batch stride not a multiple of 16 bytes
        return MIX_SIZE, (T * H * W, H * W, W, 1), n + 1, 0
    if kind == "nodd":               # clip bytes not a multiple of 16
        return (3, 1, 5, 7), (35, 35, 7, 1), 112, 0
    if kind == "perm1":              # channels-last with a size-1 dim whose stride is arbitrary: dense in another order
        return (3, 1, 4, 8), (1, 999, 24, 3), 96, 0
    if kind == "cl":                 # (T, H, W, C) storage
        return MIX_SIZE, (1, H * W * C, W * C, C), n, 0
    if kind == "sliced":             # a W-slice of wider rows
        Wp = W + 3
        return MIX_SIZE, (T * H * Wp, H * Wp, Wp, 1), C * T * H * Wp + 8, 0
    if kind == "one":                # one-element clips
        return (1, 1, 1, 1), (1, 1, 1, 1), 1, 0
    raise KeyError(kind)


def mixup_dispatch(kind, dt):
    """pv_mixup's rule restated: ("vec" | "flat" | "strided", why) for a layout."""
    es = {"f16": 2, "f32": 4}[dt]
    sizes, strides, s_batch, off = _mix_layout(kind, es)
    dims = sorted((st, sz) for sz, st in zip(sizes, strides) if sz > 1)
    expect, dense = 1, True
    for st, sz in dims:
        dense &= st == expect
        expect *= sz
    if not dense:
        return "strided", "not dense"
    if (expect * es) % 16:
        return "flat", "clip bytes"
    if (s_batch * es) % 16:
        return "flat", "batch stride"
    if (off * es) % 16:
        return "flat", "pointer"
    return "vec", "aligned"


def mixup_instance(kind, dt):
    return "mixup_%skernel<%s>" % ("vec_" if mixup_dispatch(kind, dt)[0] == "vec" else "", CT[dt])


MIXUP_ROWS = [(dt, B, lam, kind, "rand") for dt in ("f16", "f32")
              for (B, lam, kind) in ((2, "drawn", "dense"), (3, 0.5, "dense"), (8, 0.0, "dense"), (3, 1.0, "off1"),
                                     (2, "drawn", "off1"), (8, "drawn", "sbatch"), (3, "drawn", "nodd"),
                                     (2, 0.5, "perm1"), (3, "drawn", "perm1"), (8, "drawn", "cl"), (3, 0.0, "sliced"),
                                     (2, 1.0, "sliced"), (8, "drawn", "sliced"), (131070, "drawn", "one"))]
MIXUP_ROWS += [("f16", 3, lam, kind, "special") for lam in (0.5, "drawn", 0.0, 1.0) for kind in ("dense", "sliced")]


def _lam(row, g):
    lam = row[2]
    lam = f32(float(torch.rand(1, generator=g)) if lam == "drawn" else lam)
    return float(lam), float(f32(1.0) - lam)


def mixup_case(row):
    dt, B, lam, kind, values = row
    g = _gen(row)
    sizes = _mix_layout(kind, 0)[0]
    x = (torch.randn((B,) + tuple(sizes), generator=g) * 3).to(TDT[dt])
    if values == "special":     # f16: ties of the product, subnormals, the largest value, inf, NaN, signed zeros
        sp = torch.tensor([65504.0, -65504.0, float("inf"), float("-inf"), float("nan"), 0.0, -0.0, 6e-8, -6e-8,
                           5.97e-8, 3e-5, 6.1e-5, 1.0009765625, 3.0, 2049.0, 2051.0, 0.333251953125, 1e-7])
        x.view(B, -1)[:, :len(sp)] = sp.to(TDT[dt])
        x.view(B, -1)[1, :len(sp)] = sp.flip(0).to(TDT[dt])
    lam_f, oml_f = _lam(row, g)
    return dict(x=x, lam=lam_f, oml=oml_f)


def _mix_buffer(x, kind):
    """In-place buffer: sentinel everywhere, the clip values at their strided places; (buffer, index, offset)."""
    es = x.element_size()
    sizes, strides, s_batch, off = _mix_layout(kind, es)
    B = x.shape[0]
    idx = _strided_index((B,) + tuple(sizes), (s_batch,) + tuple(strides), off)
    # 16-byte aligned device allocations: the row's offset alone decides the pointer's alignment
    buf = _sentinel(int(idx.max()) + 1 + TAIL, x.dtype)
    buf[idx.reshape(-1)] = x.reshape(-1)
    return buf, idx, off


def _mix_desc(B, dt, kind):
    L = _L()
    sizes, strides, s_batch, off = _mix_layout(kind, 0)
    d = L.MixDesc()
    d.B, d.dtype = B, _code(dt)
    d.size = (ctypes.c_longlong * 4)(*sizes)
    d.stride = (ctypes.c_longlong * 4)(*strides)
    d.s_batch = s_batch
    return d


def mixup_emulate(x, lam, oml, mutation=None):
    """mix1 of pv_mix.cu in torch: fp32 products, every intermediate stored in the element type."""
    a, b = x.float(), x.flip(0).float()
    lam_t, oml_t = torch.tensor(lam, dtype=torch.float32), torch.tensor(oml, dtype=torch.float32)
    if mutation == "round_once":
        return (a * lam_t + b * oml_t).to(x.dtype)
    return ((a * lam_t).to(x.dtype).float() + (b * oml_t).to(x.dtype).float()).to(x.dtype)


def _check_inplace(out, idx, want, what):
    mask = torch.zeros(out.numel(), dtype=torch.bool)
    mask[idx.reshape(-1)] = True
    _assert_untouched(out, mask, what)
    _same_bits(out[idx.reshape(-1)].view(want.shape), want, what)


@pytest.mark.gpu
@pytest.mark.parametrize("row", MIXUP_ROWS, ids=[_rid(r) for r in MIXUP_ROWS])
def test_mixup_row(row):
    dt, B, lam, kind, values = row
    case = mixup_case(row)
    buf, idx, off = _mix_buffer(case["x"], kind)
    d = _mix_desc(B, dt, kind)
    xd = buf.to(_dev())
    assert xd.data_ptr() % 16 == 0
    launched = _launch("pv_mixup", ctypes.byref(d), xd.data_ptr() + off * buf.element_size(), case["lam"], case["oml"],
                       _stream())
    _expect(mixup_instance(kind, dt), launched)
    idx0 = idx                                           # offsets include the base offset
    _check_inplace(xd.cpu(), idx0, MO.mixup(case["x"], case["lam"], case["oml"]), _rid(row))
    print("RATIO mixup %s 0.0000 0.0000 %s bit-exact" % (_rid(row), sorted(launched)))


CUTMIX_BOXES = {   # (yl, yh, xl, xh) on the 4 x 8 frame
    "tl": (0, 1, 0, 1), "tr": (0, 1, 7, 8), "bl": (3, 4, 0, 1), "br": (3, 4, 7, 8), "whole": (0, 4, 0, 8),
    "row": (2, 3, 0, 8), "col": (0, 4, 5, 6), "empty-h": (2, 2, 1, 5), "empty-w": (1, 3, 4, 4), "inner": (1, 3, 2, 7),
}
CUTMIX_ROWS = [(dt, B, box, layout) for dt, B, layout in (("u8", 2, "dense"), ("f16", 3, "cl"), ("f32", 5, "sliced"))
               for box in CUTMIX_BOXES]
CUTMIX_ROWS += [("u8", 5, "inner", "sliced"), ("u8", 3, "whole", "cl"), ("f16", 2, "inner", "sliced"),
                ("f16", 8, "row", "dense"), ("f32", 2, "col", "cl"), ("f32", 3, "inner", "dense")]


def cutmix_case(row):
    """Clips as raw bit patterns (every float pattern: NaN payloads, -0.0, subnormals), viewed in the row's type."""
    dt, B, box, layout = row
    g = _gen(row)
    it = INT[TDT[dt]]
    info = torch.iinfo(it)
    bits = torch.randint(info.min, info.max + 1, (B,) + MIX_SIZE, generator=g, dtype=torch.int64).to(it)
    if dt != "u8":
        z = torch.tensor([-0.0, float("nan")], dtype=TDT[dt]).view(it)
        bits[:, 0, 0, 1:3, 2] = z
    return bits


def cutmix_emulate(bits, box, mutation=None):
    yl, yh, xl, xh = box
    if mutation == "box_off_by_one":
        yh, xh = yh + (yh < bits.shape[-2]), xh + (xh < bits.shape[-1])
    return MO.cutmix(bits, (yl, yh, xl, xh))


@pytest.mark.gpu
@pytest.mark.parametrize("row", CUTMIX_ROWS, ids=[_rid(r) for r in CUTMIX_ROWS])
def test_cutmix_row(row):
    dt, B, box, layout = row
    bits = cutmix_case(row)
    buf, idx, off = _mix_buffer(bits.view(TDT[dt]), layout)
    d = _mix_desc(B, dt, layout)
    xd = buf.to(_dev())
    yl, yh, xl, xh = CUTMIX_BOXES[box]
    launched = _launch("pv_cutmix", ctypes.byref(d), xd.data_ptr(), yl, yh, xl, xh, _stream())
    empty = yl == yh or xl == xh
    _expect(None if empty else "cutmix_kernel<%d>" % buf.element_size(), launched)
    want = MO.cutmix(bits, CUTMIX_BOXES[box])
    if B % 2:
        assert torch.equal(want[B // 2], bits[B // 2])
    out = xd.cpu()
    mask = torch.zeros(out.numel(), dtype=torch.bool)
    mask[idx.reshape(-1)] = True
    _assert_untouched(out, mask, _rid(row))
    got = _bits(out)[idx.reshape(-1)].view(bits.shape)
    assert torch.equal(got, want), "%s: %d elements differ" % (_rid(row), int((got != want).sum()))
    print("RATIO cutmix %s 0.0000 0.0000 %s bit-exact" % (_rid(row), sorted(launched)))


LABEL_ROWS = [
    # (kind, mode, B, K, label smoothing, layout, bad label: None | "high" | "neg")
    ("index", 0, 5, 1000, 0.1, "dense", None), ("index", 0, 2, 1, 0.0, "dense", None), ("index", 0, 3, 7, 0.3, "strided", None),
    ("index", 1, 5, 1000, 0.1, "dense", None), ("index", 1, 3, 1, 0.2, "strided", None),
    ("index", 2, 4, 1000, 0.0, "dense", None), ("index", 2, 3, 5, 0.0, "strided", None),
    ("index", 0, 5, 7, 0.1, "dense", "high"), ("index", 0, 5, 7, 0.1, "strided", "neg"), ("index", 2, 3, 1, 0.0, "dense", "high"),
    ("index", 1, 1, 9, 0.1, "dense", "neg"),
    ("onehot", 0, 5, 1000, 0.0, "dense", None), ("onehot", 0, 3, 1, 0.0, "strided", None), ("onehot", 0, 2, 7, 0.0, "strided", None),
    ("onehot", 0, 1, 7, 0.0, "dense", None),
]


def label_case(row):
    kind, mode, B, K, ls, layout, bad = row
    g = _gen(row)
    lam, oml = _lam((None, None, "drawn"), g)
    on = float(torch.tensor(1.0 - ls + ls / K, dtype=torch.float32)) if mode != 2 else 1.0
    off = float(torch.tensor(ls / K, dtype=torch.float32)) if mode != 2 else 0.0
    if kind == "index":
        lab = torch.randint(0, K, (B,), generator=g)
        if bad:
            lab[B // 2] = K if bad == "high" else -1
        rows = torch.full((B, K), off, dtype=torch.float32)
        ok = (lab >= 0) & (lab < K)
        rows[torch.arange(B)[ok], lab[ok]] = on
        if not bad and mode != 2:
            assert torch.equal(rows, MO.one_hot_rows(lab, K, ls))
    else:
        lab = torch.rand(B, K, generator=g)
        rows = lab
    if mode == 0:
        want = rows * lam + rows.flip(0) * oml
        if not bad:
            assert torch.equal(want, MO.mix_labels(lab, K, lam, oml, ls, kind == "onehot"))
    else:
        want = rows if mode == 1 else rows.long()
    return dict(lab=lab, want=want, lam=lam, oml=oml, on=on, off=off, flag={None: 0, "high": 1, "neg": 2}[bad])


@pytest.mark.gpu
@pytest.mark.parametrize("row", LABEL_ROWS, ids=[_rid(r) for r in LABEL_ROWS])
def test_mix_labels_row(row):
    kind, mode, B, K, ls, layout, bad = row
    L = _L()
    case = label_case(row)
    lab = case["lab"]
    s_row, s_col = ((K * 2 + 3, 2) if kind == "onehot" else (3, 0)) if layout == "strided" else \
                   ((K, 1) if kind == "onehot" else (1, 0))
    big = 60000.0 if kind == "onehot" else -7
    idx = _strided_index(lab.shape, (s_row, s_col)[:lab.dim()])
    lbuf = torch.full((int(idx.max()) + 4,), big, dtype=lab.dtype)
    lbuf[idx.reshape(-1)] = lab.reshape(-1)
    d = L.MixLabelDesc()
    d.B, d.K, d.one_hot, d.mode = B, K, int(kind == "onehot"), mode
    d.lam, d.oml, d.on, d.off = case["lam"], case["oml"], case["on"], case["off"]
    d.s_row, d.s_col = s_row, s_col
    dev = _dev()
    odt = torch.int64 if mode == 2 else torch.float32
    out = _sentinel(B * K + TAIL, odt).to(dev)
    flag = torch.full((1 + TAIL,), 0x5A, dtype=torch.int32).to(dev)
    ld = lbuf.to(dev)
    launched = _launch("pv_mix_labels", ctypes.byref(d), ld.data_ptr(), out.data_ptr(),
                       None if kind == "onehot" else flag.data_ptr(), _stream())
    _expect("mix_labels_kernel<%s>" % kind, launched)
    o = out.cpu()
    mask = torch.zeros(o.numel(), dtype=torch.bool)
    mask[:B * K] = True
    _assert_untouched(o, mask, "out")
    _same_bits(o[:B * K].view(B, K), case["want"], _rid(row))
    fl = flag.cpu()
    assert bool((fl[1:] == 0x5A).all())
    assert int(fl[0]) == (0x5A if kind == "onehot" else case["flag"]), (int(fl[0]), case["flag"])
    print("RATIO labels %s 0.0000 0.0000 %s bit-exact" % (_rid(row), sorted(launched)))


# =====================================================================================================================
# pv_colorjitter.cu
# =====================================================================================================================
def _perms4():
    import itertools
    return [list(p) for p in itertools.permutations(range(4))]


def _view(order=(), factors=(1.0, 1.0, 1.0), hue=0.0, gray=False, sigma=None, clip=0):
    return dict(order=list(order), factors=tuple(float(f32(f)) for f in factors), hue=hue, gray=gray, sigma=sigma,
                clip=clip)


def _view_sets(kind):
    F = (1.3, 0.6, 1.7)
    if kind == "orders":         # every order of the four ops, then every prefix length
        vs = [_view(p, F, 0.37 if i % 2 else -0.21, clip=i % 2) for i, p in enumerate(_perms4())]
        vs += [_view([3, 1, 0, 2][:n], (0.5, 1.8, 0.0), 0.5, gray=bool(n % 2), clip=n % 2) for n in range(5)]
        return vs
    if kind == "mixed":          # views without Contrast (the stats block returns early) between views with it
        return [_view([0, 2], F, 0.1, sigma=0.1), _view([2, 1], F, 0.0, gray=True, sigma=2.0, clip=1), _view(),
                _view([1], (1.0, 0.2, 1.0), sigma=1.0), _view([3], F, -0.5, clip=1, sigma=8.0), _view([0, 3, 1], F, 0.499)]
    if kind == "blur2":          # the two views of the contrastive chain, both blurred
        return [_view([1, 3], F, 0.3, sigma=2.0), _view([2, 0], F, -0.1, gray=True, sigma=0.1, clip=1),
                _view([3, 1, 2, 0], F, 0.2, sigma=1.1)]
    if kind == "wide":           # a blur radius beyond the image's width and height
        return [_view([1], F, sigma=8.0), _view([], F, sigma=30.0, clip=1), _view([0], F, gray=True)]
    raise KeyError(kind)


CJ_ROWS = [
    # (source, n_t, H, W, views, layout, frame order)
    ("u8", 2, 9, 13, "orders", "cont", "id"), ("f32s0", 2, 9, 13, "orders", "thwc", "id"),
    ("f32s1", 3, 7, 5, "orders", "wslice", "rep"), ("u8", 3, 8, 1, "mixed", "wslice", "rep"),
    ("u8", 1, 1, 1, "mixed", "cont", "id"), ("f32s0", 2, 5, 300, "mixed", "cont", "rep"),
    ("f32s1", 2, 33, 47, "mixed", "thwc", "id"), ("u8", 1, 3, 4, "wide", "thwc", "id"),
    ("f32s0", 2, 2, 3, "wide", "wslice", "rep"), ("u8", 4, 70, 65, "mixed", "cont", "rep"),
    # the vertical blur's strip width and shared-memory size follow the stacked height (see vblur_plan)
    ("u8", 3, 256, 40, "blur2", "cont", "id"),            # 768 rows: strip 32, 48 KiB, no opt-in
    ("u8", 8, 224, 224, "blur2", "cont", "id"),           # 1792 rows: strip 16, 56 KiB (the contrastive workload)
    ("f32s1", 8, 224, 43, "blur2", "thwc", "rep"),        # partial last strip
    ("u8", 8, 400, 19, "blur2", "wslice", "id"),          # 3200 rows: strip 8
    ("f32s0", 1, 24600, 3, "blur2", "cont", "id"),        # strip 1
    ("u8", 2, 12300, 1, "blur2", "cont", "rep"),          # strip 1, W = 1
]


def vblur_plan(rows):
    """(strip, dynamic shared memory bytes) pv_colorjitter_vblur picks for a stack of ``rows`` rows."""
    s = 32
    while s > 1 and 2 * s * rows > 96 * 1024:
        s >>= 1
    return s, 2 * s * rows


def cj_case(row):
    src, n_t, H, W, views, layout, order = row
    g = _gen(row)
    T = n_t + 1
    shape = (2, 3, T, H, W)
    if src == "u8":
        x = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
    else:
        k = torch.randint(0, 256, shape, generator=g).float()
        x = k / 255.0                                       # exactly k / 255
        r = torch.rand(shape, generator=g)
        x = torch.where(r < 0.3, torch.nextafter(x, torch.zeros(())), x)
        x = torch.where((r >= 0.3) & (r < 0.5), torch.rand(shape, generator=g) * 1.2 - 0.1, x)   # below 0, above 1
        if src == "f32s1":
            x = x * 255.0
    x[:, :, :, 0, 0] = x[:, :1, :, 0, 0]                    # grey pixels (s == 0)
    idx = list(range(n_t)) if order == "id" else [(T - 1 - 2 * i) % T for i in range(n_t)]
    return dict(x=x, idx=idx, views=_view_sets(views))


def cj_bytes(x, src):
    """The byte Pillow sees of each source element (src_byte of pv_colorjitter.cu)."""
    if src == "u8":
        return x.numpy()
    v = x.numpy().astype(f32)
    if src == "f32s1":
        v = v / f32(255)
    v = v * f32(255)
    return np.where(v <= 0, 0, np.where(v >= 255, 255, np.trunc(np.clip(v, 0, 255)))).astype(np.uint8)


def _blur_params(sigma):
    return None if sigma is None else CJ.box_blur_params(sigma)


def cj_expected(row, case, mutation=None):
    """(views [n, 3, n_t, H, W] uint8, Contrast's luma sums [n]) from oracle.color_ref."""
    src, n_t, H, W = row[:4]
    b = cj_bytes(case["x"], src)
    outs, sums = [], []
    for vw in case["views"]:
        img = np.ascontiguousarray(b[vw["clip"]][:, case["idx"]].reshape(3, n_t * H, W).transpose(1, 2, 0))
        s = 0
        for op in vw["order"]:
            if op == 0:
                img = CO.brightness(img, vw["factors"][0])
            elif op == 1:
                s = int(CO.rgb_to_l(img).astype(np.int64).sum())
                img = CO.contrast(img, vw["factors"][1])
            elif op == 2:
                img = CO.saturation(img, vw["factors"][2])
            else:
                img = CO.hue(img, vw["hue"])
        if vw["gray"]:
            img = CO.gray3(img)
        p = _blur_params(vw["sigma"])
        if p is not None:
            r, ww, fw = p
            for axis in (1, 0):
                for _ in range(3):
                    if mutation == "no_rounding_term":
                        a = np.moveaxis(img.astype(np.int64), axis, -1)
                        n = a.shape[-1]
                        xs = np.arange(n)
                        acc = sum(a[..., np.clip(xs + k, 0, n - 1)] for k in range(-r, r + 1))
                        far = a[..., np.clip(xs - r - 1, 0, n - 1)] + a[..., np.clip(xs + r + 1, 0, n - 1)]
                        img = np.moveaxis(((acc * ww + far * fw) >> 24).astype(np.uint8), -1, axis)
                    else:
                        img = CO.box_pass(img, r, ww, fw, axis)
        outs.append(img.transpose(2, 0, 1).reshape(3, n_t, H, W))
        sums.append(s)
    return torch.from_numpy(np.stack(outs)), sums


def _cj_src_buffer(x, layout):
    n, C, T, H, W = x.shape
    big = 0xEE if x.dtype == torch.uint8 else 60000.0
    if layout == "thwc":
        strides = (T * H * W * 4, 1, H * W * 4, W * 4, 4)
    elif layout == "wslice":
        Wp = W + 3
        strides = (3 * T * H * Wp + 7, T * H * Wp, H * Wp, Wp, 1)
    else:
        strides = (3 * T * H * W, T * H * W, H * W, W, 1)
    size = 1 + sum((d - 1) * s for d, s in zip(x.shape, strides))
    buf = torch.full((size + 16,), big, dtype=x.dtype)
    buf.as_strided(x.shape, strides).copy_(x)
    return buf, strides


def run_cj(row):
    src, n_t, H, W, views, layout, order = row
    L = _L()
    case = cj_case(row)
    vs = case["views"]
    draws = [CJ.ViewDraw(True, v["order"] + [i for i in range(4) if i not in v["order"]],
                         [v["factors"][i] if i in v["order"] else None for i in range(3)] +
                         [v["hue"] if 3 in v["order"] else None], v["gray"], v["sigma"]) for v in vs]
    table = torch.frombuffer(bytearray(bytes(CJ._encode(draws, [v["clip"] for v in vs]))), dtype=torch.uint8)
    buf, (s_clip, sc, st, sh, sw) = _cj_src_buffer(case["x"], layout)
    d = L.ColorJitterDesc()
    d.n_views, d.n_t, d.H, d.W = len(vs), n_t, H, W
    d.s_clip, d.sc, d.st, d.sh, d.sw = s_clip, sc, st, sh, sw
    d.src_dtype, d.src_scale = (L.PV_U8 if src == "u8" else L.PV_F32), int(src == "f32s1")
    dev = _dev()
    n_out = len(vs) * 3 * n_t * H * W
    dst = _sentinel(n_out + TAIL, torch.uint8).to(dev)
    sums = _sentinel(len(vs) + TAIL, torch.int64).to(dev)
    xd, vd = buf.to(dev), table.to(dev)
    it = torch.tensor(case["idx"], dtype=torch.int32, device=dev)
    ct = "uint8_t" if src == "u8" else "float"
    ran = []
    launched = _launch("pv_colorjitter_stats", ctypes.byref(d), xd.data_ptr(), it.data_ptr(), vd.data_ptr(),
                       sums.data_ptr(), _stream())
    _expect("colorjitter_stats_kernel<%s>" % ct, launched)
    ran += sorted(launched)
    launched = _launch("pv_colorjitter_apply", ctypes.byref(d), xd.data_ptr(), it.data_ptr(), vd.data_ptr(),
                       sums.data_ptr(), dst.data_ptr(), _stream())
    _expect("colorjitter_apply_kernel<%s>" % ct, launched)
    ran += sorted(launched)
    launched = _launch("pv_colorjitter_vblur", ctypes.byref(d), vd.data_ptr(), dst.data_ptr(), _stream())
    _expect("colorjitter_vblur_kernel", launched)
    ran += sorted(launched)
    want, want_sums = cj_expected(row, case)
    s = sums.cpu()
    assert bool((_bits(s[len(vs):]) == SENT[torch.int64]).all()), "sums: tail changed"
    assert s[:len(vs)].tolist() == want_sums, (s[:len(vs)].tolist(), want_sums)
    out = dst.cpu()
    mask = torch.zeros(out.numel(), dtype=torch.bool)
    mask[:n_out] = True
    _assert_untouched(out, mask, "dst")
    got = out[:n_out].view(want.shape)
    for k in range(len(vs)):
        n = int((got[k] != want[k]).sum())
        assert n == 0, "%s view %d (%s): %d bytes differ" % (_rid(row), k, vs[k], n)
    strip, smem = vblur_plan(n_t * H)
    print("RATIO colorjitter %s 0.0000 0.0000 %s bit-exact strip=%d smem=%d" % (_rid(row), ran, strip, smem))


@pytest.mark.gpu
@pytest.mark.parametrize("row", CJ_ROWS, ids=[_rid(r) for r in CJ_ROWS])
def test_colorjitter_row(row):
    run_cj(row)


@pytest.mark.gpu
def test_vblur_sizes_in_one_process_do_not_disturb_each_other():
    """The opt-in for more than 48 KiB of shared memory is a per-function attribute set to the size at hand: a short
    stack, then the tall ones (56 KiB, 50 KiB, strip 1), then the short one and the 56 KiB one again."""
    by_rows = {r[1] * r[2]: r for r in CJ_ROWS if r[4] == "blur2" and r[0] == "u8"}
    for rows in (768, 1792, 3200, 24600, 768, 1792):
        run_cj(by_rows[rows])


# =====================================================================================================================
# pv_boxes.cu
# =====================================================================================================================
BOX_STARTS = {   # n_boxes -> box_start
    "front-empty": lambda n: [0, 0, 0, n // 2, n], "mid-empty": lambda n: [0, n // 3, n // 3, n // 3, n],
    "last-empty": lambda n: [0, n // 2, n, n, n], "one-clip": lambda n: [0, n], "even": lambda n: [0, n // 4, n // 2, n],
    "only-last": lambda n: [0, 0, 0, n],
}
SRC_CHAIN, CROP_CHAIN = 1 | 2 | 4 | 8, 2 | 4 | 8 | 16 | 32
BOX_ROWS = [(dt, 130, "even", step, "desc", 0) for dt in ("f32", "f64") for step in (1, 2, 4, 8, 16, 32)]
BOX_ROWS += [
    # (dtype, n_boxes, box_start, steps, geometry from: the descriptor | per clip, in == out)
    ("f32", 1, "one-clip", SRC_CHAIN, "desc", 0), ("f64", 1, "only-last", CROP_CHAIN, "geom", 1),
    ("f32", 128, "front-empty", CROP_CHAIN, "geom", 0), ("f64", 128, "mid-empty", SRC_CHAIN, "geom", 1),
    ("f32", 129, "last-empty", CROP_CHAIN, "geom", 1), ("f64", 129, "front-empty", CROP_CHAIN, "desc", 0),
    ("f32", 1000, "mid-empty", 63, "geom", 0), ("f64", 1000, "last-empty", 63, "geom", 1),
    ("f32", 1000, "one-clip", SRC_CHAIN, "desc", 1), ("f64", 1000, "even", CROP_CHAIN, "geom", 0),
    ("f32", 0, "one-clip", 63, "desc", 0),
]
BOX_FRAME = dict(in_h=240, in_w=320, out_h=224, out_w=224)


def box_instance(dt):
    return "clip_boxes_kernel<%s>" % CT[dt]


def box_case(row):
    dt, n, start, steps, gsrc, inplace = row
    g = _gen(row)
    ndt = f32 if dt == "f32" else f64
    H, W = BOX_FRAME["in_h"], BOX_FRAME["in_w"]
    b = TS.synthetic_xyxy(max(n, 1), H, W, zlib.crc32(repr(row).encode()) % 1000, torch.float64).numpy()[:n]
    if n >= 8:
        b[0] = [np.nan, 3.0, 50.0, np.nan]
        b[1] = [-0.0, -0.0, 0.0, 7.5]
        b[2] = [-40.0, -1e-30, 1e6, 5000.0]
        b[3] = [W - 1.0, H - 1.0, float(W), float(H)]
        b[4] = [1 / 3, 2 / 3, 100 + 1 / 3, 200 + 1e-9]            # float64 values whose float RoI cast rounds
    b = b.astype(ndt)
    bs = BOX_STARTS[start](n)
    n_clips = len(bs) - 1
    geom = [[256 + 16 * c, 341 + 21 * c, int(torch.randint(0, 30, (1,), generator=g)),
             int(torch.randint(0, 100, (1,), generator=g)), c % 2, 0] for c in range(n_clips)]
    return dict(boxes=b, start=bs, geom=geom, n_clips=n_clips, desc=dict(new_h=256, new_w=341, top=17, left=60, hflip=1))


def boxes_ref(row, case, mutation=None):
    """clip_boxes_kernel in numpy, one rounding per operation in the boxes' own type; returns (boxes, rois)."""
    dt, n, start, steps, gsrc, inplace = row
    T = f32 if dt == "f32" else f64
    b = case["boxes"].copy()
    clip_of = np.searchsorted(np.asarray(case["start"][1:]), np.arange(n), side="right")
    fr = BOX_FRAME
    edge = 0 if mutation == "clip_to_size" else 1

    def clip(v, hi):
        return np.minimum(T(hi), np.maximum(T(0), v))

    def clip_all(b, w, h):
        b[:, 0::2] = clip(b[:, 0::2], w - edge)
        b[:, 1::2] = clip(b[:, 1::2], h - edge)
    per = []
    for k in range(n):
        gm = case["geom"][clip_of[k]] if gsrc == "geom" else [case["desc"][f] for f in ("new_h", "new_w", "top", "left", "hflip")]
        per.append(gm[:5])
    per = np.asarray(per, np.int64).reshape(n, 5)
    if steps & 1:
        clip_all(b, fr["in_w"], fr["in_h"])
    if steps & 2:
        f = np.where(fr["in_w"] < fr["in_h"], per[:, 0] / f64(fr["in_h"]), per[:, 1] / f64(fr["in_w"])).astype(T)
        b = b * f[:, None]
    if steps & 4:
        b[:, 0::2] = b[:, 0::2] - per[:, 3].astype(T)[:, None]
        b[:, 1::2] = b[:, 1::2] - per[:, 2].astype(T)[:, None]
    if steps & 8:
        clip_all(b, fr["out_w"], fr["out_h"])
    if steps & 16:
        fl = per[:, 4] != 0
        w = T(fr["out_w"])
        nx1, nx2 = (w - b[:, 2]) - T(1), (w - b[:, 0]) - T(1)
        b[:, 0], b[:, 2] = np.where(fl, nx1, b[:, 0]), np.where(fl, nx2, b[:, 2])
    if steps & 32:
        clip_all(b, fr["out_w"], fr["out_h"])
    rois = np.concatenate([clip_of.astype(f32)[:, None], b.astype(f32)], 1)
    return b, rois


@pytest.mark.gpu
@pytest.mark.parametrize("row", BOX_ROWS, ids=[_rid(r) for r in BOX_ROWS])
def test_boxes_row(row):
    dt, n, start, steps, gsrc, inplace = row
    L = _L()
    case = box_case(row)
    d = L.BoxesDesc()
    d.n_clips, d.n_boxes, d.steps, d.dtype = case["n_clips"], n, steps, L.BOX_F32 if dt == "f32" else L.BOX_F64
    for k, v in dict(BOX_FRAME, **case["desc"]).items():
        setattr(d, k, v)
    dev = _dev()
    tdt = TDT[dt]
    src = _sentinel(4 * n + TAIL, tdt)
    src[:4 * n] = torch.from_numpy(case["boxes"].reshape(-1))
    sd = src.to(dev)
    od = sd if inplace else _sentinel(4 * n + TAIL, tdt).to(dev)
    rois = _sentinel(5 * n + TAIL, torch.float32).to(dev)
    bs = torch.tensor(case["start"], dtype=torch.int32, device=dev)
    gm = torch.tensor(case["geom"], dtype=torch.int32, device=dev) if gsrc == "geom" else None
    launched = _launch("pv_clip_boxes_transform", ctypes.byref(d), sd.data_ptr(), bs.data_ptr(),
                       None if gm is None else gm.data_ptr(), od.data_ptr(), rois.data_ptr(), _stream())
    _expect(box_instance(dt) if n else None, launched)
    want, want_rois = boxes_ref(row, case)
    for buf, m, ref, what in ((od.cpu(), 4, want, "boxes"), (rois.cpu(), 5, want_rois, "rois")):
        mask = torch.zeros(buf.numel(), dtype=torch.bool)
        mask[:m * n] = True
        _assert_untouched(buf, mask, what)
        # zeros compare by value: numpy leaves the sign of maximum(0.0, -0.0) to its build (-0.0 with AVX-512, where
        # the kernel gives +0.0), so the reference does not fix it
        _same_bits(buf[:m * n].view(n, m) + 0.0, torch.from_numpy(ref) + 0.0, "%s %s" % (_rid(row), what))
    if not inplace:
        assert torch.equal(_bits(sd.cpu()), _bits(src)), "the input boxes changed"
    if n:
        assert want_rois[:, 0].tolist() == [float(c) for c in np.repeat(np.arange(case["n_clips"]), np.diff(case["start"]))]
    print("RATIO boxes %s 0.0000 0.0000 %s bit-exact" % (_rid(row), sorted(launched)))


# =====================================================================================================================
# CPU: ledger, argument limits, coverage, restatements and mutations
# =====================================================================================================================
def expected_instances():
    out = {aug_instance("apply", r[2]) for r in AUG_ROWS}
    out |= {aug_instance("stats", r[2]) for r in AUG_ROWS if r[0] in STATS_OPS}
    out |= {aug_instance("mix", r[0]) for r in AUGMIX_ROWS}
    out |= {mixup_instance(r[3], r[0]) for r in MIXUP_ROWS}
    out |= {"cutmix_kernel<%d>" % {"u8": 1, "f16": 2, "f32": 4}[r[0]] for r in CUTMIX_ROWS
            if CUTMIX_BOXES[r[2]][0] != CUTMIX_BOXES[r[2]][1] and CUTMIX_BOXES[r[2]][2] != CUTMIX_BOXES[r[2]][3]}
    out |= {"mix_labels_kernel<%s>" % r[0] for r in LABEL_ROWS}
    for r in CJ_ROWS:
        ct = "uint8_t" if r[0] == "u8" else "float"
        out |= {"colorjitter_stats_kernel<%s>" % ct, "colorjitter_apply_kernel<%s>" % ct, "colorjitter_vblur_kernel"}
    out |= {box_instance(r[0]) for r in BOX_ROWS if r[1]}
    return out


def test_ledger_launch_sites_are_the_rows_instances():
    names = set()
    for f in ("pv_augment.cu", "pv_mix.cu", "pv_colorjitter.cu", "pv_boxes.cu"):
        found = re.findall(r'PV_LAUNCH_OK\("([^"]+)"\)', open(os.path.join(CSRC, f)).read())
        assert found, f
        names |= set(found)
    want = expected_instances()
    assert len(names) == 22
    assert names == want, (sorted(names - want), sorted(want - names))


def test_frame_and_batch_limits_are_argument_errors():
    """One launch covers at most 65535 (clip, frame) pairs and 2 * 65535 clips; the next size is refused by the host
    check, before any launch (so this runs without a device)."""
    L = _L()
    lib = L.load()
    dummy = ctypes.create_string_buffer(64)
    p = ctypes.addressof(dummy)
    before = TS.kernel_counts()
    for n_clips, T in ((65536, 1), (4369, 16), (1, 65536)):
        d = _aug_desc((None, None, "u8", T, 1, 1, "cont", n_clips, 1, None), (T * 3, 3, 1, 1, 1))
        assert lib.pv_augment_apply(ctypes.byref(d), p, p, p, p, None) == -1
        assert "too many frames" in L.last_error()
        assert lib.pv_augment_stats(ctypes.byref(d), p, p, None) == -1
    for B in (131071, 131072, 1):
        d = _mix_desc(B, "f32", "one")
        assert lib.pv_mixup(ctypes.byref(d), p, 0.5, 0.5, None) == -1
        assert "131070" in L.last_error()
        assert lib.pv_cutmix(ctypes.byref(d), p, 0, 1, 0, 1, None) == -1
    assert max(r[7] * r[3] for r in AUG_ROWS) == 65535 and max(r[1] for r in MIXUP_ROWS) == 131070
    assert TS.kernel_count_diff(before, TS.kernel_counts()) == {}


def test_mixup_rows_take_every_dispatch_outcome():
    for dt in ("f16", "f32"):
        got = {mixup_dispatch(r[3], dt) for r in MIXUP_ROWS if r[0] == dt}
        assert got == {("vec", "aligned"), ("flat", "clip bytes"), ("flat", "batch stride"), ("flat", "pointer"),
                       ("strided", "not dense")}, got
    assert mixup_dispatch("perm1", "f32") == ("vec", "aligned") and mixup_dispatch("cl", "f16") == ("vec", "aligned")
    assert {r[1] for r in MIXUP_ROWS} >= {2, 3, 8, 131070}
    assert {r[2] for r in MIXUP_ROWS} == {0.0, 0.5, 1.0, "drawn"}
    # the f16 specials reach a tie, a subnormal and an overflow of the rounded sum
    row = next(r for r in MIXUP_ROWS if r[4] == "special" and r[2] == 0.5 and r[3] == "dense")
    case = mixup_case(row)
    x = case["x"].float()
    prod = x * 0.5
    assert bool(((prod.half().float() != prod) & torch.isfinite(prod)).any())
    out = MO.mixup(case["x"], 0.5, 0.5)
    assert bool(torch.isinf(out).any()) and bool(torch.isnan(out).any())
    assert bool(((out.float().abs() < 6.2e-5) & (out.float() != 0)).any())


def test_augment_rows_reach_their_edges():
    sizes = {(r[4], r[5]) for r in AUG_ROWS}
    assert set(AUG_SIZES) | {(720, 1280)} <= sizes
    for name, arg in EXACT_OPS + BOUNDED_OPS:
        mine = [r for r in AUG_ROWS if (r[0], r[1]) == (name, arg)]
        assert {(r[4], r[5]) for r in mine} >= set(AUG_SIZES), (name, arg)
        assert {r[2] for r in mine} == {"u8", "f32"} and {r[6] for r in mine} == set(AUG_LAYOUTS), (name, arg)
        assert {r[8] for r in mine} == {1, 3}, (name, arg)
    # statistics: more than one stride of the 512-thread loop, and fewer pixels than 255
    assert any(r[0] in STATS_OPS and r[4] * r[5] > 512 for r in AUG_ROWS)
    eq = [r for r in AUG_ROWS if r[0] == "Equalize" and r[4] * r[5] <= 224 * 224]
    kinds = set()
    for r in eq:
        case = aug_case(r)
        for c in range(3):
            v = case["vals"][0, 0, c].numpy().astype(f32)
            hist = np.bincount(_byte_of(v, r[2] == "u8").reshape(-1), minlength=256)
            ident = scale_channel_lut(hist) is None
            kinds.add((ident, bool((hist > 0).sum() > 1), r[4] * r[5] >= 255, r[2]))
    for dt in ("u8", "f32"):
        assert (True, True, False, dt) in kinds      # step == 0 on a varying frame with fewer than 255 pixels
        assert (True, True, True, dt) in kinds       # the last bin holds more than hw - 255 pixels
        assert (False, True, True, dt) in kinds      # a real table
    ac = aug_case(next(r for r in AUG_ROWS if r[0] == "AutoContrast" and r[4] * r[5] > 9))
    mn, mx, _, _ = frame_stats(ac["vals"][0, 0].numpy().astype(f32), False)
    assert mn[1] == mx[1] and mn[0] != mx[0]
    sol = aug_case(next(r for r in AUG_ROWS if r[:3] == ("Solarize", 0.5, "u8") and r[4] * r[5] >= 240))
    assert bool((sol["vals"] == 127).any()) and bool((sol["vals"] == 126).any())
    solf = aug_case(next(r for r in AUG_ROWS if r[:3] == ("Solarize", 0.5, "f32") and r[4] * r[5] >= 240))
    assert bool((solf["vals"] == 0.5).any())
    fl = aug_case(next(r for r in AUG_ROWS if r[:3] == ("Posterize", 7, "f32") and r[4] * r[5] >= 240))["vals"]
    k = fl * 255
    assert bool((fl == 0).any()) and bool((fl == 1).any()) and bool(((k == k.round()) & (fl > 0) & (fl < 1)).any())
    assert {r[1] for r in AUG_ROWS if r[0] == "Posterize"} == {0, 1, 7}
    assert any(r[0] == "AdjustSharpness" and (r[4], r[5]) == (3, 3) for r in AUG_ROWS)


def test_warp_rows_reach_the_discontinuities():
    seen = set()
    ties = 0
    for r in AUG_ROWS:
        name, arg, dt, T, H, W = r[:6]
        if (name, arg) not in WARP_OPS or H * W > 64 * 80:
            continue
        rec = AUG.encode_op((name, arg), TDT[dt], H, W, AO.FILL)
        x0, y0, wt, inside, tx, ty = affine_geometry(H, W, rec[4:10])
        if inside.any():
            seen |= {"x0=-1"} if (x0[inside] == -1).any() else set()
            seen |= {"y0=-1"} if (y0[inside] == -1).any() else set()
            seen |= {"x0=W-1"} if (x0[inside] == W - 1).any() else set()
            seen |= {"y0=H-1"} if (y0[inside] == H - 1).any() else set()
            seen |= {"tx=0"} if ((tx == 0) & inside).any() else set()
            seen |= {"tx=0.5"} if ((tx == 0.5) & inside).any() else set()
        seen |= {"outside"} if (~inside).any() else set()
        seen |= {"all-outside"} if not inside.any() else set()
        if dt == "u8" and H * W >= 240:
            v = aug_case(r)["vals"][0, 0].numpy().astype(f32)
            ref = bounded_range(v, rec, True)[2]
            ties += int((np.abs(ref - np.floor(ref) - 0.5) == 0).sum() - (~inside).sum() * 3)
    assert seen == {"x0=-1", "y0=-1", "x0=W-1", "y0=H-1", "tx=0", "tx=0.5", "outside", "all-outside"}, seen
    assert ties > 0, "no uint8 warp row has an exact .5 before rintf apart from the fill"


def test_other_rows_reach_their_edges():
    plans = {vblur_plan(r[1] * r[2]) for r in CJ_ROWS if r[4] == "blur2"}
    assert {s for s, _ in plans} == {32, 16, 8, 1}
    assert (32, 48 * 1024) in plans and (16, 56 * 1024) in plans           # the largest without, 8 x 224 with the opt-in
    assert any(m > 48 * 1024 for _, m in plans) and all(m <= 200 * 1024 for _, m in plans)
    assert any(r[3] % vblur_plan(r[1] * r[2])[0] for r in CJ_ROWS if r[4] == "blur2")
    assert any(r[3] == 1 for r in CJ_ROWS) and {r[0] for r in CJ_ROWS} == {"u8", "f32s0", "f32s1"}
    wide = next(r for r in CJ_ROWS if r[4] == "wide")
    assert max(_blur_params(v["sigma"])[0] for v in _view_sets("wide") if v["sigma"]) > max(wide[1] * wide[2], wide[3])
    assert {tuple(v["order"]) for v in _view_sets("orders")} >= {tuple(p) for p in _perms4()}
    assert {len(v["order"]) for v in _view_sets("orders")} == {0, 1, 2, 3, 4}
    assert any(CO.hue_shift(v["hue"]) + 200 > 255 for v in _view_sets("orders"))
    assert {_blur_params(s) is not None for s in (0.1, 2.0)} == {True}
    f = cj_case(next(r for r in CJ_ROWS if r[0] == "f32s0"))["x"]
    assert bool((f < 0).any()) and bool((f > 1).any())
    assert {r[1] for r in BOX_ROWS} == {0, 1, 128, 129, 130, 1000} and {r[2] for r in BOX_ROWS} == set(BOX_STARTS)
    assert {r[3] for r in BOX_ROWS} >= {1, 2, 4, 8, 16, 32, SRC_CHAIN, CROP_CHAIN}
    assert {(r[0], r[5]) for r in BOX_ROWS} >= {("f32", 0), ("f32", 1), ("f64", 0), ("f64", 1)}
    r64 = next(r for r in BOX_ROWS if r[0] == "f64" and r[1] >= 8 and r[3] == 2)
    b, rois = boxes_ref(r64, box_case(r64))
    assert bool((rois[:, 1:].astype(f64) != b)[np.isfinite(b)].any())
    assert {CUTMIX_BOXES[r[2]] for r in CUTMIX_ROWS} == set(CUTMIX_BOXES.values())
    assert {(r[0], r[3]) for r in CUTMIX_ROWS} >= {(dt, ly) for dt in ("u8", "f16", "f32") for ly in ("cl", "sliced")}
    assert any(r[1] % 2 for r in CUTMIX_ROWS) and any(r[1] % 2 == 0 for r in CUTMIX_ROWS)
    assert {(r[0], r[1]) for r in LABEL_ROWS} == {("index", 0), ("index", 1), ("index", 2), ("onehot", 0)}
    assert {r[6] for r in LABEL_ROWS} == {None, "high", "neg"} and {1, 1000} <= {r[3] for r in LABEL_ROWS}
    assert {r[1] for r in AUGMIX_ROWS} == {1, 3, 5} and {r[2] for r in AUGMIX_ROWS} == {0.0, 1.0, "drawn"}


CPU_AUG_ROWS = [r for r in AUG_ROWS if r[4] * r[5] <= 64 * 80 and r[7] < 100]


@pytest.mark.parametrize("row", CPU_AUG_ROWS, ids=[_rid(r) for r in CPU_AUG_ROWS])
def test_augment_restatement_passes_its_check(row):
    """The fp32 restatement of augment_apply_kernel equals torchvision on the exact ops and passes the float64 bound
    on the others, so a kernel that computes what its comments state passes its row."""
    case = aug_case(row)
    res = aug_check(row, case, aug_emulate(row, case))
    if res is not None:
        print("RATIO emulation-augment %s %.4f %.6f" % (_rid(row), res[0], res[1] / max(res[2], 1)))


def _arow(name, dt, pred=lambda r: r[4] * r[5] in (240, 256, 527)):
    return next(r for r in CPU_AUG_ROWS if r[0] == name and r[2] == dt and pred(r))


def _aug_mut(row, mutation):
    case = aug_case(row)
    aug_check(row, case, aug_emulate(row, case, mutation))


AUG_MUTATIONS = {
    "autocontrast_scale_in_one_division": (lambda: _arow("AutoContrast", "u8", lambda r: (r[4], r[5]) == (3, 3)),
                                           "one_division"),
    "saturation_blend_contracted": (lambda: _arow("AdjustSaturation", "f32"), "fma"),
    "sharpness_blurs_the_border_u8": (lambda: _arow("AdjustSharpness", "u8"), "blur_border"),
    "sharpness_blurs_the_border_f32": (lambda: _arow("AdjustSharpness", "f32"), "blur_border"),
    "equalize_table_not_shifted_u8": (lambda: _arow("Equalize", "u8", lambda r: r[9] == "rand" and r[4] * r[5] > 255),
                                      "lut_unshifted"),
    "equalize_table_not_shifted_f32": (lambda: _arow("Equalize", "f32", lambda r: r[9] == "rand" and r[4] * r[5] > 255),
                                       "lut_unshifted"),
    "solarize_gt_u8": (lambda: _arow("Solarize", "u8"), "solarize_gt"),
    "solarize_gt_f32": (lambda: _arow("Solarize", "f32", lambda r: r[1] == 0.3 and r[4] * r[5] >= 240), "solarize_gt"),
    "warp_truncates": (lambda: next(r for r in CPU_AUG_ROWS if r[0] == "Rotate" and r[2] == "u8" and r[4] * r[5] >= 240),
                       "warp_trunc"),
    "warp_drops_the_border_column_u8": (lambda: next(r for r in CPU_AUG_ROWS if r[0] == "TranslateX" and r[2] == "u8"
                                                     and abs(r[1]) == 0.28125 and r[5] >= 16), "ix_ge_0"),
    "warp_drops_the_border_column_f32": (lambda: next(r for r in CPU_AUG_ROWS if r[0] == "TranslateX" and r[2] == "f32"
                                                      and abs(r[1]) == 0.28125 and r[5] >= 16), "ix_ge_0"),
}


@pytest.mark.parametrize("name", sorted(AUG_MUTATIONS))
def test_augment_check_rejects_wrong_kernels(name):
    pick, mutation = AUG_MUTATIONS[name]
    row = pick()
    _aug_mut(row, None)
    with pytest.raises(AssertionError):
        _aug_mut(row, mutation)


def test_warp_cutoff_is_an_early_out_only():
    """`ix > -1` against `ix >= -1`: at ix == -1 the left taps are outside and the right taps have weight tx == 0, so
    the result is the fill either way; no test can tell the two apart, and none needs to."""
    hit = 0
    for r in CPU_AUG_ROWS:
        if r[0] not in ("TranslateX", "Rotate") or r[4] * r[5] < 9:
            continue
        case = aug_case(r)
        hit += int((affine_geometry(r[4], r[5], case["recs"][0][4:10], "ix_ge_m1")[3] !=
                    affine_geometry(r[4], r[5], case["recs"][0][4:10])[3]).sum())
        assert torch.equal(aug_emulate(r, case), aug_emulate(r, case, "ix_ge_m1")), _rid(r)
    assert hit > 0, "no row has a pixel at ix == -1"


@pytest.mark.parametrize("row", AUGMIX_ROWS, ids=[_rid(r) for r in AUGMIX_ROWS])
def test_augmix_restatement_is_the_oracle(row):
    case = augmix_case(row)
    want = augmix_expected(row, case)
    _same_bits(augmix_emulate(row, case), want, _rid(row))
    if row[1] >= 3 and row[2] == "drawn":
        for mutation in (("round",) if row[0] == "u8" else ("reverse",)):
            with pytest.raises(AssertionError):
                _same_bits(augmix_emulate(row, case, mutation), want, mutation)


CPU_MIXUP_ROWS = [r for r in MIXUP_ROWS if r[1] <= 8]


@pytest.mark.parametrize("row", CPU_MIXUP_ROWS, ids=[_rid(r) for r in CPU_MIXUP_ROWS])
def test_mixup_restatement_is_the_oracle(row):
    case = mixup_case(row)
    want = MO.mixup(case["x"], case["lam"], case["oml"])
    _same_bits(mixup_emulate(case["x"], case["lam"], case["oml"]), want, _rid(row))
    if row[0] == "f16" and row[2] == "drawn":
        with pytest.raises(AssertionError):
            _same_bits(mixup_emulate(case["x"], case["lam"], case["oml"], "round_once"), want, "round once")


def test_cutmix_box_off_by_one_is_visible():
    for row in CUTMIX_ROWS:
        bits = cutmix_case(row)
        box = CUTMIX_BOXES[row[2]]
        want = MO.cutmix(bits, box)
        assert torch.equal(cutmix_emulate(bits, box), want)
        if box[1] < 4 or box[3] < 8:
            assert not torch.equal(cutmix_emulate(bits, box, "box_off_by_one"), want), _rid(row)


def test_blur_without_the_rounding_term_is_visible():
    row = next(r for r in CJ_ROWS if r[4] == "mixed" and r[2] >= 33)
    case = cj_case(row)
    want, _ = cj_expected(row, case)
    bad, _ = cj_expected(row, case, "no_rounding_term")
    blurred = [k for k, v in enumerate(case["views"]) if _blur_params(v["sigma"])]
    assert blurred and all(not torch.equal(want[k], bad[k]) for k in blurred)
    # and the restatement used here is oracle.color_ref's whole chain
    b = cj_bytes(case["x"], row[0])
    for k, v in enumerate(case["views"]):
        img = np.ascontiguousarray(b[v["clip"]][:, case["idx"]].reshape(3, -1, row[3]).transpose(1, 2, 0))
        if _blur_params(v["sigma"]) is None and v["sigma"] is not None:
            continue
        ref = CO.color_jitter_view(img, v["order"], v["factors"], v["hue"], v["gray"], v["sigma"])
        assert np.array_equal(ref.transpose(2, 0, 1).reshape(want[k].shape), want[k].numpy()), k


def test_float_source_bytes_clamp_and_truncate():
    x = torch.tensor([-0.5, 0.0, 1.0, 1.5, 0.5, float(f32(7) / f32(255)), float(np.nextafter(f32(7) / f32(255), f32(0)))])
    assert cj_bytes(x, "f32s0").tolist() == [0, 0, 255, 255, 127, 7, 6]
    assert cj_bytes(x * 255, "f32s1").tolist()[:5] == [0, 0, 255, 255, 127]
    inside = torch.rand(1000, generator=torch.Generator().manual_seed(1))
    assert np.array_equal(cj_bytes(inside, "f32s0"), CO.to_bytes(inside.numpy()))


def test_boxes_clipped_to_size_is_visible():
    for row in BOX_ROWS:
        if row[1] < 8 or not row[3] & (1 | 8 | 32):
            continue
        case = box_case(row)
        good, bad = boxes_ref(row, case)[0], boxes_ref(row, case, "clip_to_size")[0]
        ok = ~np.isnan(good)
        assert not np.array_equal(good[ok], bad[ok]), _rid(row)

