"""The clip-transform, RoIAlign and view-reduce kernels against float64, one row per instance and edge.

These are the kernels a clip passes through before the model (pv_clip_transform_batch, pv_clip_transform_fwd,
pv_clip_transform_rrc) and the ones that turn model output into a detection or a video-level answer
(pv_roi_align_fwd, pv_view_reduce).  Every GPU test calls the C ABI directly (ctypes), so a row sets its own strides,
offsets and destination alignment.  It asserts from the library's launch counts which kernel instance ran, puts a
sentinel after every output buffer, between output clips and in output row padding and checks that they survive,
fills source row / channel padding with a large value (a kernel that reads it moves the result far), and compares:
  - bit-exact: the uint8 pass-through (against index_select plus crop) and view_reduce (against a torch fp32
    restatement of the reference's per-video loop: zeros, then += or torch.max in view order, then / count);
  - bounded (testing.assert_close_to_f64) for the resizing transforms and RoIAlign, against float64 at the fp32
    geometry ATen and torchvision define: the bilinear taps of oracle.transforms_ref.bilinear_table (pinned to ATen
    by test_oracle_pinning.py) with l0 = fl32(1 - l1), and oracle.interp.roi_align_ref's sample positions, indices,
    weights and count.  Everything after the geometry is float64.
CPU tests check that the compiled instances are exactly the reachable ones and that the rows reach all of them, that
an fp32 emulation of each bounded kernel passes its bound while known bugs fail it, and that the RoIAlign geometry
must be evaluated without FMA contraction (committed boxes where a contracted evaluation crosses a discontinuity).

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit), per bounded family: the largest err / tol, and in brackets
the largest share of the accumulation term a result used beyond its own storage rounding.  A correctly rounded f16
result may use nearly all of the rounding term, hence ratios near 1 with small shares:
  batch transform 0.998 (0.229), single-clip transform 0.991 (0.269), RandomResizedCrop mode 0.965 (0.104),
  RoIAlign 0.996 (0.330).
The uint8 pass-through and view_reduce matched bit for bit.  With the RoIAlign geometry contracted again (the build
before the explicit-rounding fix), all 12 'contract' rows failed, and so did three 'inside' rows (scales 1/16 and 1/4,
where only `start + ph * bin` contracts); each committed box on its own fails the bound under the contracted fp32
emulation (test_contraction_boxes_are_visible).  With view_reduce's "max" seeded from -inf and folded with fmaxf, the
all-negative and NaN max rows failed.

Not verified: the 2^31 offset guards of pv_clip_transform_batch (an output over 2 GB).
"""
import ctypes
import os
import re
import shutil
import subprocess
import zlib

import numpy as np
import pytest
import torch

from pytorchvideo_b200 import testing as TS
from oracle.transforms_ref import bilinear_table
from pytorchvideo_b200.transforms import functional as FV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorchvideo_b200", "csrc")

U = TS.F32_EPS
# Transforms: each tap value is three fp32 roundings from (|u'| + |mean|) / |std| (u' = u / 255 or u: the division by
# 255, the subtraction, the division by std); the blend adds two roundings per level of the nested lerp on the same
# magnitude (weights are the exact fp32 table weights, non-negative, summing to 1): 7 roundings, plus one of slack.
TR_EPS = 8 * U
TAIL = 64                       # sentinel elements after every output buffer
GAP = 5                         # sentinel elements between output clips
SENT = {torch.uint8: 0x5A, torch.float16: 0x5A5A, torch.float32: 0x5A5A5A5A}
INT = {torch.uint8: torch.uint8, torch.float16: torch.int16, torch.float32: torch.int32}
TDT = {"u8": torch.uint8, "f16": torch.float16, "f32": torch.float32}
CT = {"u8": "uint8_t", "f16": "__half", "f32": "float"}
BIG = {"u8": 255.0, "f16": 60000.0, "f32": 60000.0}    # source padding filler
MEAN = (0.45, 0.40, 0.35, 0.30)
STD = (0.225, 0.25, 0.20, 0.30)


def _dev():
    return torch.device("cuda:0")


def _L():
    from pytorchvideo_b200 import _lib as L
    return L


def _code(dt):
    L = _L()
    return {"u8": L.PV_U8, "f16": L.PV_F16, "f32": L.PV_F32}[dt]


def _rnd(dt):
    return TS.F16_EPS if dt == "f16" else TS.F32_EPS


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
    assert launched == {name: 1}, "expected one launch of %s, launched %s" % (name, launched)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bound(got, ref, absref, acc_eps, rnd, what):
    """TS.assert_close_to_f64 with k_len = 0 (acc_eps is the whole accumulation term); returns (err / tol, share of
    the accumulation term used beyond the storage rounding)."""
    r = TS.assert_close_to_f64(got, ref.reshape(got.shape), absref.reshape(got.shape), 0, acc_eps=acc_eps, what=what,
                               rnd_eps=rnd)
    return r[0], r[1]


def _ratio(family, row, ratio, launched):
    print("RATIO %s %s %.4f %.4f %s" % (family, _rid(row), ratio[0], ratio[1], sorted(launched)))


def _to_f16_trunc(v):
    """f32 -> f16 rounded toward zero (the bug the comparator's bias check must see)."""
    h = v.half()
    b = h.view(torch.int16).clone()
    over = h.float().abs() > v.abs()
    b[over] -= 1
    return b.view(torch.float16)


def _store(v, ddt, mutation=None):
    if ddt == "f16":
        return _to_f16_trunc(v) if mutation == "trunc16" else v.half()
    return v


# =====================================================================================================================
# Transforms: float64 reference and fp32 emulation on gathered taps
# =====================================================================================================================
def col_taps(in_w, new_w, left, out_w, flip, mutation=None, table=bilinear_table):
    """Column taps (i0, i1, l1) of output columns 0..out_w-1 from the ATen-pinned table (or another table)."""
    i0, i1, l1 = table(in_w, new_w)
    xo = np.arange(out_w)
    if flip:
        xo = (out_w - xo) if mutation == "flip_off" else (out_w - 1 - xo)
    pos = np.minimum(left + xo, new_w - 1)
    return i0[pos], i1[pos], l1[pos]


def row_taps(in_h, new_h, top, out_h, table=bilinear_table):
    i0, i1, l1 = table(in_h, new_h)
    return i0[top:top + out_h], i1[top:top + out_h], l1[top:top + out_h]


def _gather(S, yt, xt):
    """S [C, n, H, W] -> four tap planes [C, n, oh, ow] (v00, v01, v10, v11)."""
    y0, y1 = torch.as_tensor(yt[0]).long(), torch.as_tensor(yt[1]).long()
    x0, x1 = torch.as_tensor(xt[0]).long(), torch.as_tensor(xt[1]).long()
    r0, r1 = S[:, :, y0], S[:, :, y1]
    return r0[..., x0], r0[..., x1], r1[..., x0], r1[..., x1]


def _weights(yt, xt, dtype):
    ly1 = torch.as_tensor(yt[2], dtype=torch.float32)
    lx1 = torch.as_tensor(xt[2], dtype=torch.float32)
    ly0, lx0 = 1 - ly1, 1 - lx1                          # fl32(1 - l1), as the kernels compute it
    return [w.to(dtype) for w in (ly0.view(-1, 1), ly1.view(-1, 1), lx0.view(1, -1), lx1.view(1, -1))]


def transform_ref64(S, yt, xt, div255, norm, C):
    """S [C, n, H, W] source values (any dtype), the fp32 mean / std of the descriptor; returns (ref, absref)."""
    S = S.double()
    m = torch.tensor(MEAN[:C], dtype=torch.float32).double().view(C, 1, 1, 1)
    s = torch.tensor(STD[:C], dtype=torch.float32).double().view(C, 1, 1, 1)
    t = S / 255 if div255 else S
    v = (t - m) / s if norm else t
    a = (t.abs() + m.abs()) / s.abs() if norm else t.abs()
    ly0, ly1, lx0, lx1 = _weights(yt, xt, torch.float64)

    def blend(P):
        v00, v01, v10, v11 = _gather(P, yt, xt)
        return ly0 * (lx0 * v00 + lx1 * v01) + ly1 * (lx0 * v10 + lx1 * v11)
    return blend(v), blend(a)


def transform_emulate(S, yt, xt, div255, norm, C, mutation=None):
    """The kernels' fp32 order of operations: u / 255, (u - mean) / std per tap, then the nested lerp."""
    t = S.float()
    m = torch.tensor(MEAN[:C], dtype=torch.float32)
    if mutation == "mean_prev":
        m = torch.roll(m, 1)
    s = torch.tensor(STD[:C], dtype=torch.float32)
    if div255 and mutation != "no255":
        t = t / 255.0
    if norm:
        t = (t - m.view(C, 1, 1, 1)) / s.view(C, 1, 1, 1)
    if mutation == "tap_shift":
        W = S.shape[-1]
        xt = (np.minimum(xt[0] + 1, W - 1), np.minimum(xt[1] + 1, W - 1), xt[2])
    ly0, ly1, lx0, lx1 = _weights(yt, xt, torch.float32)
    if mutation == "swap_l":
        lx0, lx1 = lx1, lx0
    v00, v01, v10, v11 = _gather(t, yt, xt)
    return ly0 * (lx0 * v00 + lx1 * v01) + ly1 * (lx0 * v10 + lx1 * v11)


# =====================================================================================================================
# Batch transform (pv_clip_transform_batch)
# =====================================================================================================================
def batch_instance(sdt, ddt, C, arith):
    """The dispatch rule of pv_clip_transform_batch: one instance per (src, dst, C); a uint8 source with a float
    destination and any arithmetic (/255 or normalize) takes the shared-memory value table (LUT)."""
    lut = sdt == "u8" and ddt != "u8" and arith
    return "clip_transform_batch_kernel<%s,%s,%d,%s>" % (CT[sdt], CT[ddt], C, "true" if lut else "false")


def reachable_batch():
    out = set()
    for sdt, ddts in (("u8", ("f16", "f32", "u8")), ("f32", ("f16", "f32")), ("f16", ("f16", "f32"))):
        for ddt in ddts:
            for C in (1, 2, 3, 4):
                for arith in ((False,) if ddt == "u8" else (False, True)):
                    out.add(batch_instance(sdt, ddt, C, arith))
    return out


# name: (in_h, in_w, new_h, new_w, top, left, out_h, out_w, hflip)
GEOS = {
    "down1080x1920-7x455": (1080, 1920, 7, 455, 0, 0, 7, 455, 0),
    "up7x9-13x17-far-flip": (7, 9, 13, 17, 4, 0, 9, 17, 1),
    "h1-up1x40-9x80-w3-far": (1, 40, 9, 80, 0, 77, 9, 3, 0),
    "identity9x224": (9, 224, 9, 224, 0, 0, 9, 224, 0),
    "w1-up64x1-7x1030": (64, 1, 7, 1030, 0, 0, 7, 1030, 0),
    "down30x700-h1-w513-far-flip": (30, 700, 20, 513, 19, 0, 1, 513, 1),
    "down7x33-w2": (7, 33, 7, 2, 0, 0, 7, 2, 0),
    "down12x12-w1-flip": (12, 12, 9, 1, 0, 0, 9, 1, 1),
    "up1x1-5x5-flip": (1, 1, 5, 5, 2, 0, 1, 5, 1),
    "down360x640-9x224-far": (360, 640, 256, 455, 247, 231, 9, 224, 0),
    "train256x340-224": (256, 340, 224, 297, 0, 36, 224, 224, 0),
    # uint8 pass-through: no resize, crop (and flip) only
    "pt-crop-far": (9, 40, 9, 40, 2, 23, 7, 17, 0),
    "pt-w1030": (9, 1040, 9, 1040, 8, 10, 1, 1030, 0),
    "pt-w1-flip": (3, 5, 3, 5, 1, 4, 1, 1, 1),
    "pt-crop-far-flip": (9, 40, 9, 40, 0, 21, 9, 19, 1),
}
# modes: cthw (CTHW source, padded rows), thwc (interleaved source, sw = C + 1 with a padding channel), geom (per-clip
# short side, crop and flip), views (clip stride 0, per-view crop / flip and first-frame offset), slow (second output,
# n_t = 7 with alpha 2), mis (destination one element off its alignment: scalar stores), idx (repeated and reversed
# frame indices)
BATCH_ROWS = [
    # (src, dst, C, div255, normalize, geometry, mode)
    ("u8", "f16", 1, 1, 1, "down1080x1920-7x455", "cthw"),
    ("u8", "f16", 2, 1, 0, "up7x9-13x17-far-flip", "thwc"),
    ("u8", "f16", 3, 1, 1, "down360x640-9x224-far", "geom"),
    ("u8", "f16", 4, 0, 1, "w1-up64x1-7x1030", "mis"),
    ("u8", "f32", 1, 1, 1, "up1x1-5x5-flip", "idx"),
    ("u8", "f32", 2, 1, 1, "down30x700-h1-w513-far-flip", "slow"),
    ("u8", "f32", 3, 1, 1, "identity9x224", "views"),
    ("u8", "f32", 4, 1, 0, "down7x33-w2", "cthw"),
    ("u8", "f16", 1, 0, 0, "down12x12-w1-flip", "thwc"),
    ("u8", "f16", 2, 0, 0, "h1-up1x40-9x80-w3-far", "cthw"),
    ("u8", "f16", 3, 0, 0, "up7x9-13x17-far-flip", "slow"),
    ("u8", "f16", 4, 0, 0, "down30x700-h1-w513-far-flip", "views"),
    ("u8", "f32", 1, 0, 0, "down7x33-w2", "mis"),
    ("u8", "f32", 2, 0, 0, "identity9x224", "geom"),
    ("u8", "f32", 3, 0, 0, "w1-up64x1-7x1030", "idx"),
    ("u8", "f32", 4, 0, 0, "h1-up1x40-9x80-w3-far", "thwc"),
    ("u8", "u8", 1, 0, 0, "pt-crop-far", "cthw"),
    ("u8", "u8", 2, 0, 0, "pt-w1030", "thwc"),
    ("u8", "u8", 3, 0, 0, "pt-w1-flip", "slow"),
    ("u8", "u8", 4, 0, 0, "pt-crop-far-flip", "mis"),
    ("f32", "f16", 1, 1, 1, "h1-up1x40-9x80-w3-far", "views"),
    ("f32", "f16", 2, 0, 1, "down1080x1920-7x455", "cthw"),
    ("f32", "f16", 3, 0, 0, "down12x12-w1-flip", "geom"),
    ("f32", "f16", 4, 1, 1, "identity9x224", "slow"),
    ("f32", "f32", 1, 0, 1, "down30x700-h1-w513-far-flip", "thwc"),
    ("f32", "f32", 2, 1, 1, "w1-up64x1-7x1030", "views"),
    ("f32", "f32", 3, 0, 0, "up1x1-5x5-flip", "mis"),
    ("f32", "f32", 4, 1, 0, "up7x9-13x17-far-flip", "idx"),
    ("f16", "f16", 1, 0, 1, "identity9x224", "mis"),
    ("f16", "f16", 2, 1, 1, "down7x33-w2", "views"),
    ("f16", "f16", 3, 0, 1, "down360x640-9x224-far", "thwc"),
    ("f16", "f16", 4, 0, 0, "h1-up1x40-9x80-w3-far", "idx"),
    ("f16", "f32", 1, 1, 1, "down12x12-w1-flip", "slow"),
    ("f16", "f32", 2, 0, 1, "up1x1-5x5-flip", "geom"),
    ("f16", "f32", 3, 1, 0, "w1-up64x1-7x1030", "cthw"),
    ("f16", "f32", 4, 0, 0, "down30x700-h1-w513-far-flip", "mis"),
    # the train chain's shape: 256x340 uint8 clips, short side 224, 224 crop, per-clip flips, f16 out
    ("u8", "f16", 3, 1, 1, "train256x340-224", "geom"),
]


def _src_values(g, sdt, shape):
    if sdt == "u8":
        v = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
        flat = v.view(-1)
        flat[:2] = torch.tensor([0, 255], dtype=torch.uint8)      # both ends of the value table
        return v
    v = torch.rand(shape, generator=g) * 300 - 20                   # a decoded float clip, 0..255 plus overshoot
    return v.to(TDT[sdt])


def batch_case(row):
    """Everything a batch row needs on the host: source values, layout, per-clip geometry, frame indices."""
    sdt, ddt, C, div255, norm, geo, mode = row
    in_h, in_w, new_h, new_w, top, left, oh, ow, flip = GEOS[geo]
    g = _gen(row)
    B = {"views": 3, "geom": 3}.get(mode, 2)
    idx = {"idx": [3, 3, 1, 0], "slow": list(range(7))}.get(mode, [2, 0])
    T = {"views": 5, "slow": 8}.get(mode, 4)
    n_src = 1 if mode == "views" else B
    vals = _src_values(g, sdt, (n_src, C, T, in_h, in_w))
    geoms = []
    for b in range(B):
        if mode in ("geom", "views"):
            nh, nw = new_h + b, new_w + 2 * b
            tp = int(torch.randint(0, nh - oh + 1, (1,), generator=g)) if b else nh - oh   # clip 0: the far corner
            lf = int(torch.randint(0, nw - ow + 1, (1,), generator=g)) if b else nw - ow
            geoms.append((nh, nw, tp, lf, (flip + b) % 2, b if mode == "views" else 0))
        else:
            geoms.append((new_h, new_w, top, left, flip, 0))
    n_slow = len(idx) // 2 if mode == "slow" else 0
    slow_pos = None
    if mode == "slow":
        sel = torch.linspace(0, len(idx) - 1, n_slow).long().tolist()
        slow_pos = [sel.index(j) if j in sel else -1 for j in range(len(idx))]
    return dict(vals=vals, B=B, idx=idx, T=T, geoms=geoms, n_slow=n_slow, slow_pos=slow_pos, oh=oh, ow=ow,
                in_hw=(in_h, in_w))


def batch_expected(row, case, mutation=None, emulate=False):
    """[B, C, n_t, oh, ow] reference (ref, absref) or the fp32 emulation, and the pass-through values."""
    sdt, ddt, C, div255, norm, geo, mode = row
    in_h, in_w = case["in_hw"]
    oh, ow = case["oh"], case["ow"]
    refs, abss = [], []
    for b, (nh, nw, tp, lf, fl, t_off) in enumerate(case["geoms"]):
        frames = [i + t_off for i in case["idx"]]
        S = case["vals"][0 if mode == "views" else b][:, frames]
        if ddt == "u8":
            cols = np.arange(ow)[::-1] if fl else np.arange(ow)
            refs.append(S[:, :, tp:tp + oh][..., torch.as_tensor(lf + cols.copy())])
            continue
        yt = row_taps(in_h, nh, tp, oh)
        xt = col_taps(in_w, nw, lf, ow, fl, mutation)
        if emulate:
            refs.append(transform_emulate(S, yt, xt, div255, norm, C, mutation))
        else:
            r, a = transform_ref64(S, yt, xt, div255, norm, C)
            refs.append(r)
            abss.append(a)
    ref = torch.stack(refs)
    return ref, (torch.stack(abss) if abss else None)


def _src_buffer(vals, sdt, mode):
    """Physical source: CTHW with 3 padding columns per row, or THWC with one padding channel; padding holds BIG."""
    n, C, T, H, W = vals.shape
    if mode == "thwc":
        Cp = C + 1
        strides = (T * H * W * Cp, 1, H * W * Cp, W * Cp, Cp)
    else:
        Wp = W + 3
        strides = (C * T * H * Wp + 7, T * H * Wp, H * Wp, Wp, 1)
    size = 1 + sum((d - 1) * s for d, s in zip(vals.shape, strides))
    buf = torch.full((size + 16,), BIG[sdt], dtype=TDT[sdt])
    buf.as_strided(vals.shape, strides).copy_(vals)
    return buf, strides


def run_batch(row, case):
    sdt, ddt, C, div255, norm, geo, mode = row
    L = _L()
    B, n_t, oh, ow = case["B"], len(case["idx"]), case["oh"], case["ow"]
    in_h, in_w = case["in_hw"]
    buf, (s_clip, sc, st, sh, sw) = _src_buffer(case["vals"], sdt, mode)
    if mode == "views":
        s_clip = 0
    plane = oh * ow
    d_clip = C * n_t * plane + GAP
    off = 1 if mode == "mis" else 0
    dst = _sentinel(off + B * d_clip + TAIL, TDT[ddt]).to(_dev())
    nh, nw, tp, lf, fl, _ = case["geoms"][0]
    d = L.ClipBatchDesc()
    d.C, d.n_clips, d.n_t, d.n_slow = C, B, n_t, case["n_slow"]
    d.in_h, d.in_w, d.new_h, d.new_w, d.top, d.left, d.out_h, d.out_w, d.hflip = in_h, in_w, nh, nw, tp, lf, oh, ow, fl
    d.sc, d.st, d.sh, d.sw, d.s_clip = sc, st, sh, sw, s_clip
    d.d_clip = d_clip
    d.mean = (ctypes.c_float * 4)(*MEAN)
    d.stdv = (ctypes.c_float * 4)(*STD)
    d.div255, d.normalize, d.src_dtype, d.dst_dtype = div255, norm, _code(sdt), _code(ddt)
    src = buf.to(_dev())
    idx = torch.tensor(case["idx"], dtype=torch.int32, device=_dev())
    geom = None
    if mode in ("geom", "views"):
        geom = torch.tensor(case["geoms"], dtype=torch.int32, device=_dev())
    slow, spos = None, None
    if mode == "slow":
        d.d_slow_clip = C * case["n_slow"] * plane + GAP
        slow = _sentinel(B * d.d_slow_clip + TAIL, TDT[ddt]).to(_dev())
        spos = torch.tensor(case["slow_pos"], dtype=torch.int32, device=_dev())
    ptr = lambda t: None if t is None else t.data_ptr()
    launched = _launch("pv_clip_transform_batch", ctypes.byref(d), src.data_ptr(), idx.data_ptr(), ptr(spos),
                       ptr(geom), dst.data_ptr() + off * dst.element_size(), ptr(slow), _stream())
    return launched, dst.cpu(), (None if slow is None else slow.cpu()), d_clip, off


def _unpack(buf, B, clip_stride, C, n, oh, ow, off=0):
    """Output values [B, C, n, oh, ow] of a flat buffer with clip stride, and the mask of what they occupy."""
    idx = (off + torch.arange(B).view(B, 1) * clip_stride + torch.arange(C * n * oh * ow).view(1, -1)).reshape(-1)
    mask = torch.zeros(buf.numel(), dtype=torch.bool)
    mask[idx] = True
    return buf[idx].view(B, C, n, oh, ow), mask


@pytest.mark.gpu
@pytest.mark.parametrize("row", BATCH_ROWS, ids=[_rid(r) for r in BATCH_ROWS])
def test_batch_transform_row(row):
    sdt, ddt, C, div255, norm, geo, mode = row
    case = batch_case(row)
    launched, dst, slow, d_clip, off = run_batch(row, case)
    _expect(batch_instance(sdt, ddt, C, bool(div255 or norm)), launched)
    B, n_t, oh, ow = case["B"], len(case["idx"]), case["oh"], case["ow"]
    got, mask = _unpack(dst, B, d_clip, C, n_t, oh, ow, off)
    _assert_untouched(dst, mask, "dst")
    ref, absref = batch_expected(row, case)
    outs = [(got, ref, absref)]
    if slow is not None:
        sel = [j for j, p in enumerate(case["slow_pos"]) if p >= 0]
        sgot, smask = _unpack(slow, B, C * case["n_slow"] * oh * ow + GAP, C, case["n_slow"], oh, ow)
        _assert_untouched(slow, smask, "slow")
        outs.append((sgot, ref[:, :, sel], None if absref is None else absref[:, :, sel]))
    for g_, r_, a_ in outs:
        if ddt == "u8":
            assert torch.equal(g_, r_), "pass-through differs from index_select + crop"
            print("RATIO batch %s 0.0000 0.0000 %s bit-exact" % (_rid(row), sorted(launched)))
        else:
            _ratio("batch", row, _bound(g_, r_, a_, TR_EPS, _rnd(ddt), _rid(row)), launched)


# =====================================================================================================================
# Single-clip transform (pv_clip_transform_fwd, host tap tables)
# =====================================================================================================================
SINGLE_GEOS = {   # (in_h, in_w, new_h, new_w, top, left, out_h, out_w, flip)
    "down": (40, 60, 20, 31, 2, 3, 16, 25, 0),
    "up": (7, 9, 13, 17, 0, 0, 13, 17, 0),
    "flip": (30, 41, 24, 33, 3, 1, 18, 29, 1),
}
SINGLE_ROWS = [(s, d, C, div, geo, 0) for (s, d, C, div) in (("u8", "f16", 3, 1), ("u8", "f32", 1, 1),
                                                           ("f32", "f16", 2, 0), ("f32", "f32", 4, 1),
                                                           ("f16", "f16", 3, 0), ("f16", "f32", 2, 1))
               for geo in SINGLE_GEOS] + [("u8", "f16", 3, 1, "down", 1), ("f32", "f32", 2, 0, "flip", 1)]


def single_instance(sdt, ddt):
    return "clip_transform_kernel<%s,%s>" % (CT[sdt], CT[ddt])


@pytest.mark.gpu
@pytest.mark.parametrize("row", SINGLE_ROWS, ids=[_rid(r) for r in SINGLE_ROWS])
def test_single_clip_transform_row(row):
    sdt, ddt, C, div255, geo, mis = row
    in_h, in_w, nh, nw, top, left, oh, ow, flip = SINGLE_GEOS[geo]
    L = _L()
    g = _gen(row)
    T, idx = 4, [3, 1, 1]
    vals = _src_values(g, sdt, (1, C, T, in_h, in_w))
    buf, (_, sc, st, sh, sw) = _src_buffer(vals, sdt, "cthw")
    yt = row_taps(in_h, nh, top, oh)
    xt = col_taps(in_w, nw, left, ow, flip)
    dev_tabs = (*row_taps(in_h, nh, top, oh, FV.bilinear_table),
                *col_taps(in_w, nw, left, ow, flip, table=FV.bilinear_table))
    d = L.ClipTransformDesc()
    d.C, d.n_t, d.out_h, d.out_w = C, len(idx), oh, ow
    d.sc, d.st, d.sh, d.sw = sc, st, sh, sw
    d.mean = (ctypes.c_float * 4)(*MEAN)
    d.stdv = (ctypes.c_float * 4)(*STD)
    d.src_dtype, d.dst_dtype, d.div255 = _code(sdt), _code(ddt), div255
    dev = _dev()
    tabs = [torch.as_tensor(np.ascontiguousarray(a)).to(dev) for a in dev_tabs]    # the product's host tables
    n_out = C * len(idx) * oh * ow
    dst = _sentinel(mis + n_out + TAIL, TDT[ddt]).to(dev)
    src = buf.to(dev)
    it = torch.tensor(idx, dtype=torch.int32, device=dev)
    launched = _launch("pv_clip_transform_fwd", ctypes.byref(d), src.data_ptr(), it.data_ptr(),
                       *[t.data_ptr() for t in tabs], dst.data_ptr() + mis * dst.element_size(), _stream())
    _expect(single_instance(sdt, ddt), launched)
    out = dst.cpu()
    got, mask = _unpack(out, 1, n_out, C, len(idx), oh, ow, mis)
    _assert_untouched(out, mask, "dst")
    ref, absref = transform_ref64(vals[0][:, idx], yt, xt, div255, True, C)    # this entry point always normalises
    _ratio("single", row, _bound(got[0], ref, absref, TR_EPS, _rnd(ddt), _rid(row)), launched)


# =====================================================================================================================
# RandomResizedCrop mode (pv_clip_transform_rrc): window edges (its instance ledger is in test_gpu_augment.py)
# =====================================================================================================================
RRC_ROWS = [
    # (src, dst, window kind)
    ("u8", "f16", "corner"),          # window touching the bottom-right corner
    ("u8", "f32", "1x1"),             # a 1x1 window upscaled to the whole output
    ("f32", "f16", "flip"),           # flipped, odd output width
    ("f32", "f32", "corner"),
]


def _rrc_windows(kind, H, W, g):
    out = []
    for _ in range(4):                # (clip, frame) pairs: 2 clips x 2 kept frames
        if kind == "1x1":
            out.append([int(torch.randint(0, H, (1,), generator=g)), int(torch.randint(0, W, (1,), generator=g)), 1, 1,
                        0])
        else:
            h, w = int(torch.randint(1, H + 1, (1,), generator=g)), int(torch.randint(1, W + 1, (1,), generator=g))
            out.append([H - h, W - w, h, w, 1 if kind == "flip" else 0])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("row", RRC_ROWS, ids=[_rid(r) for r in RRC_ROWS])
def test_rrc_window_edge_row(row):
    sdt, ddt, kind = row
    L = _L()
    g = _gen(row)
    H, W, oh, ow, idx = 20, 30, 9, 11, [2, 0]
    vals = _src_values(g, sdt, (2, 3, 3, H, W))
    win = _rrc_windows(kind, H, W, g)
    buf, (s_clip, sc, st, sh, sw) = _src_buffer(vals, sdt, "cthw")
    d = L.ClipBatchDesc()
    d.C, d.n_clips, d.n_t, d.in_h, d.in_w, d.new_h, d.new_w, d.out_h, d.out_w = 3, 2, 2, H, W, oh, ow, oh, ow
    d.sc, d.st, d.sh, d.sw, d.s_clip = sc, st, sh, sw, s_clip
    d_clip = 3 * 2 * oh * ow + GAP
    d.d_clip = d_clip
    d.mean = (ctypes.c_float * 4)(*MEAN)
    d.stdv = (ctypes.c_float * 4)(*STD)
    d.div255, d.normalize, d.src_dtype, d.dst_dtype = 1, 1, _code(sdt), _code(ddt)
    dev = _dev()
    dst = _sentinel(2 * d_clip + TAIL, TDT[ddt]).to(dev)
    src, it = buf.to(dev), torch.tensor(idx, dtype=torch.int32, device=dev)
    boxes = torch.tensor(win, dtype=torch.int32, device=dev)
    launched = _launch("pv_clip_transform_rrc", ctypes.byref(d), src.data_ptr(), it.data_ptr(), boxes.data_ptr(),
                       dst.data_ptr(), _stream())
    _expect("clip_transform_rrc_kernel<%s,%s>" % (CT[sdt], CT[ddt]), launched)
    out = dst.cpu()
    got, mask = _unpack(out, 2, d_clip, 3, 2, oh, ow)
    _assert_untouched(out, mask, "dst")
    refs, abss = [], []
    for b in range(2):
        rr, aa = [], []
        for j in range(2):
            top, left, h, w, fl = win[b * 2 + j]
            y0, y1, ly = bilinear_table(h, oh)
            xt = col_taps(w, ow, 0, ow, fl)
            S = vals[b][:, [idx[j]]]
            r, a = transform_ref64(S, (y0 + top, y1 + top, ly), (xt[0] + left, xt[1] + left, xt[2]), 1, 1, 3)
            rr.append(r)
            aa.append(a)
        refs.append(torch.cat(rr, 1))
        abss.append(torch.cat(aa, 1))
    _ratio("rrc", row, _bound(got, torch.stack(refs), torch.stack(abss), TR_EPS, _rnd(ddt), _rid(row)), launched)


# =====================================================================================================================
# RoIAlign (pv_roi_align_fwd)
# =====================================================================================================================
f32 = np.float32


def contraction_discontinuity(box, H, W, ph_n, pw_n, scale, sr):
    """Where the contracted geometry differs from torchvision's at a discontinuity: 'grid' (another ceil count) or
    'cutoff' (a sample on the other side of -1 / H / W), else None."""
    a = TS.roi_geometry(box, H, W, ph_n, pw_n, scale, sr)
    b = TS.roi_geometry(box, H, W, ph_n, pw_n, scale, sr, contract=True)
    if a[2] != b[2]:
        return "grid"
    if [len(s) for s in a[0]] != [len(s) for s in b[0]]:
        return "cutoff"
    return None


# Boxes where nvcc's contraction of torchvision's geometry crosses a discontinuity and moves the result past its bound,
# found by a seeded search over fp32 box coordinates near the targets (roi_h = k * pooled_h with every sample inside
# the map for 'grid'; the last / first sample at H or -1 for 'cutoff') at non-power-of-two scales, keeping a box only
# when contraction_discontinuity finds a discontinuity and the contracted fp32 emulation fails the bound on the row's
# own f16 and f32 inputs (test_contraction_boxes_are_visible).  (scale, pooled_h, pooled_w, sampling_ratio, box)
CONTRACTION_BOXES = [
    (1 / 12, 3, 2, 0, (0, 1.0, 10.73066520690918, 40.0, 82.73066711425781)),
    (1 / 12, 2, 2, 2, (0, 1.0, -62.9288444519043, 40.0, 18.55730628967285)),
    (1 / 12, 2, 2, 2, (0, 1.0, -78.20991516113281, 40.0, 27.725948333740234)),
    (0.3, 3, 2, 0, (0, 1.0, 4.633927822113037, 40.0, 24.633928298950195)),
    (0.3, 2, 2, 2, (0, 1.0, 27.937053680419922, 40.0, 56.96137237548828)),
    (0.3, 2, 2, 2, (0, 1.0, 22.472389221191406, 40.0, 57.74203872680664)),
    (1 / 7, 3, 2, 0, (0, 1.0, 11.989120483398438, 40.0, 53.98912048339844)),
    (1 / 7, 2, 2, 2, (0, 1.0, -57.94064712524414, 40.0, 23.56438636779785)),
    (1 / 7, 2, 2, 2, (0, 1.0, 62.26563262939453, 40.0, 119.10490417480469)),
    # the second box transposed: the sample crosses -1 in x instead of y
    (1 / 12, 2, 2, 2, (0, -62.9288444519043, 1.0, 18.55730628967285, 40.0)),
]
CONTRACTION_HW = (16, 16)


def _roi_boxes(kind, row, g):
    dt, N, H, W, C, ph_n, pw_n, scale, sr = row[:9]
    ih, iw = H / scale, W / scale                    # the map in input-image pixels

    def u(lo, hi):
        return float(torch.empty(1).uniform_(lo, hi, generator=g))
    if kind in ("inside", "inside+huge"):
        out = []
        for k in range(4):
            x1, y1 = u(0, iw * 0.6), u(0, ih * 0.6)
            out.append((k % N, x1, y1, u(x1, iw - 1e-3), u(y1, ih - 1e-3)))
        if kind == "inside+huge":                    # 9x the map each way: an adaptive grid of 9 x 9 per bin
            out.append((N - 1, -4 * iw, -4 * ih, 5 * iw, 5 * ih))
        return out
    if kind == "cross":                              # one box over each side, one over everything
        return [(0, u(-iw / 2, -1), u(0, ih / 2), u(1, iw / 2), u(ih / 2, ih)),
                (N - 1, u(0, iw / 2), u(-ih / 2, -1), u(iw / 2, iw), u(1, ih / 2)),
                (0, u(iw / 2, iw), u(0, ih / 2), u(iw + 1, 1.5 * iw), u(ih / 2, ih)),
                (N - 1, u(0, iw / 2), u(ih / 2, ih), u(iw / 2, iw), u(ih + 1, 1.5 * ih)),
                (0, -iw / 4, -ih / 4, 1.25 * iw, 1.25 * ih)]
    if kind == "outside":
        return [(0, -3 * iw, 0.0, -1.5 * iw, ih), (N - 1, 0.0, 2.5 * ih, iw, 4 * ih), (0, 0.5, 0.5, iw / 2, ih / 2)]
    if kind == "exact":
        # scale 1/2, sampling_ratio 1, 1x1 bins: the sample sits at ((y1 + y2) / 4), exactly -1, 0, H-1, H (x alike)
        t = [-1.0, 0.0, H - 1.0, float(H)]
        s = [-1.0, 0.0, W - 1.0, float(W)]
        return [(k % N, 2 * s[k % 4] - 1, 2 * t[(k + 1) % 4] - 1, 2 * s[k % 4] + 1, 2 * t[(k + 1) % 4] + 1)
                for k in range(8)] + [(0, 2 * s[0] - 1.5, 2 * t[0] - 1.5, 2 * s[0] + 0.5, 2 * t[0] + 0.5)]
    if kind == "degenerate":                         # x2 < x1 and y2 < y1: roi size clamps to 1
        return [(0, u(iw / 2, iw), u(ih / 2, ih), u(0, iw / 2), u(0, ih / 2)), (N - 1, 5.0, 5.0, 5.0, 5.0)]
    if kind == "badn":                               # batch indices -1 and N give zeros
        return [(-1, 0.0, 0.0, iw / 2, ih / 2), (N, 0.0, 0.0, iw / 2, ih / 2), (0, 0.0, 0.0, iw / 2, ih / 2)]
    if kind == "contract":
        return [b for (sc, p_h, p_w, s_r, b) in CONTRACTION_BOXES
                if (sc, p_h, p_w, s_r) == (scale, ph_n, pw_n, sr)]
    raise KeyError(kind)


ROI_ROWS = [
    # (dtype, N, H, W, C, pooled_h, pooled_w, scale, sampling_ratio, boxes, x row pad, y row pad)
    ("f16", 2, 9, 11, 24, 7, 7, 1 / 16, 0, "inside", 0, 0),
    ("f32", 2, 9, 11, 24, 7, 7, 1 / 16, 2, "inside", 8, 8),
    ("f16", 2, 14, 12, 8, 1, 1, 1 / 16, 0, "cross", 0, 8),
    ("f32", 1, 14, 12, 16, 3, 5, 0.25, 1, "cross", 16, 0),
    ("f16", 2, 14, 14, 2048, 14, 14, 1 / 16, 0, "inside+huge", 0, 0),   # grids of 1 and of 9 x 9 per bin
    ("f32", 1, 6, 7, 2056, 3, 5, 1 / 16, 4, "cross", 8, 8),            # channel loop past 256 threads x 8
    ("f16", 1, 6, 7, 2056, 7, 7, 0.25, 2, "inside", 0, 8),
    ("f16", 2, 8, 9, 24, 3, 5, 0.5, 4, "outside", 8, 0),
    ("f16", 2, 9, 9, 24, 1, 1, 0.5, 1, "exact", 0, 8),
    ("f32", 2, 7, 5, 8, 1, 1, 0.5, 1, "exact", 8, 0),
    ("f16", 2, 9, 11, 24, 7, 7, 1 / 16, 0, "degenerate", 0, 0),
    ("f32", 2, 9, 11, 24, 3, 5, 1 / 16, 2, "badn", 0, 8),
    ("f16", 1, 1, 11, 24, 3, 5, 0.25, 0, "cross", 8, 0),                # H = 1
    ("f32", 1, 9, 1, 24, 7, 7, 0.25, 2, "cross", 0, 8),                 # W = 1
] + [(dt, 1, 16, 16, 24, p_h, p_w, sc, s_r, "contract", 0, 8)
     for dt in ("f16", "f32") for (sc, p_h, p_w, s_r) in sorted({b[:4] for b in CONTRACTION_BOXES})]


def roi_inputs(row):
    dt, N, H, W, C = row[:5]
    g = _gen(row)
    x = torch.randn(N, H, W, C, generator=g)
    x = x.half().float() if dt == "f16" else x
    return x, _roi_boxes(row[9], row, g)


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROI_ROWS, ids=[_rid(r) for r in ROI_ROWS])
def test_roi_align_row(row):
    dt, N, H, W, C, ph_n, pw_n, scale, sr, kind, xpad, ypad = row
    x, rois = roi_inputs(row)
    K = len(rois)
    xrs, yrs = C + xpad, C + ypad
    dev = _dev()
    xb = torch.full((N * H * W * xrs + TAIL,), BIG["f16"], dtype=TDT[dt])
    xb[:N * H * W * xrs].view(N * H * W, xrs)[:, :C] = x.reshape(-1, C).to(TDT[dt])
    y = _sentinel(K * ph_n * pw_n * yrs + TAIL, TDT[dt]).to(dev)
    r = torch.tensor(rois, dtype=torch.float32, device=dev)
    xd = xb.to(dev)
    launched = _launch("pv_roi_align_fwd", xd.data_ptr(), _code(dt), xrs, N, H, W, C, r.data_ptr(), K, ph_n, pw_n,
                       scale, sr, y.data_ptr(), yrs, _stream())
    _expect("roi_align_kernel<%s>" % CT[dt], launched)
    out = y.cpu()
    mask = torch.zeros(out.numel(), dtype=torch.bool)
    mask[:K * ph_n * pw_n * yrs].view(-1, yrs)[:, :C] = True
    _assert_untouched(out, mask, "y")
    got = out[:K * ph_n * pw_n * yrs].view(K, ph_n, pw_n, yrs)[..., :C]
    ref, absref = TS.roi_ref64(x, rois, row[5:9])
    if kind == "badn":
        assert bool((got[:2] == 0).all())
    _ratio("roi", row, _bound(got, ref, absref, TS.roi_acc_eps(rois, row[5:9], H, W), _rnd(dt), _rid(row)), launched)


# =====================================================================================================================
# View reduce (pv_view_reduce): bit-exact against the reference's per-video loop
# =====================================================================================================================
VIEW_ROWS = [
    # (n_videos, n_views, K, mode, values)
    (4, 1, 400, "sum", "randn"), (4, 1, 400, "max", "neg"), (3, 3, 700, "mean", "randn"),
    (3, 3, 1, "max", "randn"), (2, 30, 400, "sum", "randn"), (2, 30, 400, "mean", "randn"),
    (2, 30, 700, "max", "randn"), (5, 3, 400, "max", "neg"), (2, 30, 1, "max", "neg"),
    (3, 3, 400, "max", "nan"), (3, 3, 400, "sum", "nan"), (2, 30, 700, "mean", "nan"),
]


def view_inputs(row):
    nv, nw, K, mode, kind = row
    g = _gen(row)
    p = torch.randn(nv * nw, K, generator=g) * 4
    if kind == "neg":
        p = -p.abs() - 0.5
        p[:, :K // 2] = p[:, :K // 2] + 1.0            # half the classes mixed, the rest all negative
    if kind == "nan":
        p[nw - 1, ::3] = float("nan")                  # one view of the first video
        p[-1, 1] = float("nan")
    return p


def view_reduce_ref(p, n_views, mode):
    """video_classification.py:290-311 and :279-282 in torch fp32: per video, zeros, then += or torch.max per view in
    order; "mean" divides by the clip count."""
    nv = p.shape[0] // n_views
    out = []
    for v in range(nv):
        acc = torch.zeros(p.shape[1], dtype=torch.float32)
        for i in range(n_views):
            acc = torch.max(acc, p[v * n_views + i]) if mode == "max" else acc + p[v * n_views + i]
        out.append(acc / n_views if mode == "mean" else acc)
    return torch.stack(out)


def _assert_same(got, want, what):
    gn, wn = torch.isnan(got), torch.isnan(want)
    assert torch.equal(gn, wn), "%s: NaN positions differ (%d vs %d)" % (what, int(gn.sum()), int(wn.sum()))
    gb, wb = _bits(got)[~gn], _bits(want)[~wn]
    assert torch.equal(gb, wb), "%s: %d values differ" % (what, int((gb != wb).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("row", VIEW_ROWS, ids=[_rid(r) for r in VIEW_ROWS])
def test_view_reduce_row(row):
    nv, nw, K, mode, kind = row
    p = view_inputs(row)
    dev = _dev()
    out = _sentinel(nv * K + TAIL, torch.float32).to(dev)
    pd = p.to(dev)
    launched = _launch("pv_view_reduce", pd.data_ptr(), out.data_ptr(), nv, nw, K, {"sum": 0, "mean": 1, "max": 2}[mode],
                       _stream())
    _expect("view_reduce_kernel", launched)
    o = out.cpu()
    mask = torch.zeros(o.numel(), dtype=torch.bool)
    mask[:nv * K] = True
    _assert_untouched(o, mask, "out")
    _assert_same(o[:nv * K].view(nv, K), view_reduce_ref(p, nw, mode), _rid(row))
    print("RATIO view %s 0.0000 0.0000 %s bit-exact" % (_rid(row), sorted(launched)))


def test_view_reduce_reference_is_the_zero_seeded_max():
    p = torch.tensor([[-3.0, 1.0, float("nan")], [-2.0, -5.0, 0.5]])
    assert view_reduce_ref(p, 2, "max").tolist()[0][:2] == [0.0, 1.0]
    assert torch.isnan(view_reduce_ref(p, 2, "max")[0, 2])
    assert view_reduce_ref(p, 2, "mean").tolist()[0][:2] == [-2.5, -2.0]


# =====================================================================================================================
# CPU: comparator, geometry, routing and the instance ledger
# =====================================================================================================================
CPU_BATCH_ROWS = [r for r in BATCH_ROWS if r[1] != "u8" and GEOS[r[5]][0] * GEOS[r[5]][1] <= 360 * 640]


def _check_batch(row, mutation=None):
    case = batch_case(row)
    ref, absref = batch_expected(row, case)
    emu, _ = batch_expected(row, case, mutation=mutation, emulate=True)
    got = _store(emu, row[1], mutation)
    return _bound(got, ref, absref, TR_EPS, _rnd(row[1]), "%s %s" % (_rid(row), mutation))


def _check_roi(row, mutation=None):
    x, rois = roi_inputs(row)
    ref, absref = TS.roi_ref64(x, rois, row[5:9])
    emu, _ = TS.roi_ref64(x, rois, row[5:9], mutation=mutation, emulate=True)
    got = _store(emu, row[0], mutation)
    return _bound(got, ref, absref, TS.roi_acc_eps(rois, row[5:9], row[2], row[3]), _rnd(row[0]),
                  "%s %s" % (_rid(row), mutation))


@pytest.mark.parametrize("row", CPU_BATCH_ROWS, ids=[_rid(r) for r in CPU_BATCH_ROWS])
def test_transform_emulation_passes_its_bound(row):
    print("RATIO emulation-batch %s %.4f %.4f" % ((_rid(row),) + _check_batch(row)))


CPU_ROI_ROWS = [r for r in ROI_ROWS if r[4] <= 24]


@pytest.mark.parametrize("row", CPU_ROI_ROWS, ids=[_rid(r) for r in CPU_ROI_ROWS])
def test_roi_emulation_passes_its_bound(row):
    print("RATIO emulation-roi %s %.4f %.4f" % ((_rid(row),) + _check_roi(row)))


def _brow(pred):
    return next(r for r in CPU_BATCH_ROWS if pred(r))


def _rrow(pred):
    return next(r for r in CPU_ROI_ROWS if pred(r))


MUTATIONS = {
    "taps_shifted_one_pixel": (_check_batch, _brow(lambda r: r[5] == "down360x640-9x224-far"), "tap_shift"),
    "l0_l1_swapped": (_check_batch, _brow(lambda r: r[5] == "up7x9-13x17-far-flip"), "swap_l"),
    "flip_off_by_one": (_check_batch, _brow(lambda r: GEOS[r[5]][8] and GEOS[r[5]][7] > 3), "flip_off"),
    "mean_of_previous_channel": (_check_batch, _brow(lambda r: r[4] and r[2] > 1), "mean_prev"),
    "div255_dropped": (_check_batch, _brow(lambda r: r[3]), "no255"),
    "f16_store_truncated": (_check_batch, _brow(lambda r: r[1] == "f16" and r[5] == "down360x640-9x224-far"),
                            "trunc16"),
    "roi_sample_at_iy": (_check_roi, _rrow(lambda r: r[9] == "inside"), "iy"),
    "roi_grid_floor": (_check_roi, _rrow(lambda r: r[9] == "inside" and r[8] == 0), "floor"),
    "roi_cutoff_y_ge_H": (_check_roi, _rrow(lambda r: r[9] == "exact"), "ge_H"),
    "roi_f16_store_truncated": (_check_roi, _rrow(lambda r: r[0] == "f16" and r[9] == "inside"), "trunc16"),
}


@pytest.mark.parametrize("name", sorted(MUTATIONS))
def test_comparator_rejects_input_kernel_bugs(name):
    fn, row, mutation = MUTATIONS[name]
    with pytest.raises(AssertionError):
        fn(row, mutation)


def test_host_tables_equal_the_pinned_table():
    """The single-clip entry point reads functional.bilinear_table; at every size the rows use it equals the table
    pinned to ATen (including one output pixel, where a scalar once came back instead of an array)."""
    sizes = {(g[0], g[2]) for g in SINGLE_GEOS.values()} | {(g[1], g[3]) for g in SINGLE_GEOS.values()}
    sizes |= {(g[0], g[2]) for g in GEOS.values()} | {(g[1], g[3]) for g in GEOS.values()} | {(12, 1), (1, 1)}
    for i, o in sorted(sizes):
        for a, b in zip(FV.bilinear_table(i, o), bilinear_table(i, o)):
            assert a.shape == (o,) and a.dtype == b.dtype and np.array_equal(a, b), (i, o)


def test_column_taps_follow_the_pinned_table():
    """col_taps / row_taps index oracle.transforms_ref.bilinear_table (pinned to ATen in test_oracle_pinning.py);
    check the flip and crop indexing against a direct restatement of the batch kernel's tap arithmetic."""
    for in_w, new_w, left, out_w, flip in ((9, 17, 0, 17, 1), (1920, 455, 3, 451, 0), (1, 5, 0, 5, 1), (40, 80, 77, 3, 1),
                                           (33, 2, 0, 2, 0), (12, 1, 0, 1, 1)):
        i0, i1, l1 = col_taps(in_w, new_w, left, out_w, flip)
        scale = f32(in_w) / f32(new_w)
        for xo in range(out_w):
            dst = left + (out_w - 1 - xo if flip else xo)
            src = max(f32(float(scale) * (dst + 0.5) - 0.5), f32(0))
            j0 = min(int(np.floor(src)), in_w - 1)
            lam = min(max(src - f32(j0), f32(0)), f32(1))
            assert (i0[xo], l1[xo]) == (j0, lam), (in_w, new_w, xo)
            assert l1[xo] == 0 or i1[xo] == j0 + (j0 < in_w - 1)


def test_roi_geometry_is_the_oracle():
    """roi_ref64's fp32 emulation, which shares roi_geometry with the float64 reference, equals
    oracle.interp.roi_align_ref bit for bit."""
    from oracle.interp import roi_align_ref
    for row in (ROI_ROWS[0], ROI_ROWS[3], ROI_ROWS[8], ROI_ROWS[-1]):
        x, rois = roi_inputs(row)
        emu, _ = TS.roi_ref64(x, rois, row[5:9], emulate=True)
        want = roi_align_ref(x.permute(0, 3, 1, 2), torch.tensor(rois, dtype=torch.float32), (row[5], row[6]), row[7],
                             row[8]).permute(0, 2, 3, 1)
        assert torch.equal(emu, want), _rid(row)


def test_contraction_boxes_cross_a_discontinuity():
    H, W = CONTRACTION_HW
    kinds = set()
    for scale, ph_n, pw_n, sr, box in CONTRACTION_BOXES:
        k = contraction_discontinuity(box, H, W, ph_n, pw_n, scale, sr)
        assert k is not None, box
        kinds.add(k)
    assert kinds == {"grid", "cutoff"}
    # and the geometry the detection models use (scale 1/16) is immune to the first contraction
    assert all(contraction_discontinuity(b, 9, 11, 7, 7, 1 / 16, 0) != "grid" for b in _roi_boxes("inside", ROI_ROWS[0],
                                                                                                  _gen(ROI_ROWS[0])))


def _contract_row(dt, key):
    return next(r for r in ROI_ROWS if r[9] == "contract" and r[0] == dt and (r[7], r[5], r[6], r[8]) == key)


@pytest.mark.parametrize("i", range(len(CONTRACTION_BOXES)))
def test_contraction_boxes_are_visible(i):
    """Each committed box, on its GPU rows' own inputs: the uncontracted fp32 emulation passes the bound and the
    contracted one fails it, so a kernel whose geometry nvcc contracts fails those rows."""
    scale, ph_n, pw_n, sr, box = CONTRACTION_BOXES[i]
    for dt in ("f16", "f32"):
        row = _contract_row(dt, (scale, ph_n, pw_n, sr))
        x = roi_inputs(row)[0]
        ref, absref = TS.roi_ref64(x, [box], row[5:9])
        eps = TS.roi_acc_eps([box], row[5:9], row[2], row[3])
        good, _ = TS.roi_ref64(x, [box], row[5:9], emulate=True)
        _bound(_store(good, dt), ref, absref, eps, _rnd(dt), "uncontracted")
        bad, _ = TS.roi_ref64(x, [box], row[5:9], emulate=True, contract=True)
        with pytest.raises(AssertionError):
            _bound(_store(bad, dt), ref, absref, eps, _rnd(dt), "contracted")


def test_rows_have_grids_of_one_and_of_at_least_eight():
    grids = {TS.roi_geometry(b, r[2], r[3], r[5], r[6], r[7], r[8])[2] for r in ROI_ROWS if r[8] == 0
             for b in roi_inputs(r)[1]}
    assert (1, 1) in grids and any(min(g) >= 8 for g in grids)
    big = ROI_ROWS[4]
    assert big[4] == 2048 and (9, 9) in {TS.roi_geometry(b, big[2], big[3], big[5], big[6], big[7], 0)[2]
                                          for b in roi_inputs(big)[1]}


def test_contraction_search_finds_boxes():
    """A seeded search near roi_h = k * pooled_h at scale 0.3 finds a box whose ceil grid count the contraction
    changes (how the 'grid' boxes above were found)."""
    rng = np.random.default_rng(1)
    s = f32(0.3)
    for _ in range(200):
        y1 = f32(rng.uniform(0, 100))
        y2 = f32(float(y1) + 2 * 3 / float(s))
        for _ in range(20):
            if contraction_discontinuity((0, 1.0, float(y1), 40.0, float(y2)), 16, 16, 3, 2, 0.3, 0) == "grid":
                return
            y2 = np.nextafter(y2, f32(np.inf))
    raise AssertionError("no contraction-sensitive box found")


def test_rows_reach_every_reachable_batch_instance():
    want = reachable_batch()
    assert len(want) == 36
    rows = {batch_instance(r[0], r[1], r[2], bool(r[3] or r[4])) for r in BATCH_ROWS}
    assert rows == want, sorted(want - rows)
    assert {single_instance(r[0], r[1]) for r in SINGLE_ROWS} == {single_instance(s, d) for s in CT for d in
                                                                   ("f16", "f32")}
    assert {r[0] for r in ROI_ROWS} == {"f16", "f32"}
    edges = {GEOS[r[5]][7] for r in BATCH_ROWS} | {GEOS[r[5]][6] for r in BATCH_ROWS}
    assert {1, 2, 3, 17, 224, 513, 1030, 7, 9} <= edges
    assert {r[6] for r in BATCH_ROWS} == {"cthw", "thwc", "geom", "views", "slow", "mis", "idx"}


def _compiled_instances():
    """Kernel instances the built library contains, read from its host stubs with binutils `nm` (as test_abi.py
    reads the exported entry points).  Loading first builds the library when it is missing or older than its
    sources, so the ledger checks what the current sources compile to."""
    from pytorchvideo_b200 import _lib
    _lib.load()
    nm = shutil.which("nm")
    assert nm, "the instance ledger reads the library's symbols with binutils `nm`, which is not installed"
    res = subprocess.run([nm, "-D", "-C", "--defined-only", _lib.lib_path()], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    out = res.stdout
    names = set()
    for m in re.finditer(r"pv::((?:clip_transform_batch_kernel|clip_transform_kernel|roi_align_kernel)<[^>]*>)", out):
        n = m.group(1).replace("unsigned char", "uint8_t").replace(" ", "")
        if n.startswith("clip_transform_kernel<"):
            n = n.rsplit(",", 1)[0] + ">"           # the pixels-per-thread argument is fixed at 2
        names.add(n)
    return names


def test_ledger_compiled_instances_are_the_rows_instances():
    names = _compiled_instances()
    batch = {n for n in names if n.startswith("clip_transform_batch_kernel<")}
    single = {n for n in names if n.startswith("clip_transform_kernel<")}
    roi = {n for n in names if n.startswith("roi_align_kernel<")}
    assert (len(batch), len(single), len(roi)) == (36, 6, 2), sorted(names)
    assert not any(n.startswith("clip_transform_batch_kernel<uint8_t,uint8_t,") and n.endswith(",true>")
                   for n in batch)
    expected = ({batch_instance(r[0], r[1], r[2], bool(r[3] or r[4])) for r in BATCH_ROWS} |
                {single_instance(r[0], r[1]) for r in SINGLE_ROWS} | {"roi_align_kernel<%s>" % CT[r[0]] for r in ROI_ROWS})
    assert names == expected, (sorted(names - expected), sorted(expected - names))


def test_ledger_launch_sites_name_their_template_arguments():
    tr = open(os.path.join(CSRC, "pv_transform.cu")).read()
    roi = open(os.path.join(CSRC, "pv_roi.cu")).read()
    assert 'PV_LAUNCH_OK("clip_transform_batch_kernel<" #ST "," #OT "," #NC "," #LUT ">")' in tr
    assert 'PV_LAUNCH_OK("clip_transform_kernel<" #ST "," #OT ">")' in tr
    assert 'PV_LAUNCH_OK("view_reduce_kernel")' in tr
    assert 'PV_LAUNCH_OK("roi_align_kernel<__half>")' in roi and 'PV_LAUNCH_OK("roi_align_kernel<float>")' in roi
    for src in (tr, roi):                       # no launch site records a bare family name
        for name in re.findall(r'PV_LAUNCH_OK\("([^"]+)"\)', src):
            assert name == "view_reduce_kernel" or "<" in name, name
