"""CUDA-core kernels of csrc/pv_simt.cu against float64, one row per launch site and edge.

Every GPU test calls the C ABI directly (ctypes, as engine/plan.py does), so a row sets the row strides, batch
strides, pointer offsets and in-place aliasing itself.  It asserts from the library's launch counts which kernel ran,
fills every output element outside the written slice with a sentinel bit pattern and checks that it survived, and
compares with float64:
  - bit-exact (bit patterns equal to a torch emulation) where the operation is exact or rounds once from fp32: the
    layout conversions (f32 -> f16 is round-to-nearest-even, with ties, subnormals and overflow to inf), copy_rows,
    max pooling, add_pos_cls and the fp32 sum of add_layernorm;
  - bounded (testing.assert_close_to_f64) everywhere else, with a bound derived per family next to its reference.
CPU tests check that an fp32 emulation of each bounded kernel, in the kernel's order of operations, passes its
bound while known bugs fail it, that the launch-name ledger covers every launch site and entry point of pv_simt.cu,
and that the rows reach every route of the dispatchers.

Measured on an NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit), per bounded family: the largest err / tol, and in
brackets the largest share of the fp32 term (accumulation plus extra64 together) a result used beyond its own
storage rounding.  A correctly rounded f16 result may use nearly all of the rounding term, hence ratios near 1 with
small shares:
  average pooling 0.948 (0.002), channel_sum 0.003 (0.003), se_gate 0.009 (0.003), scale_act 0.998 (0.468),
  head_reduce 0.081 (0.068), LayerNorm (both kernels) 0.978 (0.024), add_layernorm 0.979 (0.019),
  temporal_tap_sum 0.947 (0.022).
The layout conversions, copy_rows, max pooling, add_pos_cls and the add_layernorm sum matched bit for bit.

Not verified: the 64-bit index branch of scale_act_kernel (N * npos * C / 8 >= 2^31, i.e. more than 32 GB of f16
input).
"""
import ctypes
import math
import os
import re
import zlib

import pytest
import torch
import torch.nn.functional as F

from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.testing import LIP, SUM_EPS, act64, act_err64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorchvideo_b200", "csrc")
TESTS = os.path.dirname(os.path.abspath(__file__))

U = TS.F32_EPS                  # fp32 unit roundoff
TAIL = 64                       # sentinel elements after every output buffer
SENT = {torch.float16: 0x5A5A, torch.float32: 0x5A5A5A5A, torch.int64: 0x5A5A5A5A5A5A5A5A}
TDT = {"f16": torch.float16, "f32": torch.float32}
BIG = 60000.0                   # pad-channel filler (f16-representable): a kernel reading it moves the result far


def _dev():
    return torch.device("cuda:0")


def _L():
    from pytorchvideo_b200 import _lib as L
    return L


def _code(dt):
    return _L().PV_F16 if dt == "f16" else _L().PV_F32


def _rnd(dt):
    return TS.F16_EPS if dt == "f16" else TS.F32_EPS


def _gen(row):
    return torch.Generator().manual_seed(zlib.crc32(repr(row).encode()))


def _rid(row):
    return "-".join(str(v) for v in row).replace(" ", "")


def _ids(rows):
    return [_rid(r) for r in rows]


def _int_type(dtype):
    return {torch.float16: torch.int16, torch.float32: torch.int32, torch.int64: torch.int64}[dtype]


def _sentinel_cpu(n, dtype):
    return torch.full((n,), SENT[dtype], dtype=_int_type(dtype)).view(dtype)


def _bits(t):
    return t.detach().cpu().contiguous().view(_int_type(t.dtype))


def _assert_bits(got, want, what):
    """Bit patterns equal (so -0.0 != +0.0 and the sentinel counts too)."""
    gb, wb = _bits(got), _bits(want)
    diff = (gb != wb).reshape(-1)
    if bool(diff.any()):
        i = int(diff.nonzero()[0])
        raise AssertionError("%s: %d elements differ, first at flat %d: got %r, want %r" % (
            what, int(diff.sum()), i, got.reshape(-1)[i].item(), want.reshape(-1)[i].item()))


def _assert_untouched(buf, written, what):
    """Every element of the flat buffer outside the boolean mask still holds the sentinel."""
    b = _bits(buf).reshape(-1)
    bad = (b != SENT[buf.dtype]) & ~written.reshape(-1)
    assert not bool(bad.any()), "%s: %d elements outside the output slice changed (first at flat %d)" % (
        what, int(bad.sum()), int(bad.nonzero()[0]))


def _launch(entry, *args):
    """Call a C entry point, wait for it, return {kernel: launches} of what it ran."""
    L = _L()
    before = TS.kernel_counts()
    L.check(getattr(L.load(), entry)(*args), entry)
    torch.cuda.synchronize()
    return TS.kernel_count_diff(before, TS.kernel_counts())


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _expect(name, launched):
    assert set(launched) == {name}, "expected %s, launched %s" % (name, launched)


def _assert_bound(got, ref64, absref64, k_len, acc_eps, what, extra64=None, rnd_eps=TS.F16_EPS):
    """TS.assert_close_to_f64, returning (largest err / tol, largest share of the fp32 term used): the error beyond
    the storage rounding over the fp32 term, accumulation and extra64 together (the margin of the derived bound)."""
    ratio = TS.assert_close_to_f64(got, ref64, absref64, k_len, acc_eps=acc_eps, what=what, extra64=extra64,
                                   rnd_eps=rnd_eps)
    got64, ref64 = got.detach().double().cpu(), ref64.double().cpu()
    term = acc_eps * (1.0 + k_len / 64.0) * absref64.double().cpu()
    if extra64 is not None:
        term = term + extra64.double().cpu()
    excess = ((got64 - ref64).abs() - rnd_eps * ref64.abs() - 2.0 ** -24 * (rnd_eps / TS.F16_EPS)).clamp_min(0)
    return ratio[0], float((excess / term.clamp_min(1e-300)).max())


def _ratio(family, row, ratio, launched):
    print("RATIO %s %s %.4f %.4f %s" % (family, _rid(row), ratio[0], ratio[1], sorted(launched)))


def _exact(family, row, launched):
    print("RATIO %s %s 0.0000 0.0000 %s bit-exact" % (family, _rid(row), sorted(launched)))


def _rows_buffer(vals, stride, dtype, fill=None):
    """[R, C] values -> flat [R * stride + TAIL] buffer of dtype; pad channels / tail hold `fill` or the sentinel."""
    R, C = vals.shape
    buf = _sentinel_cpu(R * stride + TAIL, dtype) if fill is None else torch.full((R * stride + TAIL,), fill, dtype=dtype)
    buf[:R * stride].view(R, stride)[:, :C] = vals.to(dtype)
    return buf


def _written(R, stride, C, off=0):
    m = torch.zeros(R * stride + TAIL + off, dtype=torch.bool)
    m[off:off + R * stride].view(R, stride)[:, :C] = True
    return m


# ---- activations: float64 reference, Lipschitz constant, error of the kernel's own fp32 evaluation ------------------
ACTS = ("none", "relu", "swish", "gelu", "sigmoid", "hswish")


def _act_code(act):
    L = _L()
    return {"none": L.ACT_NONE, "relu": L.ACT_RELU, "swish": L.ACT_SWISH, "gelu": L.ACT_GELU,
            "sigmoid": L.ACT_SIGMOID, "hswish": L.ACT_HSWISH}[act]


def act32(v, act):
    """apply_act in fp32 torch (the CPU emulation)."""
    if act == "none":
        return v
    if act == "relu":
        return v.clamp_min(0)
    if act == "swish":
        return v / (1 + torch.exp(-v))
    if act == "gelu":
        return 0.5 * v * (1 + torch.erf(v * 0.70710678118654752440))
    if act == "sigmoid":
        return 1 / (1 + torch.exp(-v))
    return v * (v + 3).clamp(0, 6) / 6


def _fma32(a, b, c):
    """fmaf in fp32: the exact product-sum rounded once (double rounding through float64 is within the bounds)."""
    return (a.double() * b.double() + c.double()).float()


def _f16(t):
    return t.half().float()


# =====================================================================================================================
# Layout conversions (bit-exact)
# =====================================================================================================================
# f32 values whose f16 rounding is an edge: ties to even (1 + 2^-11, 2049, 3 * 2^-25), subnormals, the largest
# finite f16 and values past it (65520 rounds to inf), signed zero
F32_SPECIALS = [1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, -(1 + 2.0 ** -11), 2049.0, 2051.0, 2.0 ** -25, 3 * 2.0 ** -25,
                1.5 * 2.0 ** -24, 2.0 ** -15 + 2.0 ** -26, -2.0 ** -20, 65504.0, 65519.99, 65520.0, -65520.0, 1e6, -1e6,
                0.0, -0.0, 1e-10, 0.1]
F16_SPECIALS = [2.0 ** -24, -3 * 2.0 ** -24, 2.0 ** -14 - 2.0 ** -24, 65504.0, -65504.0, -0.0, 0.0, 1 + 2.0 ** -10]


def _src_values(g, shape, dt):
    x = torch.randn(shape, generator=g) * 2
    sp = torch.tensor(F32_SPECIALS if dt == "f32" else F16_SPECIALS, dtype=torch.float32)
    flat = x.reshape(-1)
    n = min(flat.numel() // 3, 3 * sp.numel())
    flat[:3 * n:3] = sp.repeat(3)[:n]
    return x.to(TDT[dt])


NCDHW_ROWS = [
    # (launch, entry, src dtype, dst dtype, N, C, T, H, W, c_pad, dst row stride)
    ("ncdhw_to_ndhwc_kernel", "pv_ncdhw_to_ndhwc", "f32", "f16", 2, 3, 3, 9, 11, 4, 8),
    ("ncdhw_to_ndhwc_kernel", "pv_ncdhw_to_ndhwc", "f32", "f32", 2, 3, 3, 9, 11, 4, 8),
    ("ncdhw_to_ndhwc_kernel", "pv_ncdhw_to_ndhwc", "f16", "f16", 2, 3, 2, 7, 9, 4, 16),
    ("ncdhw_to_ndhwc_kernel", "pv_ncdhw_to_ndhwc", "f16", "f32", 1, 3, 2, 7, 9, 4, 8),
    ("ncdhw_to_ndhwc_kernel", "pv_ncdhw_to_ndhwc", "f32", "f16", 2, 10, 2, 7, 9, 16, 24),
    ("ncdhw_to_ndhwc_kernel", "pv_ncdhw_to_ndhwc", "f32", "f32", 1, 10, 2, 7, 9, 16, 24),
    ("ncdhw_to_ndhwc_kernel", "pv_ncdhw_to_ndhwc", "f16", "f16", 1, 10, 3, 5, 9, 16, 24),
    ("ncdhw_to_ndhwc_kernel", "pv_ncdhw_to_ndhwc", "f16", "f32", 2, 10, 3, 5, 9, 16, 32),
    # the token cast of engine/plan.py: N = C = T = H = 1, W = every element (not a multiple of 256)
    ("ncdhw_to_ndhwc_kernel", "pv_ncdhw_to_ndhwc", "f32", "f16", 1, 1, 1, 1, 18920, 1, 1),
    ("ncdhw_to_ndhwc_kernel", "pv_ncdhw_to_ndhwc", "f32", "f32", 1, 1, 1, 1, 18920, 1, 1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("row", NCDHW_ROWS, ids=_ids(NCDHW_ROWS))
def test_ncdhw_to_ndhwc_row(row):
    name, entry, sdt, ddt, N, C, T, H, W, c_pad, drs = row
    x = _src_values(_gen(row), (N, C, T, H, W), sdt)
    M = N * T * H * W
    want = _sentinel_cpu(M * drs + TAIL, TDT[ddt])
    wv = want[:M * drs].view(M, drs)
    wv[:, :C] = x.permute(0, 2, 3, 4, 1).reshape(M, C).to(TDT[ddt])
    wv[:, C:c_pad] = 0
    out = _sentinel_cpu(M * drs + TAIL, TDT[ddt]).to(_dev())
    xd = x.to(_dev())
    launched = _launch(entry, xd.data_ptr(), _code(sdt), out.data_ptr(), _code(ddt), N, C, T, H, W, c_pad, drs,
                       _stream())
    _expect(name, launched)
    _assert_bits(out, want, name)
    _exact("layout", row, launched)


QUAD = "ncdhw_f32_to_ndhwc4_padw_kernel"
GENERIC_PADW = "ncdhw_to_ndhwc_padw_kernel"
PADW_ROWS = [
    # (launch, entry, src dtype, dst dtype, N, C, T, H, W, c_pad, w_pad, w_phys, source offset in elements)
    (QUAD, "pv_ncdhw_to_ndhwc_padw", "f32", "f16", 1, 1, 2, 5, 16, 4, 0, 16, 0),
    (QUAD, "pv_ncdhw_to_ndhwc_padw", "f32", "f16", 2, 2, 2, 5, 16, 4, 4, 24, 0),
    (QUAD, "pv_ncdhw_to_ndhwc_padw", "f32", "f16", 1, 3, 3, 4, 20, 4, 8, 32, 0),
    (QUAD, "pv_ncdhw_to_ndhwc_padw", "f32", "f16", 2, 4, 2, 3, 12, 4, 4, 24, 0),
    (QUAD, "pv_ncdhw_to_ndhwc_padw", "f32", "f16", 1, 3, 2, 3, 8, 4, 0, 12, 0),       # right padding only
    # every condition that refuses the quad path, one per row
    (GENERIC_PADW, "pv_ncdhw_to_ndhwc_padw", "f32", "f16", 1, 3, 2, 5, 10, 4, 4, 16, 0),   # W % 4
    (GENERIC_PADW, "pv_ncdhw_to_ndhwc_padw", "f32", "f16", 1, 3, 2, 5, 12, 4, 3, 16, 0),   # w_pad % 4
    (GENERIC_PADW, "pv_ncdhw_to_ndhwc_padw", "f32", "f16", 1, 3, 2, 5, 12, 4, 4, 18, 0),   # w_phys % 4
    (GENERIC_PADW, "pv_ncdhw_to_ndhwc_padw", "f16", "f16", 2, 3, 2, 5, 16, 4, 4, 24, 0),   # f16 source
    (GENERIC_PADW, "pv_ncdhw_to_ndhwc_padw", "f32", "f32", 1, 3, 2, 5, 16, 4, 4, 24, 0),   # f32 destination
    (GENERIC_PADW, "pv_ncdhw_to_ndhwc_padw", "f32", "f16", 1, 3, 2, 5, 16, 8, 4, 24, 0),   # c_pad 8
    (GENERIC_PADW, "pv_ncdhw_to_ndhwc_padw", "f16", "f32", 1, 5, 2, 3, 9, 8, 2, 13, 0),    # C > 4
    (GENERIC_PADW, "pv_ncdhw_to_ndhwc_padw", "f32", "f16", 2, 3, 2, 5, 16, 4, 4, 24, 1),   # source 4 bytes off 16
]


def quad_route(sdt, ddt, C, c_pad, W, w_pad, w_phys, src_off):
    """The condition under which pv_ncdhw_to_ndhwc_padw takes the quad kernel (16-byte aligned buffers assumed
    apart from the source offset)."""
    return (sdt == "f32" and ddt == "f16" and c_pad == 4 and C <= 4 and W % 4 == 0 and w_pad % 4 == 0 and
            w_phys % 4 == 0 and (src_off * 4) % 16 == 0)


def _padw_ref(x, ddt, c_pad, w_pad, w_phys):
    N, C, T, H, W = x.shape
    out = torch.zeros(N, T, H, w_phys, c_pad, dtype=TDT[ddt])
    out[:, :, :, w_pad:w_pad + W, :C] = x.permute(0, 2, 3, 4, 1).to(TDT[ddt])
    return out.reshape(-1)


def _padw_run(row, x, src_off):
    _, entry, sdt, ddt, N, C, T, H, W, c_pad, w_pad, w_phys, _ = row
    src = torch.zeros(x.numel() + 8, dtype=TDT[sdt], device=_dev())
    src[src_off:src_off + x.numel()] = x.reshape(-1).to(_dev())
    total = N * T * H * w_phys * c_pad
    out = _sentinel_cpu(total + TAIL, TDT[ddt]).to(_dev())
    launched = _launch(entry, src.data_ptr() + src_off * src.element_size(), _code(sdt), out.data_ptr(), _code(ddt),
                       N, C, T, H, W, c_pad, w_pad, w_phys, _stream())
    return out, launched


@pytest.mark.gpu
@pytest.mark.parametrize("row", PADW_ROWS, ids=_ids(PADW_ROWS))
def test_ncdhw_to_ndhwc_padw_row(row):
    name, entry, sdt, ddt, N, C, T, H, W, c_pad, w_pad, w_phys, off = row
    x = _src_values(_gen(row), (N, C, T, H, W), sdt)
    want = _sentinel_cpu(N * T * H * w_phys * c_pad + TAIL, TDT[ddt])
    want[:-TAIL] = _padw_ref(x, ddt, c_pad, w_pad, w_phys)
    out, launched = _padw_run(row, x, off)
    _expect(name, launched)
    _assert_bits(out, want, name)
    if name == GENERIC_PADW and quad_route(sdt, ddt, C, c_pad, W, w_pad, w_phys, 0):
        # the same operands 16-byte aligned take the quad kernel: byte-identical output
        out_q, launched_q = _padw_run(row, x, 0)
        _expect(QUAD, launched_q)
        assert torch.equal(_bits(out_q), _bits(out)), "quad and generic outputs differ"
    _exact("layout-padw", row, launched)


TO_NCDHW_ROWS = [
    # (launch, entry, src dtype, N, C, T, H, W, src row stride): pad channels hold BIG, which must not appear
    ("ndhwc_to_ncdhw_kernel", "pv_ndhwc_to_ncdhw", "f16", 2, 24, 3, 5, 7, 32),
    ("ndhwc_to_ncdhw_kernel", "pv_ndhwc_to_ncdhw", "f32", 2, 24, 3, 5, 7, 40),
    ("ndhwc_to_ncdhw_kernel", "pv_ndhwc_to_ncdhw", "f16", 1, 400, 1, 1, 1, 408),
    ("ndhwc_to_ncdhw_kernel", "pv_ndhwc_to_ncdhw", "f32", 3, 10, 2, 9, 9, 16),
]


@pytest.mark.gpu
@pytest.mark.parametrize("row", TO_NCDHW_ROWS, ids=_ids(TO_NCDHW_ROWS))
def test_ndhwc_to_ncdhw_row(row):
    name, entry, sdt, N, C, T, H, W, srs = row
    x = _src_values(_gen(row), (N, C, T, H, W), sdt)
    M = N * T * H * W
    src = _rows_buffer(x.permute(0, 2, 3, 4, 1).reshape(M, C), srs, TDT[sdt], fill=BIG).to(_dev())
    want = _sentinel_cpu(x.numel() + TAIL, torch.float32)
    want[:-TAIL] = x.float().reshape(-1)
    out = _sentinel_cpu(x.numel() + TAIL, torch.float32).to(_dev())
    launched = _launch(entry, src.data_ptr(), _code(sdt), srs, out.data_ptr(), N, C, T, H, W, _stream())
    _expect(name, launched)
    _assert_bits(out, want, name)
    _exact("layout", row, launched)


COPY_ROWS = [
    # (launch, entry, dtype, rows, C, src row stride, dst row stride): rows * C / 8 not a multiple of 256
    ("copy_rows_kernel", "pv_copy_rows", "f16", 37, 24, 32, 40),
    ("copy_rows_kernel", "pv_copy_rows", "f32", 37, 24, 40, 32),
    ("copy_rows_kernel", "pv_copy_rows", "f16", 301, 96, 288, 96),
    ("copy_rows_kernel", "pv_copy_rows", "f32", 3, 2000, 2008, 2016),
]


@pytest.mark.gpu
@pytest.mark.parametrize("row", COPY_ROWS, ids=_ids(COPY_ROWS))
def test_copy_rows_row(row):
    name, entry, dt, R, C, ss, ds = row
    x = _src_values(_gen(row), (R, C), dt)
    src = _rows_buffer(x, ss, TDT[dt], fill=BIG).to(_dev())
    want = _rows_buffer(x, ds, TDT[dt])
    out = _sentinel_cpu(R * ds + TAIL, TDT[dt]).to(_dev())
    launched = _launch(entry, src.data_ptr(), out.data_ptr(), _code(dt), R, C, ss, ds, _stream())
    _expect(name, launched)
    _assert_bits(out, want, name)
    _exact("copy_rows", row, launched)


# =====================================================================================================================
# Pooling
# =====================================================================================================================
# Max pooling is exact (bit-exact against F.max_pool3d: padding is -inf).  Average pooling sums the in-bounds taps in
# fp32 in (kt, kh, kw) order and multiplies by the fp32 1 / (kt kh kw) (torch's count_include_pad=True): the sum of
# at most K = kt kh kw terms is off by (K - 1) 2^-24 sum|x|, the rounded reciprocal and the product add 2 roundings,
# so |err| <= (K + 1) 2^-24 avg|x| + the storage rounding.  The global kernel sums npos / 32 positions per lane, then
# the 32 lanes in sequence: K = ceil(npos / 32) + 32.
GLOBAL = "global_pool_kernel"
POOL3D = "pool3d_kernel"
POOL_ROWS = [
    # (launch, entry, dtype, mode, N, C, (T, H, W), kernel, stride, padding, x row stride, y row stride,
    #  cls rows ahead of every sample (batch strides, pointers one row in), input kind)
    (POOL3D, "pv_pool3d_fwd", "f32", "max", 2, 24, (4, 11, 11), (1, 3, 3), (1, 2, 2), (0, 1, 1), 24, 24, 0, "randn"),
    (POOL3D, "pv_pool3d_fwd", "f32", "avg", 2, 24, (4, 11, 11), (4, 5, 5), (1, 1, 1), (0, 0, 0), 24, 24, 0, "randn"),
    (POOL3D, "pv_pool3d_fwd", "f32", "max", 2, 24, (4, 11, 11), (3, 3, 3), (1, 2, 2), (1, 1, 1), 24, 24, 0, "randn"),
    (POOL3D, "pv_pool3d_fwd", "f32", "avg", 2, 24, (4, 11, 11), (2, 1, 1), (2, 1, 1), (0, 0, 0), 24, 24, 0, "randn"),
    # padding on every axis / on one axis over all-negative inputs: the padding must not act as 0
    (POOL3D, "pv_pool3d_fwd", "f16", "max", 2, 16, (3, 6, 5), (3, 3, 3), (1, 1, 1), (1, 1, 1), 16, 16, 0, "neg"),
    (POOL3D, "pv_pool3d_fwd", "f32", "max", 1, 16, (5, 4, 4), (3, 1, 1), (2, 1, 1), (1, 0, 0), 16, 16, 0, "neg"),
    (POOL3D, "pv_pool3d_fwd", "f16", "max", 1, 8, (2, 3, 7), (1, 3, 1), (1, 2, 1), (0, 1, 0), 8, 8, 0, "neg"),
    (POOL3D, "pv_pool3d_fwd", "f16", "max", 1, 8, (2, 3, 7), (1, 1, 3), (1, 1, 2), (0, 0, 1), 8, 8, 0, "neg"),
    # padded average pool: divides by kt kh kw, padded taps included
    (POOL3D, "pv_pool3d_fwd", "f16", "avg", 2, 16, (4, 7, 7), (3, 3, 3), (2, 2, 2), (1, 1, 1), 16, 16, 0, "randn"),
    (POOL3D, "pv_pool3d_fwd", "f32", "avg", 1, 8, (3, 5, 9), (3, 3, 3), (1, 2, 2), (1, 1, 1), 8, 8, 0, "neg"),
    # stride larger than the kernel, odd extents
    (POOL3D, "pv_pool3d_fwd", "f16", "max", 2, 16, (5, 9, 7), (1, 2, 2), (2, 3, 3), (0, 0, 0), 16, 16, 0, "randn"),
    (POOL3D, "pv_pool3d_fwd", "f32", "avg", 1, 16, (5, 9, 7), (1, 2, 2), (2, 3, 3), (0, 0, 0), 16, 16, 0, "randn"),
    # row strides wider than C
    (POOL3D, "pv_pool3d_fwd", "f16", "avg", 2, 16, (3, 6, 6), (1, 3, 3), (1, 2, 2), (0, 1, 1), 24, 32, 0, "randn"),
    (POOL3D, "pv_pool3d_fwd", "f32", "max", 1, 16, (3, 6, 6), (1, 3, 3), (1, 2, 2), (0, 1, 1), 32, 24, 0, "randn"),
    # MViT's K / Q / V pools: one cls row ahead of every sample, q|k|v buffer rows (x row stride 3 C)
    (POOL3D, "pv_pool3d_fwd", "f16", "max", 2, 96, (2, 8, 8), (3, 3, 3), (1, 2, 2), (1, 1, 1), 288, 96, 1, "randn"),
    (POOL3D, "pv_pool3d_fwd", "f32", "avg", 3, 32, (2, 6, 6), (3, 3, 3), (1, 4, 4), (1, 1, 1), 96, 40, 1, "randn"),
    (POOL3D, "pv_pool3d_fwd", "f16", "max", 2, 16, (2, 5, 5), (3, 3, 3), (1, 1, 1), (1, 1, 1), 16, 16, 1, "neg"),
    # global pools (the head): last 64-channel slab partial (432), one position, wide rows
    (GLOBAL, "pv_pool3d_fwd", "f16", "avg", 2, 432, (4, 14, 14), (4, 14, 14), (1, 1, 1), (0, 0, 0), 432, 440, 0, "randn"),
    (GLOBAL, "pv_pool3d_fwd", "f16", "max", 2, 432, (4, 14, 14), (4, 14, 14), (1, 1, 1), (0, 0, 0), 440, 432, 0, "neg"),
    (GLOBAL, "pv_pool3d_fwd", "f32", "avg", 2, 2048, (4, 14, 14), (4, 14, 14), (1, 1, 1), (0, 0, 0), 2048, 2056, 0, "randn"),
    (GLOBAL, "pv_pool3d_fwd", "f32", "max", 1, 2048, (1, 1, 1), (1, 1, 1), (1, 1, 1), (0, 0, 0), 2048, 2048, 0, "randn"),
    (GLOBAL, "pv_pool3d_fwd", "f16", "avg", 3, 432, (1, 1, 1), (1, 1, 1), (1, 1, 1), (0, 0, 0), 432, 440, 0, "randn"),
    # whole-extent pools that must NOT take the global kernel: batch strides (cls row), padding
    (POOL3D, "pv_pool3d_fwd", "f16", "avg", 2, 64, (2, 5, 5), (2, 5, 5), (1, 1, 1), (0, 0, 0), 64, 64, 1, "randn"),
    (POOL3D, "pv_pool3d_fwd", "f16", "max", 2, 64, (2, 5, 5), (2, 7, 7), (1, 1, 1), (0, 1, 1), 64, 64, 0, "neg"),
    (POOL3D, "pv_pool3d_fwd", "f32", "avg", 1, 16, (2, 5, 5), (2, 7, 7), (1, 1, 1), (0, 1, 1), 16, 16, 0, "randn"),
]


def _pool_out(shape, k, s, p):
    return tuple((shape[i] + 2 * p[i] - k[i]) // s[i] + 1 for i in range(3))


def pool_route(shape, k, p, cls):
    out = _pool_out(shape, k, (1, 1, 1), p)
    return GLOBAL if (out == (1, 1, 1) and tuple(k) == tuple(shape) and tuple(p) == (0, 0, 0) and not cls) else POOL3D


def pool_inputs(row):
    name, entry, dt, mode, N, C, shape, k, s, p, xrs, yrs, cls, kind = row
    x = torch.randn(N, C, *shape, generator=_gen(row))
    if kind == "neg":
        x = -(x.abs() + 0.25)
    return _f16(x)


def pool_ref64(x, row):
    """(ref, absref, K) as [N, npos_out, C]."""
    name, entry, dt, mode, N, C, shape, k, s, p, xrs, yrs, cls, kind = row
    pad = (p[2], p[2], p[1], p[1], p[0], p[0])
    x64 = x.double()
    if mode == "max":       # explicit padding: torch rejects extents below the kernel even when padded
        ref = F.max_pool3d(F.pad(x64, pad, value=-math.inf), k, s)
        absref = ref.abs()
    else:                   # count_include_pad=True: zero padding, divide by kt kh kw
        ref = F.avg_pool3d(F.pad(x64, pad), k, s)
        absref = F.avg_pool3d(F.pad(x64.abs(), pad), k, s)
    K = (math.ceil(math.prod(shape) / 32) + 32) if name == GLOBAL else math.prod(k)
    rows = lambda t: t.permute(0, 2, 3, 4, 1).reshape(N, -1, C)       # noqa: E731
    return rows(ref), rows(absref), K


def avg_pool_emulate(x, row, mutation=None):
    """pool3d_kernel's average in fp32: in-bounds taps summed in (kt, kh, kw) order, times the fp32 reciprocal of
    kt kh kw.  mutation "valid_count": divide by the number of in-bounds taps."""
    name, entry, dt, mode, N, C, shape, k, s, p, xrs, yrs, cls, kind = row
    To, Ho, Wo = _pool_out(shape, k, s, p)
    xp = F.pad(x.float(), (p[2], p[2], p[1], p[1], p[0], p[0]))
    ones = F.pad(torch.ones(1, 1, *shape), (p[2], p[2], p[1], p[1], p[0], p[0]))
    acc = torch.zeros(N, C, To, Ho, Wo)
    cnt = torch.zeros(1, 1, To, Ho, Wo)
    for a in range(k[0]):
        for b in range(k[1]):
            for c in range(k[2]):
                sl = (slice(None), slice(None), slice(a, a + s[0] * (To - 1) + 1, s[0]),
                      slice(b, b + s[1] * (Ho - 1) + 1, s[1]), slice(c, c + s[2] * (Wo - 1) + 1, s[2]))
                acc = acc + xp[sl]
                cnt = cnt + ones[sl]
    if mutation == "valid_count":
        y = acc / cnt
    else:
        y = acc * torch.tensor(1.0 / math.prod(k), dtype=torch.float32)
    return y.permute(0, 2, 3, 4, 1).reshape(N, -1, C)


def max_pool_emulate(x, row, mutation=None):
    """mutation "pad_zero": the padding taps read as 0."""
    name, entry, dt, mode, N, C, shape, k, s, p, xrs, yrs, cls, kind = row
    pad = (p[2], p[2], p[1], p[1], p[0], p[0])
    y = F.max_pool3d(F.pad(x, pad, value=0.0 if mutation == "pad_zero" else -math.inf), k, s)
    return y.permute(0, 2, 3, 4, 1).reshape(N, -1, C)


@pytest.mark.gpu
@pytest.mark.parametrize("row", POOL_ROWS, ids=_ids(POOL_ROWS))
def test_pool_row(row):
    L = _L()
    name, entry, dt, mode, N, C, shape, k, s, p, xrs, yrs, cls, kind = row
    x = pool_inputs(row)
    To, Ho, Wo = _pool_out(shape, k, s, p)
    npi, npo = math.prod(shape), To * Ho * Wo
    xr = torch.full((N, cls + npi, C), BIG)          # cls rows hold BIG: a pool that reads them shows it
    xr[:, cls:] = x.permute(0, 2, 3, 4, 1).reshape(N, npi, C)
    xb = _rows_buffer(xr.reshape(-1, C), xrs, TDT[dt], fill=BIG).to(_dev())
    yn = N * (cls + npo) * yrs
    yb = _sentinel_cpu(yn + TAIL, TDT[dt]).to(_dev())
    d = L.Pool3dDesc()
    d.dtype, d.mode = _code(dt), L.POOL_MAX if mode == "max" else L.POOL_AVG
    d.N, d.Ti, d.Hi, d.Wi, d.C = N, shape[0], shape[1], shape[2], C
    d.To, d.Ho, d.Wo = To, Ho, Wo
    d.kt, d.kh, d.kw = k
    d.st, d.sh, d.sw = s
    d.pt, d.ph, d.pw = p
    d.x_row_stride, d.y_row_stride = xrs, yrs
    d.x_batch_stride, d.y_batch_stride = ((cls + npi) * xrs, (cls + npo) * yrs) if cls else (0, 0)
    esz = xb.element_size()
    launched = _launch(entry, ctypes.byref(d), xb.data_ptr() + cls * xrs * esz, yb.data_ptr() + cls * yrs * esz,
                       _stream())
    _expect(name, launched)
    yc = yb.cpu()
    written = torch.zeros(yn + TAIL, dtype=torch.bool)
    written[:yn].view(N, cls + npo, yrs)[:, cls:, :C] = True
    _assert_untouched(yc, written, name)
    got = yc[:yn].view(N, cls + npo, yrs)[:, cls:, :C]
    ref, absref, K = pool_ref64(x, row)
    if mode == "max":
        _assert_bits(got.contiguous(), ref.to(TDT[dt]), name)
        _exact("pool-max", row, launched)
    else:
        ratio = _assert_bound(got, ref, absref, K, acc_eps=SUM_EPS, what=name, rnd_eps=_rnd(dt))
        _ratio("pool-avg", row, ratio, launched)


# =====================================================================================================================
# Squeeze-Excitation
# =====================================================================================================================
# channel_sum: a CTA sums `chunk` positions; each thread adds its positions in fp32 (Lp of them), converts the partial
# to 64-bit fixed point (round to nearest of v 2^24: <= 2^-25 per partial, pv_common.cuh se_fix) and adds it with an
# integer atomic (exact).  |err| <= (Lp - 1) 2^-24 sum|x| + P 2^-25 over the P partials of a channel; the fixed-point
# term goes in extra64.
CS_ROWS = [
    # (launch, entry, dtype, N, npos, C, row stride): 256 / (C / 8) leaves idle threads; C > 2048 takes the
    # one-thread-per-channel-group branch; npos > 2048 splits into chunks; 2048 * 1024 + 40 hits the 1024-chunk cap
    ("channel_sum_kernel", "pv_channel_sum", "f16", 2, 300, 24, 32),
    ("channel_sum_kernel", "pv_channel_sum", "f32", 2, 5000, 56, 56),
    ("channel_sum_kernel", "pv_channel_sum", "f16", 1, 5000, 432, 440),
    ("channel_sum_kernel", "pv_channel_sum", "f32", 1, 700, 2056, 2056),
    ("channel_sum_kernel", "pv_channel_sum", "f16", 1, 2500, 4096, 4104),
    ("channel_sum_kernel", "pv_channel_sum", "f16", 1, 2048 * 1024 + 40, 8, 8),
]


def cs_geometry(npos, C):
    """(chunks, chunk, positions per iteration, Lp, P) of pv_channel_sum."""
    chunks = min(-(-npos // 2048), 1024)
    chunk = -(-npos // chunks)
    chunks = -(-npos // chunk)
    G = C // 8
    ppi = 256 // G if G <= 256 else 1
    return chunks, chunk, ppi, -(-chunk // ppi), chunks * min(ppi, chunk)


def cs_inputs(row):
    name, entry, dt, N, npos, C, rs = row
    return _f16(torch.randn(N, npos, C, generator=_gen(row)) + 0.5)


def cs_ref64(x, row):
    name, entry, dt, N, npos, C, rs = row
    _, _, _, Lp, P = cs_geometry(npos, C)
    x64 = x.double()
    return x64.sum(1), x64.abs().sum(1), Lp, torch.full((N, C), P * 2.0 ** -25, dtype=torch.float64)


def cs_emulate(x, row, mutation=None):
    """int64 fixed-point sums of channel_sum_kernel (mutation "drop_last_chunk": the last chunk never added)."""
    name, entry, dt, N, npos, C, rs = row
    chunks, chunk, ppi, Lp, P = cs_geometry(npos, C)
    xp = torch.zeros(N, chunks * chunk, C)
    xp[:, :npos] = x.float()
    xp = xp.view(N, chunks, chunk, C)
    if mutation == "drop_last_chunk":
        xp = xp[:, :chunks - 1]
    q = F.pad(xp, (0, 0, 0, Lp * ppi - chunk)).view(N, xp.shape[1], Lp, ppi, C)
    acc = torch.zeros(N, xp.shape[1], ppi, C)
    for i in range(Lp):                                  # thread pl adds positions pl, pl + ppi, ... of its chunk
        acc = acc + q[:, :, i]
    return torch.round(acc.double() * 2.0 ** 24).long().sum((1, 2))


@pytest.mark.gpu
@pytest.mark.parametrize("row", CS_ROWS, ids=_ids(CS_ROWS))
def test_channel_sum_row(row):
    name, entry, dt, N, npos, C, rs = row
    x = cs_inputs(row)
    xb = _rows_buffer(x.reshape(-1, C), rs, TDT[dt], fill=BIG).to(_dev())
    sums = torch.zeros(N * C + TAIL, dtype=torch.int64, device=_dev())
    sums[N * C:] = SENT[torch.int64]
    runs = []
    for _ in range(2):                                   # two launches: bit-identical sums
        sums[:N * C] = 0
        launched = _launch(entry, xb.data_ptr(), _code(dt), rs, N, npos, C, sums.data_ptr(), _stream())
        _expect(name, launched)
        runs.append(sums.cpu())
    assert torch.equal(runs[0], runs[1]), "channel sums differ between two launches"
    assert bool((runs[0][N * C:] == SENT[torch.int64]).all()), "written past the sums"
    got = runs[0][:N * C].view(N, C).double() * 2.0 ** -24
    ref, absref, Lp, extra = cs_ref64(x, row)
    ratio = _assert_bound(got, ref, absref, Lp, acc_eps=SUM_EPS, what=name, extra64=extra,
                                   rnd_eps=TS.F32_EPS)
    _ratio("se-channel-sum", row, ratio, launched)


# se_gate: mean = fp32(sum) * fp32(1 / npos) (3 roundings); hidden_j = relu(b1_j + sum_c w1[j, c_stride_w] mean_c) as
# an fmaf chain of C terms; a_c = b2_c + sum_j w2 hidden_j, Cr terms.  With H = |b1| + |w1| |mean| and A = |b2| + |w2| H,
# |err(a)| <= (C + Cr + 3) 2^-24 A; the sigmoid's slope is <= 1/4, so absref = A / 4.  __expf(-a) adds
# (2 + 1.173 |a|) ulp, carried by g (1 - g), and 1 + e plus the division one rounding each (extra64).
SE_GATE_ROWS = [
    # (launch, entry, N, C, Cr, c_stride_w, npos)
    ("se_gate_kernel", "pv_se_gate", 2, 24, 8, 32, 300),
    ("se_gate_kernel", "pv_se_gate", 2, 432, 1, 440, 784),
    ("se_gate_kernel", "pv_se_gate", 1, 56, 300, 64, 50),
    ("se_gate_kernel", "pv_se_gate", 3, 2056, 8, 2064, 49),
]


def se_gate_inputs(row):
    name, entry, N, C, Cr, cs, npos = row
    g = _gen(row)
    mean = torch.randn(N, C, generator=g)
    sums = torch.round(mean.double() * npos * 2.0 ** 24).long()
    w1 = torch.randn(Cr, cs, generator=g) / math.sqrt(C)          # columns [C, c_stride_w) are never read
    b1 = torch.rand(Cr, generator=g) - 0.5
    w2 = torch.randn(C, Cr, generator=g) / math.sqrt(Cr)
    b2 = torch.rand(C, generator=g) - 0.5
    return sums, w1, b1, w2, b2


def se_gate_ref64(inp, row):
    name, entry, N, C, Cr, cs, npos = row
    sums, w1, b1, w2, b2 = inp
    mean = sums.double() * 2.0 ** -24 / npos
    w1c = w1[:, :C].double()
    hid = (b1.double() + mean @ w1c.t()).clamp_min(0)
    a = b2.double() + hid @ w2.double().t()
    gate = torch.sigmoid(a)
    H = b1.double().abs() + mean.abs() @ w1c.abs().t()
    A = b2.double().abs() + H @ w2.double().abs().t()
    extra = gate * (1 - gate) * (2 + 1.173 * a.abs()) * 2.0 ** -23 + U * gate
    return gate, 0.25 * A, C + Cr + 3, extra


def se_gate_emulate(inp, row, mutation=None):
    """mutation "w1_stride_c": W1 read with row stride C instead of c_stride_w."""
    name, entry, N, C, Cr, cs, npos = row
    sums, w1, b1, w2, b2 = inp
    inv = torch.tensor(1.0 / npos, dtype=torch.float32)
    mean = (sums.double() * 2.0 ** -24).float() * inv
    w1r = w1.reshape(-1)[:Cr * C].view(Cr, C) if mutation == "w1_stride_c" else w1[:, :C]
    a = b1.view(1, Cr).expand(N, Cr).clone()
    for c in range(C):
        a = _fma32(w1r[:, c].view(1, Cr), mean[:, c:c + 1], a)
    hid = a.clamp_min(0)
    o = b2.view(1, C).expand(N, C).clone()
    for j in range(Cr):
        o = _fma32(w2[:, j].view(1, C), hid[:, j:j + 1], o)
    return 1 / (1 + torch.exp(-o))


@pytest.mark.gpu
@pytest.mark.parametrize("row", SE_GATE_ROWS, ids=_ids(SE_GATE_ROWS))
def test_se_gate_row(row):
    name, entry, N, C, Cr, cs, npos = row
    inp = se_gate_inputs(row)
    sums, w1, b1, w2, b2 = (t.to(_dev()).contiguous() for t in inp)
    gate = _sentinel_cpu(N * C + TAIL, torch.float32).to(_dev())
    launched = _launch(entry, sums.data_ptr(), npos, N, C, Cr, w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                       b2.data_ptr(), cs, gate.data_ptr(), _stream())
    _expect(name, launched)
    gc = gate.cpu()
    written = torch.zeros(N * C + TAIL, dtype=torch.bool)
    written[:N * C] = True
    _assert_untouched(gc, written, name)
    ref, absref, K, extra = se_gate_ref64(inp, row)
    ratio = _assert_bound(gc[:N * C].view(N, C), ref, absref, K, acc_eps=SUM_EPS, what=name, extra64=extra,
                                   rnd_eps=TS.F32_EPS)
    _ratio("se-gate", row, ratio, launched)


# scale_act: v = x * gate in fp32 (one rounding, 2^-24 |v|, through the activation's slope L: absref = L |v| with
# acc_eps 2^-24, K = 0), then apply_act in fp32 (act_err64) and the storage rounding.
SCALE_ACT_ROWS = [
    # (launch, entry, dtype, N, npos, C, x row stride, y row stride, gate, activation, in place)
    ("scale_act_kernel", "pv_scale_act", dt, 2, 197, 48, xrs, yrs, gate, act, inplace)
    for act in ACTS
    for dt, xrs, yrs, gate, inplace in (("f16", 56, 56, True, True), ("f32", 56, 64, False, False))
] + [
    ("scale_act_kernel", "pv_scale_act", "f16", 3, 50, 40, 48, 40, True, "hswish", False),
    ("scale_act_kernel", "pv_scale_act", "f32", 2, 33, 432, 432, 432, True, "swish", True),
    ("scale_act_kernel", "pv_scale_act", "f16", 2, 33, 24, 24, 32, False, "relu", False),
    ("scale_act_kernel", "pv_scale_act", "f32", 1, 77, 16, 24, 24, False, "gelu", True),
]


def scale_act_inputs(row):
    name, entry, dt, N, npos, C, xrs, yrs, has_gate, act, inplace = row
    g = _gen(row)
    x = torch.randn(N * npos, C, generator=g) * 3
    x = _f16(x) if dt == "f16" else x
    gate = (torch.rand(N, C, generator=g) + 0.25) if has_gate else None
    return x, gate


def scale_act_ref64(inp, row):
    name, entry, dt, N, npos, C, xrs, yrs, has_gate, act, inplace = row
    x, gate = inp
    v = x.double()
    if gate is not None:
        v = v * gate.double().repeat_interleave(npos, 0)
    return act64(v, act), LIP[act] * v.abs(), act_err64(v, act)


def scale_act_emulate(inp, row, mutation=None):
    name, entry, dt, N, npos, C, xrs, yrs, has_gate, act, inplace = row
    x, gate = inp
    v = x.float() if gate is None else x.float() * gate.repeat_interleave(npos, 0)
    return act32(v, act)


@pytest.mark.gpu
@pytest.mark.parametrize("row", SCALE_ACT_ROWS, ids=_ids(SCALE_ACT_ROWS))
def test_scale_act_row(row):
    name, entry, dt, N, npos, C, xrs, yrs, has_gate, act, inplace = row
    x, gate = scale_act_inputs(row)
    R = N * npos
    xb = _rows_buffer(x, xrs, TDT[dt]).to(_dev())          # pad channels hold the sentinel (in place: must survive)
    yb = xb if inplace else _sentinel_cpu(R * yrs + TAIL, TDT[dt]).to(_dev())
    gd = gate.to(_dev()).contiguous() if gate is not None else None
    launched = _launch(entry, xb.data_ptr(), yb.data_ptr(), _code(dt), xrs, yrs, N, npos, C,
                       gd.data_ptr() if gd is not None else None, _act_code(act), _stream())
    _expect(name, launched)
    yc = yb.cpu()
    _assert_untouched(yc, _written(R, yrs, C), name)
    got = yc[:R * yrs].view(R, yrs)[:, :C]
    ref, absref, extra = scale_act_ref64((x, gate), row)
    ratio = _assert_bound(got, ref, absref, 0, acc_eps=U, what=name, extra64=extra, rnd_eps=_rnd(dt))
    _ratio("se-scale-act", row, ratio, launched)


# =====================================================================================================================
# Head: per-position softmax over the C_valid channels (optional), then the mean over positions, fp32 out
# =====================================================================================================================
# softmax: d = x - max is one rounding (2^-24 |d| relative on e^d), expf is within 2 ulp (2^-22); the sum of the e^d
# takes D = ceil(C / 256) + 5 + 8 additions (per thread, warp butterfly, 8 warps) of positive terms, 1 / sum and the
# product 2 roundings.  Per position the probability p is off by p (rel_c + max_c rel_c + (D + 2) 2^-24); the mean adds
# npos + 1 roundings of mean(p).  acc term: absref = mean(p), K = npos + D + 3; the expf / subtraction terms go in
# extra64.  Without softmax: (npos + 1) 2^-24 mean|x|.
HEAD_ROWS = [
    # (launch, entry, dtype, N, npos, C_valid, row stride, softmax, input kind); pad channels hold 60000
    ("head_reduce_kernel", "pv_head_reduce", "f16", 2, 392, 400, 408, 1, "randn"),
    ("head_reduce_kernel", "pv_head_reduce", "f32", 2, 1, 600, 616, 1, "randn"),
    ("head_reduce_kernel", "pv_head_reduce", "f16", 3, 1, 1, 8, 1, "randn"),
    ("head_reduce_kernel", "pv_head_reduce", "f16", 2, 392, 8, 16, 1, "randn"),
    ("head_reduce_kernel", "pv_head_reduce", "f16", 2, 392, 8, 16, 0, "randn"),
    ("head_reduce_kernel", "pv_head_reduce", "f32", 1, 392, 600, 608, 0, "randn"),
    ("head_reduce_kernel", "pv_head_reduce", "f16", 2, 1, 400, 408, 0, "randn"),
    ("head_reduce_kernel", "pv_head_reduce", "f32", 1, 1, 1, 8, 0, "randn"),
    # one channel 60 above the rest (around 40: e^x of the maximum overflows fp32 without the max subtraction)
    ("head_reduce_kernel", "pv_head_reduce", "f16", 2, 7, 400, 408, 1, "peak60"),
    ("head_reduce_kernel", "pv_head_reduce", "f32", 1, 392, 600, 608, 1, "peak60"),
    # rows of equal values
    ("head_reduce_kernel", "pv_head_reduce", "f32", 2, 5, 8, 16, 1, "equal"),
    ("head_reduce_kernel", "pv_head_reduce", "f16", 1, 3, 600, 608, 1, "equal"),
]


def head_inputs(row):
    name, entry, dt, N, npos, C, rs, softmax, kind = row
    g = _gen(row)
    if kind == "equal":
        x = (torch.randn(N, npos, 1, generator=g) * 3).expand(N, npos, C).contiguous()
    elif kind == "peak60":
        x = 40 + torch.randn(N, npos, C, generator=g)
        idx = torch.randint(0, C, (N, npos, 1), generator=g)
        x.scatter_(2, idx, x.max(2, keepdim=True).values + 60)
    else:
        x = torch.randn(N, npos, C, generator=g) * 3
    return _f16(x) if dt == "f16" else x


def head_ref64(x, row):
    name, entry, dt, N, npos, C, rs, softmax, kind = row
    x64 = x.double()
    if not softmax:
        return x64.mean(1), x64.abs().mean(1), npos + 1, None
    p = torch.softmax(x64, 2)
    d = x64 - x64.max(2, keepdim=True).values
    rel = 2.0 ** -22 + U * d.abs()
    extra = (p * (rel + rel.max(2, keepdim=True).values)).mean(1)
    D = -(-C // 256) + 13
    return p.mean(1), p.mean(1), npos + D + 3, extra


def head_emulate(x, row, mutation=None):
    """head_reduce_kernel in fp32.  mutations: "no_max" (softmax without the max subtraction), "mean_over_c"."""
    name, entry, dt, N, npos, C, rs, softmax, kind = row
    x = x.float()
    acc = torch.zeros(N, C)
    for p in range(npos):
        v = x[:, p]
        if softmax:
            mx = v.max(1, keepdim=True).values
            e = torch.exp(v if mutation == "no_max" else v - mx)
            nrep = -(-C // 256)
            ep = F.pad(e, (0, nrep * 256 - C)).view(N, nrep, 256)
            t = torch.zeros(N, 256)
            for i in range(nrep):                       # thread t: channels t, t + 256, ...
                t = t + ep[:, i]
            t = t.view(N, 8, 32)
            lane = torch.arange(32)
            for o in (16, 8, 4, 2, 1):                  # warp butterfly
                t = t + t[:, :, lane ^ o]
            sm = torch.zeros(N)
            for w in range(8):
                sm = sm + t[:, w, 0]
            v = e * (1 / sm).view(N, 1)
        acc = acc + v
    return acc * torch.tensor(1.0 / (C if mutation == "mean_over_c" else npos), dtype=torch.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("row", HEAD_ROWS, ids=_ids(HEAD_ROWS))
def test_head_reduce_row(row):
    name, entry, dt, N, npos, C, rs, softmax, kind = row
    x = head_inputs(row)
    xb = _rows_buffer(x.reshape(-1, C), rs, TDT[dt], fill=BIG).to(_dev())
    out = _sentinel_cpu(N * C + TAIL, torch.float32).to(_dev())
    launched = _launch(entry, xb.data_ptr(), _code(dt), rs, N, npos, C, softmax, out.data_ptr(), _stream())
    _expect(name, launched)
    oc = out.cpu()
    written = torch.zeros(N * C + TAIL, dtype=torch.bool)
    written[:N * C] = True
    _assert_untouched(oc, written, name)
    ref, absref, K, extra = head_ref64(x, row)
    ratio = _assert_bound(oc[:N * C].view(N, C), ref, absref, K, acc_eps=SUM_EPS, what=name, extra64=extra,
                                   rnd_eps=TS.F32_EPS)
    _ratio("head", row, ratio, launched)


# =====================================================================================================================
# LayerNorm
# =====================================================================================================================
# A row is summed by `lpr` lanes, NCH * 8 values per lane in sequence, then a butterfly over the lanes: depth
# D = NCH * 8 + log2(lpr) (the generic kernel: lpr = 32, NCH = ceil(C / 256)).  The mean is off by
# dmu <= (D + 1) 2^-24 mean|x|, which shifts every output by |g| rstd dmu.  The centred sum of squares (fmaf chain,
# same depth) is off by (D + 2) 2^-24 relative plus the second-order C dmu^2; q / C and + eps one rounding each;
# rsqrtf is within 2 ulp (2^-22): rstd is off by (D + 4) / 2 2^-24 + 2^-22 + (rstd dmu)^2 / 2 relative.  The output
# (x - mean) rstd g + b takes <= 4 roundings.  acc term: absref = |g| (rstd mean|x| + |x^|) + |b|, K = D + 5; rsqrtf
# and the second-order term go in extra64.
REG, GEN = "layernorm_reg_kernel", "layernorm_kernel"
LN_ROWS = [
    # (launch, entry, dtype, rows, groups, groups per set, C, x row stride, y row stride, cls every npos rows (0: no
    #  cls rows), in place, input kind, gamma / beta offset in floats)
] + [(REG if C <= 768 else GEN, "pv_layernorm", dt, rows, 1, 1, C, C, C, 0, False, "randn", 0)
     for dt in ("f32", "f16")
     for rows, C in ((77, 96), (5, 8), (130, 192), (33, 384), (19, 768), (7, 1024), (64, 40))] + [
    # pooled K | V of an MViT block: groups = 2 heads-sets, one in-place launch, cls rows from the un-pooled buffer
    (REG, "pv_layernorm_sets", dt, B * npos, 2 * heads, heads, hd, 2 * heads * hd, 2 * heads * hd, npos, True, "randn",
     0) for dt in ("f16", "f32") for B, npos, heads, hd in ((3, 11, 2, 96), (2, 50, 4, 96), (2, 7, 1, 8))] + [
    # the remaining (lanes per row, chunks per lane) pairs and a partial last block
    (REG, "pv_layernorm", "f32", 45, 1, 1, 256, 256, 256, 0, False, "randn", 0),
    (REG, "pv_layernorm", "f16", 13, 1, 1, 520, 520, 520, 0, False, "randn", 0),
    # wide input rows, several groups of one set, in place / out of place
    (REG, "pv_layernorm", "f16", 21, 3, 3, 40, 128, 136, 0, False, "randn", 0),
    (REG, "pv_layernorm_sets", "f32", 3 * 9, 4, 2, 24, 104, 104, 9, True, "randn", 0),
    (REG, "pv_layernorm_sets", "f16", 2 * 17, 2, 1, 384, 776, 784, 17, False, "randn", 0),
    # |mean| >> std (a one-pass variance cancels) and a small std (eps inside the square root matters)
    (REG, "pv_layernorm", "f32", 33, 1, 1, 768, 768, 768, 0, False, "hard", 0),
    (REG, "pv_layernorm", "f32", 40, 1, 1, 96, 96, 96, 0, False, "hard", 0),
    (REG, "pv_layernorm", "f32", 40, 1, 1, 40, 40, 40, 0, False, "tiny", 0),
    (REG, "pv_layernorm", "f16", 40, 1, 1, 96, 96, 96, 0, False, "tiny", 0),
    # the generic kernel: C > 768, and gamma / beta 4 bytes off 16-byte alignment
    (GEN, "pv_layernorm", "f16", 9, 1, 1, 1032, 1040, 1040, 0, True, "randn", 0),
    (GEN, "pv_layernorm", "f32", 5, 1, 1, 1024, 1024, 1024, 0, False, "hard", 0),
    (GEN, "pv_layernorm", "f32", 77, 1, 1, 96, 96, 96, 0, False, "randn", 1),
    (GEN, "pv_layernorm", "f16", 33, 1, 1, 384, 392, 384, 0, False, "tiny", 1),
    (GEN, "pv_layernorm_sets", "f16", 2 * 5, 2, 1, 96, 192, 192, 5, True, "randn", 1),
]
LN_EPS = 1e-6


def ln_inputs(row):
    """(x [rows, groups * C] fp32 on the storage grid, cls source [B, src_npos, src_rs] or None, gamma, beta [sets, C])."""
    name, entry, dt, rows, groups, gps, C, xrs, yrs, cnpos, inplace, kind, goff = row
    g = _gen(row)

    def draw(*shape):
        if kind == "hard":
            v = 1e3 + 1e-2 * torch.randn(*shape, generator=g)
        elif kind == "tiny":
            v = 1e-2 * torch.randn(*shape, generator=g)
        else:
            v = torch.randn(*shape, generator=g) * 3 + 1
        return _f16(v) if dt == "f16" else v
    x = draw(rows, groups * C)
    cls = None
    if cnpos:
        B = rows // cnpos
        cls = torch.full((B, cnpos + 9, 3 * groups * C), BIG)
        cls[:, 0, groups * C:2 * groups * C] = draw(B, groups * C)
        x.view(B, cnpos, -1)[:, 0] = BIG                 # the rows the cls source replaces are never read
    nsets = groups // gps
    gamma = torch.rand(nsets, C, generator=g) + 0.5
    beta = torch.rand(nsets, C, generator=g) - 0.5
    return x, cls, gamma, beta


def _ln_eff(x, cls, row):
    """The rows the kernel normalises: x with every npos-th row taken from the cls source."""
    name, entry, dt, rows, groups, gps, C, xrs, yrs, cnpos, inplace, kind, goff = row
    v = x.clone()
    if cls is not None:
        v.view(rows // cnpos, cnpos, -1)[:, 0] = cls[:, 0, groups * C:2 * groups * C]
    return v.view(rows, groups, C)


def ln_emulate(v, gamma, beta, gps, lpr, nch, eps=LN_EPS, mutation=None):
    """The row-in-registers LayerNorm in fp32 (the generic kernel is the same with lpr = 32).  mutations:
    "one_pass" (E[x^2] - E[x]^2), "var_c_minus_1", "eps_outside" (1 / (sqrt(var) + eps)), "gamma_set0"."""
    R, G, C = v.shape
    v = v.float().reshape(R * G, C)
    cols = torch.tensor([[(sl + i * lpr) * 8 + e for i in range(nch) for e in range(8)] for sl in range(lpr)])
    vp = F.pad(v, (0, lpr * nch * 8 + 8 - C))
    cols = torch.where(cols < C, cols, torch.full_like(cols, vp.shape[1] - 1))    # a zero column
    lanes = vp[:, cols]                                  # [rows, lpr, nch * 8]
    lane = torch.arange(lpr)

    def reduce(t):
        s = torch.zeros(t.shape[0], lpr)
        for k in range(t.shape[2]):
            s = s + t[:, :, k]
        o = lpr // 2
        while o:
            s = s + s[:, lane ^ o]
            o //= 2
        return s[:, :1]
    mean = reduce(lanes) / C
    valid = (cols < C).view(1, lpr, -1)
    if mutation == "one_pass":
        q = reduce(lanes * lanes) / C - mean * mean
    else:
        dl = torch.where(valid, lanes - mean.view(-1, 1, 1), torch.zeros(()))
        q = torch.zeros(R * G, lpr)
        for k in range(dl.shape[2]):
            q = _fma32(dl[:, :, k], dl[:, :, k], q)
        o = lpr // 2
        while o:
            q = q + q[:, lane ^ o]
            o //= 2
        q = q[:, :1] / (C - 1 if mutation == "var_c_minus_1" else C)
    e32 = torch.tensor(eps, dtype=torch.float32)
    if mutation == "eps_outside":
        rstd = (1 / (torch.sqrt(q.double()) + e32.double())).float()
    else:
        rstd = (1 / torch.sqrt((q + e32).double())).float()
    idx = torch.arange(G) // gps
    if mutation == "gamma_set0":
        idx = torch.zeros_like(idx)
    g32 = gamma[idx].repeat(R, 1)
    b32 = beta[idx].repeat(R, 1)
    t = (v - mean) * rstd
    return _fma32(t, g32, b32).view(R, G, C)


def _ln_depth(row):
    name, entry, dt, rows, groups, gps, C, xrs, yrs, cnpos, inplace, kind, goff = row
    _, lpr, nch = ln_dispatch(C) if name == REG else (GEN, 32, -(-(-(-C // 8)) // 32))
    return lpr, nch, nch * 8 + int(math.log2(lpr))


@pytest.mark.gpu
@pytest.mark.parametrize("row", LN_ROWS, ids=_ids(LN_ROWS))
def test_layernorm_row(row):
    name, entry, dt, rows, groups, gps, C, xrs, yrs, cnpos, inplace, kind, goff = row
    x, cls, gamma, beta = ln_inputs(row)
    assert not inplace or xrs == yrs
    xb = _rows_buffer(x, xrs, TDT[dt]).to(_dev())
    yb = xb if inplace else _sentinel_cpu(rows * yrs + TAIL, TDT[dt]).to(_dev())
    gb = torch.zeros(goff + gamma.numel() + 8, device=_dev())
    bb = torch.zeros(goff + beta.numel() + 8, device=_dev())
    gb[goff:goff + gamma.numel()] = gamma.reshape(-1).to(_dev())
    bb[goff:goff + beta.numel()] = beta.reshape(-1).to(_dev())
    gp, bp = gb.data_ptr() + 4 * goff, bb.data_ptr() + 4 * goff
    if entry == "pv_layernorm":
        assert gps == groups and cls is None
        args = (xb.data_ptr(), yb.data_ptr(), _code(dt), rows, groups, C, xrs, yrs, gp, bp, LN_EPS, _stream())
    else:
        cd = cls.to(TDT[dt]).to(_dev()) if cls is not None else None
        esz = xb.element_size()
        args = (xb.data_ptr(), yb.data_ptr(), _code(dt), rows, groups, C, xrs, yrs, gp, bp, gps,
                cd.data_ptr() + groups * C * esz if cd is not None else None,
                cd.shape[1] * cd.shape[2] if cd is not None else 0, cnpos if cnpos else 1, LN_EPS, _stream())
    launched = _launch(entry, *args)
    _expect(name, launched)
    yc = yb.cpu()
    _assert_untouched(yc, _written(rows, yrs, groups * C), name)
    got = yc[:rows * yrs].view(rows, yrs)[:, :groups * C].reshape(rows, groups, C)
    _, _, depth = _ln_depth(row)
    ref, absref, K, extra = ln_ref64(_ln_eff(x, cls, row), gamma, beta, gps, depth)
    ratio = _assert_bound(got, ref, absref, K, acc_eps=SUM_EPS, what=name, extra64=extra, rnd_eps=_rnd(dt))
    _ratio("layernorm", row, ratio, launched)


# add_layernorm: s = a + b in fp32 (stored bit-exact), y = LayerNorm(s) stored f16 (the LayerNorm bound above with the
# row-in-registers depth).
ALN_ROWS = [
    # (launch, entry, a dtype, with b, rows, C, a / b / sum / y row strides, sum out, y out, input kind)
    ("add_layernorm_kernel", "pv_add_layernorm", adt, wb, rows, C, C, C, C, C, True, True, "randn")
    for adt in ("f32", "f16") for wb in (True, False) for rows, C in ((77, 96), (130, 192), (33, 384), (19, 768), (5, 8))
] + [
    ("add_layernorm_kernel", "pv_add_layernorm", "f32", True, 77, 96, 104, 112, 120, 128, True, True, "randn"),
    ("add_layernorm_kernel", "pv_add_layernorm", "f16", True, 37, 384, 392, 400, 384, 392, True, True, "randn"),
    ("add_layernorm_kernel", "pv_add_layernorm", "f32", True, 50, 768, 776, 768, 776, 768, False, True, "randn"),
    ("add_layernorm_kernel", "pv_add_layernorm", "f16", False, 50, 8, 16, 8, 24, 8, False, True, "randn"),
    ("add_layernorm_kernel", "pv_add_layernorm", "f32", True, 31, 192, 200, 192, 208, 192, True, False, "randn"),
    ("add_layernorm_kernel", "pv_add_layernorm", "f16", False, 31, 96, 96, 96, 104, 96, True, False, "randn"),
    ("add_layernorm_kernel", "pv_add_layernorm", "f32", False, 33, 384, 384, 384, 384, 384, True, True, "hard"),
]


def aln_inputs(row):
    name, entry, adt, wb, rows, C, ars, brs, srs, yrs, ws, wy, kind = row
    g = _gen(row)
    a = (1e3 + 1e-2 * torch.randn(rows, C, generator=g)) if kind == "hard" else torch.randn(rows, C, generator=g) * 3 + 1
    a = _f16(a) if adt == "f16" else a
    b = _f16(torch.randn(rows, C, generator=g) * 0.5) if wb else None
    gamma, beta = torch.rand(1, C, generator=g) + 0.5, torch.rand(1, C, generator=g) - 0.5
    return a, b, gamma, beta


def _aln_sum(a, b):
    return a.float() + b.float() if b is not None else a.float()


@pytest.mark.gpu
@pytest.mark.parametrize("row", ALN_ROWS, ids=_ids(ALN_ROWS))
def test_add_layernorm_row(row):
    name, entry, adt, wb, rows, C, ars, brs, srs, yrs, ws, wy, kind = row
    a, b, gamma, beta = aln_inputs(row)
    ad = _rows_buffer(a, ars, TDT[adt]).to(_dev())
    bd = _rows_buffer(b, brs, torch.float16).to(_dev()) if b is not None else None
    sd = _sentinel_cpu(rows * srs + TAIL, torch.float32).to(_dev()) if ws else None
    yd = _sentinel_cpu(rows * yrs + TAIL, torch.float16).to(_dev()) if wy else None
    gd, bed = gamma.reshape(-1).to(_dev()), beta.reshape(-1).to(_dev())
    launched = _launch(entry, ad.data_ptr(), _code(adt), ars, bd.data_ptr() if bd is not None else None, brs,
                       sd.data_ptr() if sd is not None else None, srs, yd.data_ptr() if yd is not None else None, yrs,
                       rows, C, gd.data_ptr(), bed.data_ptr(), LN_EPS, _stream())
    _expect(name, launched)
    s = _aln_sum(a, b)
    if ws:
        want = _rows_buffer(s, srs, torch.float32)
        _assert_bits(sd, want, name + " sum")
    if wy:
        yc = yd.cpu()
        _assert_untouched(yc, _written(rows, yrs, C), name)
        _, lpr, nch = ln_dispatch(C)
        ref, absref, K, extra = ln_ref64(s.view(rows, 1, C), gamma, beta, 1, nch * 8 + int(math.log2(lpr)))
        got = yc[:rows * yrs].view(rows, yrs)[:, :C].reshape(rows, 1, C)
        ratio = _assert_bound(got, ref, absref, K, acc_eps=SUM_EPS, what=name, extra64=extra)
        _ratio("add-layernorm", row, ratio, launched)
    else:
        _exact("add-layernorm-sum", row, launched)


# =====================================================================================================================
# temporal_tap_sum (factored Fast stem) and add_pos_cls
# =====================================================================================================================
# temporal_tap_sum: the in-range taps summed in fp32 (<= kt - 1 roundings), then act(acc * scale + bias) (<= 2
# roundings): absref = L (|scale| sum|taps| + |bias|), K = kt + 2, plus act_err64 and the storage rounding.
TAP_ROWS = [
    # (launch, entry, dtype, N, Ti, hw, Co, kt, st, pt, dil, act, in row stride - kt Co, out row stride - Co)
    ("temporal_tap_sum_kernel", "pv_temporal_tap_sum", "f16", 2, 8, 12, 16, 3, 1, 1, 1, "relu", 8, 8),
    ("temporal_tap_sum_kernel", "pv_temporal_tap_sum", "f32", 1, 9, 10, 8, 5, 2, 2, 1, "none", 0, 16),
    ("temporal_tap_sum_kernel", "pv_temporal_tap_sum", "f16", 1, 10, 9, 24, 5, 1, 4, 2, "swish", 16, 8),
    ("temporal_tap_sum_kernel", "pv_temporal_tap_sum", "f32", 2, 7, 6, 8, 3, 2, 2, 2, "swish", 8, 8),
    ("temporal_tap_sum_kernel", "pv_temporal_tap_sum", "f16", 1, 6, 5, 8, 5, 1, 3, 1, "none", 0, 8),
    ("temporal_tap_sum_kernel", "pv_temporal_tap_sum", "f32", 1, 16, 20, 16, 3, 2, 1, 1, "relu", 0, 0),
    ("temporal_tap_sum_kernel", "pv_temporal_tap_sum", "f16", 2, 5, 7, 32, 5, 2, 2, 2, "relu", 0, 32),
]


def tap_geometry(row):
    name, entry, dt, N, Ti, hw, Co, kt, st, pt, dil, act, irx, orx = row
    return (Ti + 2 * pt - dil * (kt - 1) - 1) // st + 1, kt * Co + irx, Co + orx


def tap_inputs(row):
    name, entry, dt, N, Ti, hw, Co, kt, st, pt, dil, act, irx, orx = row
    g = _gen(row)
    yk = torch.randn(N, Ti, hw, kt, Co, generator=g)
    yk = _f16(yk) if dt == "f16" else yk
    return yk, torch.rand(Co, generator=g) + 0.5, torch.rand(Co, generator=g) - 0.5


def _taps(Ti, To, kt, st, pt, dil, clamp=False):
    """[(t, dt, ti)] of the in-range taps (clamp: out-of-range frames clamped into the clip instead)."""
    out = []
    for t in range(To):
        for d in range(kt):
            ti = t * st + d * dil - pt
            if 0 <= ti < Ti:
                out.append((t, d, ti))
            elif clamp:
                out.append((t, d, min(max(ti, 0), Ti - 1)))
    return out


def tap_ref64(inp, row):
    name, entry, dt, N, Ti, hw, Co, kt, st, pt, dil, act, irx, orx = row
    yk, scale, bias = inp
    To, _, _ = tap_geometry(row)
    acc = torch.zeros(N, To, hw, Co, dtype=torch.float64)
    aab = torch.zeros(N, To, hw, Co, dtype=torch.float64)
    for t, d, ti in _taps(Ti, To, kt, st, pt, dil):
        acc[:, t] += yk[:, ti, :, d].double()
        aab[:, t] += yk[:, ti, :, d].double().abs()
    pre = acc * scale.double() + bias.double()
    absref = LIP[act] * (aab * scale.double().abs() + bias.double().abs())
    return act64(pre, act), absref, kt + 2, act_err64(pre, act)


def tap_emulate(inp, row, mutation=None):
    """mutation "clamp_frames": out-of-range frames clamped into the clip instead of skipped."""
    name, entry, dt, N, Ti, hw, Co, kt, st, pt, dil, act, irx, orx = row
    yk, scale, bias = inp
    To, _, _ = tap_geometry(row)
    acc = torch.zeros(N, To, hw, Co)
    for t, d, ti in _taps(Ti, To, kt, st, pt, dil, clamp=mutation == "clamp_frames"):
        acc[:, t] = acc[:, t] + yk[:, ti, :, d].float()
    return act32(_fma32(acc, scale, bias), act)


@pytest.mark.gpu
@pytest.mark.parametrize("row", TAP_ROWS, ids=_ids(TAP_ROWS))
def test_temporal_tap_sum_row(row):
    name, entry, dt, N, Ti, hw, Co, kt, st, pt, dil, act, irx, orx = row
    inp = tap_inputs(row)
    yk, scale, bias = inp
    To, irs, ors = tap_geometry(row)
    xb = _rows_buffer(yk.reshape(N * Ti * hw, kt * Co), irs, TDT[dt], fill=BIG).to(_dev())
    R = N * To * hw
    yb = _sentinel_cpu(R * ors + TAIL, TDT[dt]).to(_dev())         # the concat slice: channels [Co, ors) untouched
    sd, bd = scale.to(_dev()), bias.to(_dev())
    launched = _launch(entry, xb.data_ptr(), yb.data_ptr(), _code(dt), N, Ti, To, hw, Co, kt, st, pt, dil,
                       sd.data_ptr(), bd.data_ptr(), _act_code(act), irs, ors, _stream())
    _expect(name, launched)
    yc = yb.cpu()
    _assert_untouched(yc, _written(R, ors, Co), name)
    got = yc[:R * ors].view(R, ors)[:, :Co].reshape(N, To, hw, Co)
    ref, absref, K, extra = tap_ref64(inp, row)
    ratio = _assert_bound(got, ref, absref, K, acc_eps=SUM_EPS, what=name, extra64=extra, rnd_eps=_rnd(dt))
    _ratio("temporal-tap-sum", row, ratio, launched)


POS_ROWS = [
    # (launch, entry, x dtype, y dtype, B, n_patch, C, x row stride, has_cls)
    ("add_pos_cls_kernel", "pv_add_pos_cls", "f16", "f16", 2, 49, 96, 104, 1),
    ("add_pos_cls_kernel", "pv_add_pos_cls", "f16", "f16", 3, 33, 40, 40, 0),
    ("add_pos_cls_kernel", "pv_add_pos_cls", "f32", "f32", 2, 33, 40, 48, 0),
    ("add_pos_cls_kernel", "pv_add_pos_cls", "f32", "f32", 3, 50, 16, 16, 1),
    ("add_pos_cls_kernel", "pv_add_pos_cls_to", "f16", "f32", 3, 49, 96, 96, 1),
    ("add_pos_cls_kernel", "pv_add_pos_cls_to", "f16", "f32", 2, 50, 16, 24, 0),
    ("add_pos_cls_kernel", "pv_add_pos_cls_to", "f32", "f32", 2, 17, 24, 32, 1),
    ("add_pos_cls_kernel", "pv_add_pos_cls_to", "f16", "f16", 2, 17, 24, 32, 1),
]


def pos_inputs(row):
    name, entry, xdt, ydt, B, n, C, xrs, hc = row
    g = _gen(row)
    x = _src_values(g, (B * n, C), xdt)
    x = torch.where(x.float().abs() > 1e5, torch.zeros((), dtype=x.dtype), x)    # keep the f32 rows finite
    pos = torch.randn(hc + n, C, generator=g)
    return x, pos


def pos_emulate(x, pos, row, mutation=None):
    """fp32 x + pos, one cast to the output type.  mutation "pos_prev_row": patch row i adds pos row i - 1."""
    name, entry, xdt, ydt, B, n, C, xrs, hc = row
    out = torch.empty(B, hc + n, C)
    if hc:
        out[:, 0] = pos[0]
    prow = torch.arange(hc, hc + n) - (1 if mutation == "pos_prev_row" else 0)
    out[:, hc:] = x.float().view(B, n, C) + pos[prow.clamp_min(0)]
    return out.reshape(-1, C).to(TDT[ydt])


@pytest.mark.gpu
@pytest.mark.parametrize("row", POS_ROWS, ids=_ids(POS_ROWS))
def test_add_pos_cls_row(row):
    name, entry, xdt, ydt, B, n, C, xrs, hc = row
    x, pos = pos_inputs(row)
    xb = _rows_buffer(x, xrs, TDT[xdt], fill=BIG).to(_dev())
    R = B * (hc + n)
    yb = _sentinel_cpu(R * C + TAIL, TDT[ydt]).to(_dev())
    pd = pos.to(_dev())
    if entry == "pv_add_pos_cls":
        assert xdt == ydt
        args = (xb.data_ptr(), yb.data_ptr(), _code(xdt), B, n, C, xrs, pd.data_ptr(), hc, _stream())
    else:
        args = (xb.data_ptr(), _code(xdt), yb.data_ptr(), _code(ydt), B, n, C, xrs, pd.data_ptr(), hc, _stream())
    launched = _launch(entry, *args)
    _expect(name, launched)
    want = _sentinel_cpu(R * C + TAIL, TDT[ydt])
    want[:R * C] = pos_emulate(x, pos, row).reshape(-1)
    _assert_bits(yb, want, name)
    _exact("add-pos-cls", row, launched)


def ln_dispatch(C, aligned=True):
    """(launch, lanes per row, chunks per lane) pv_layernorm_sets picks."""
    return TS.ln_dispatch(C, aligned)


def ln_ref64(v, gamma, beta, gps, depth, eps=LN_EPS):
    return TS.ln_ref64(v, gamma, beta, gps, depth, eps)


# =====================================================================================================================
# CPU: the emulations pass their bounds, known bugs do not
# =====================================================================================================================
def _bounded_case(family, row, mutation=None):
    """(emulated result rounded to its storage type, ref, absref, K, acc_eps, extra, rnd_eps) of a row."""
    if family == "pool":
        x = pool_inputs(row)
        ref, absref, K = pool_ref64(x, row)
        got = avg_pool_emulate(x, row, mutation).to(TDT[row[2]])
        return got, ref, absref, K, SUM_EPS, None, _rnd(row[2])
    if family == "channel_sum":
        x = cs_inputs(row)
        ref, absref, K, extra = cs_ref64(x, row)
        return cs_emulate(x, row, mutation).double() * 2.0 ** -24, ref, absref, K, SUM_EPS, extra, TS.F32_EPS
    if family == "se_gate":
        inp = se_gate_inputs(row)
        ref, absref, K, extra = se_gate_ref64(inp, row)
        return se_gate_emulate(inp, row, mutation), ref, absref, K, SUM_EPS, extra, TS.F32_EPS
    if family == "scale_act":
        inp = scale_act_inputs(row)
        ref, absref, extra = scale_act_ref64(inp, row)
        return scale_act_emulate(inp, row, mutation).to(TDT[row[2]]), ref, absref, 0, U, extra, _rnd(row[2])
    if family == "head":
        x = head_inputs(row)
        ref, absref, K, extra = head_ref64(x, row)
        return head_emulate(x, row, mutation), ref, absref, K, SUM_EPS, extra, TS.F32_EPS
    if family == "layernorm":
        x, cls, gamma, beta = ln_inputs(row)
        if mutation == "cls_sample0":
            cls = cls.clone()
            cls[1:, 0] = cls[0, 0]
        lpr, nch, depth = _ln_depth(row)
        ref, absref, K, extra = ln_ref64(_ln_eff(*ln_inputs(row)[:2], row), gamma, beta, row[5], depth)
        got = ln_emulate(_ln_eff(x, cls, row), gamma, beta, row[5], lpr, nch,
                         mutation=None if mutation == "cls_sample0" else mutation)
        return got.to(TDT[row[2]]), ref, absref, K, SUM_EPS, extra, _rnd(row[2])
    if family == "add_layernorm":
        a, b, gamma, beta = aln_inputs(row)
        rows, C = row[4], row[5]
        _, lpr, nch = ln_dispatch(C)
        s = _aln_sum(a, b).view(rows, 1, C)
        ref, absref, K, extra = ln_ref64(s, gamma, beta, 1, nch * 8 + int(math.log2(lpr)))
        got = ln_emulate(s, gamma, beta, 1, lpr, nch, mutation=mutation).half()
        return got, ref, absref, K, SUM_EPS, extra, TS.F16_EPS
    if family == "tap":
        inp = tap_inputs(row)
        ref, absref, K, extra = tap_ref64(inp, row)
        return tap_emulate(inp, row, mutation).to(TDT[row[2]]), ref, absref, K, SUM_EPS, extra, _rnd(row[2])
    raise KeyError(family)


def _check(family, row, mutation=None):
    got, ref, absref, K, acc_eps, extra, rnd = _bounded_case(family, row, mutation)
    return _assert_bound(got, ref.reshape(got.shape), absref.reshape(got.shape), K, acc_eps=acc_eps,
                                  what="%s %s" % (family, mutation), rnd_eps=rnd,
                                  extra64=None if extra is None else extra.reshape(got.shape))


BOUNDED_CASES = ([("pool", r) for r in POOL_ROWS if r[3] == "avg"] + [("channel_sum", r) for r in CS_ROWS] +
                 [("se_gate", r) for r in SE_GATE_ROWS] + [("scale_act", r) for r in SCALE_ACT_ROWS] +
                 [("head", r) for r in HEAD_ROWS] + [("layernorm", r) for r in LN_ROWS] +
                 [("add_layernorm", r) for r in ALN_ROWS if r[11]] + [("tap", r) for r in TAP_ROWS])


@pytest.mark.parametrize("family,row", BOUNDED_CASES, ids=["%s-%s" % (f, _rid(r)) for f, r in BOUNDED_CASES])
def test_emulation_passes_its_bound(family, row):
    ratio = _check(family, row)
    print("RATIO emulation-%s %s %.4f %.4f" % (family, _rid(row), *ratio))


def _row(rows, pred):
    return next(r for r in rows if pred(r))


MUTATIONS = {
    "avg_pool_valid_count": ("pool", _row(POOL_ROWS, lambda r: r[3] == "avg" and r[9] == (1, 1, 1)), "valid_count"),
    "layernorm_one_pass": ("layernorm", _row(LN_ROWS, lambda r: r[11] == "hard" and r[6] == 768), "one_pass"),
    "layernorm_var_c_minus_1": ("layernorm", _row(LN_ROWS, lambda r: r[6] == 768 and r[11] == "randn"),
                                "var_c_minus_1"),
    "layernorm_eps_outside": ("layernorm", _row(LN_ROWS, lambda r: r[11] == "tiny" and r[2] == "f32"), "eps_outside"),
    "layernorm_gamma_wrong_set": ("layernorm", _row(LN_ROWS, lambda r: r[4] // r[5] > 1), "gamma_set0"),
    "layernorm_cls_from_sample0": ("layernorm", _row(LN_ROWS, lambda r: r[9] and r[3] // r[9] > 1), "cls_sample0"),
    "add_layernorm_one_pass": ("add_layernorm", _row(ALN_ROWS, lambda r: r[12] == "hard"), "one_pass"),
    "softmax_without_max": ("head", _row(HEAD_ROWS, lambda r: r[8] == "peak60"), "no_max"),
    "head_mean_over_c": ("head", _row(HEAD_ROWS, lambda r: r[4] == 392 and r[7] == 1), "mean_over_c"),
    "channel_sum_drops_last_chunk": ("channel_sum", _row(CS_ROWS, lambda r: r[4] == 5000), "drop_last_chunk"),
    "se_gate_w1_stride_c": ("se_gate", SE_GATE_ROWS[0], "w1_stride_c"),
    "tap_sum_clamps_frames": ("tap", _row(TAP_ROWS, lambda r: r[9] > 1), "clamp_frames"),
}


@pytest.mark.parametrize("name", sorted(MUTATIONS))
def test_comparator_rejects_simt_bugs(name):
    family, row, mutation = MUTATIONS[name]
    with pytest.raises(AssertionError):
        _check(family, row, mutation)


@pytest.mark.parametrize("row", [r for r in POOL_ROWS if r[3] == "max" and r[13] == "neg" and any(r[9])],
                         ids=_ids([r for r in POOL_ROWS if r[3] == "max" and r[13] == "neg" and any(r[9])]))
def test_bit_exact_check_rejects_max_pool_padding_as_zero(row):
    x = pool_inputs(row)
    good, bad = max_pool_emulate(x, row), max_pool_emulate(x, row, "pad_zero")
    ref = pool_ref64(x, row)[0].float()
    assert torch.equal(_bits(good), _bits(ref))
    assert not torch.equal(_bits(bad), _bits(ref))


@pytest.mark.parametrize("row", POS_ROWS, ids=_ids(POS_ROWS))
def test_bit_exact_check_rejects_pos_row_shift(row):
    x, pos = pos_inputs(row)
    assert not torch.equal(_bits(pos_emulate(x, pos, row)), _bits(pos_emulate(x, pos, row, "pos_prev_row")))


def test_f16_specials_round_to_nearest_even():
    """The f32 -> f16 reference the layout rows compare with: ties to even, subnormals, overflow to inf."""
    v = torch.tensor(F32_SPECIALS[:13], dtype=torch.float32).half().float().tolist()
    assert v[:5] == [1.0, 1 + 2.0 ** -9, -1.0, 2048.0, 2052.0]
    assert v[5:8] == [0.0, 2.0 ** -23, 2.0 ** -23]
    assert v[10:13] == [65504.0, 65504.0, math.inf]


# =====================================================================================================================
# CPU: routing and the launch-name ledger
# =====================================================================================================================
def test_rows_reach_every_layernorm_route():
    pairs = set()
    for r in LN_ROWS:
        name, C, goff = r[0], r[6], r[12]
        assert ln_dispatch(C, aligned=goff * 4 % 16 == 0)[0] == name, r
        if name == REG:
            pairs.add(ln_dispatch(C)[1:])
    reachable = {ln_dispatch(C)[1:] for C in range(8, 769, 8)}
    assert pairs == reachable == {(4, 1), (8, 1), (16, 1), (32, 1), (32, 2), (32, 3)}
    assert {r[6] for r in LN_ROWS if r[0] == GEN and r[12]} and {r[6] for r in LN_ROWS if r[0] == GEN and r[6] > 768}


def test_rows_reach_every_padw_route():
    for r in PADW_ROWS:
        name, _, sdt, ddt, N, C, T, H, W, c_pad, w_pad, w_phys, off = r
        assert (name == QUAD) == quad_route(sdt, ddt, C, c_pad, W, w_pad, w_phys, off), r
    assert {r[5] for r in PADW_ROWS if r[0] == QUAD} == {1, 2, 3, 4}
    assert {r[10] for r in PADW_ROWS if r[0] == QUAD} == {0, 4, 8}


def test_rows_reach_every_pool_route():
    for r in POOL_ROWS:
        assert pool_route(r[6], r[7], r[9], r[12]) == r[0], r
    whole = [r for r in POOL_ROWS if _pool_out(r[6], r[7], r[8], r[9]) == (1, 1, 1) and r[0] == POOL3D]
    assert any(r[12] for r in whole) and any(any(r[9]) for r in whole)


def test_channel_sum_rows_reach_both_branches_and_the_chunk_cap():
    geo = [cs_geometry(r[4], r[5]) for r in CS_ROWS]
    assert any(r[5] > 2048 for r in CS_ROWS) and any(r[5] <= 2048 and 256 % (r[5] // 8) for r in CS_ROWS)
    assert any(g[0] > 1 for g in geo)
    assert any(r[4] > 2048 * 1024 and g[0] == 1024 for r, g in zip(CS_ROWS, geo))


TABLES = {"NCDHW_ROWS": NCDHW_ROWS, "PADW_ROWS": PADW_ROWS, "TO_NCDHW_ROWS": TO_NCDHW_ROWS, "COPY_ROWS": COPY_ROWS,
          "POOL_ROWS": POOL_ROWS, "CS_ROWS": CS_ROWS, "SE_GATE_ROWS": SE_GATE_ROWS, "SCALE_ACT_ROWS": SCALE_ACT_ROWS,
          "HEAD_ROWS": HEAD_ROWS, "LN_ROWS": LN_ROWS, "ALN_ROWS": ALN_ROWS, "TAP_ROWS": TAP_ROWS,
          "POS_ROWS": POS_ROWS}
# launch names of pv_simt.cu whose rows live in another file (a family of PV_PRE_NAME instances is named "base…>")
COVERED_ELSEWHERE = {
    "conv3d_direct_kernel<__half>": "test_gpu_kernel_matrix.py",
    "conv3d_direct_kernel<float>": "test_gpu_grouped.py",
    "dwconv3d_kernel<…>": "test_gpu_kernel_matrix.py",
    "dwconv3d_w4_kernel<…>": "test_gpu_kernel_matrix.py",
}
# entry points of pv_simt.cu no row calls
ENTRY_NOT_CALLED = {"pv_zero_f32": "a cudaMemsetAsync of the SE sum buffer: it launches no kernel"}


def simt_source():
    return open(os.path.join(CSRC, "pv_simt.cu")).read()


def launch_names(src):
    names = set(re.findall(r'PV_LAUNCH_OK\("([^"]+)"\)', src))
    names |= {base + "…>" for base in re.findall(r'PV_PRE_NAME\("([^"]+<)"', src)}
    return names


def ledger_problems(src, tables):
    rows = [r for t in tables.values() for r in t]
    expected = {r[0] for r in rows}
    called = {r[1] for r in rows}
    names = launch_names(src)
    out = ["launch name %s: no row expects it and it is not covered elsewhere" % n
           for n in sorted(names - expected - set(COVERED_ELSEWHERE))]
    out += ["rows expect %s, which no launch site of pv_simt.cu names" % n for n in sorted(expected - names)]
    out += ["%s is listed as covered elsewhere but is no launch name" % n for n in sorted(set(COVERED_ELSEWHERE) - names)]
    for n, f in sorted(COVERED_ELSEWHERE.items()):
        if n.rstrip("…>") not in open(os.path.join(TESTS, f)).read():
            out.append("%s does not mention %s" % (f, n))
    entries = set(re.findall(r'extern "C" int (pv_\w+)\(', src))
    out += ["entry point %s: no row calls it" % e for e in sorted(entries - called - set(ENTRY_NOT_CALLED))]
    out += ["rows call %s, which pv_simt.cu does not define" % e for e in sorted(called - entries)]
    return out


def test_ledger_covers_every_launch_site_and_entry_point():
    src = simt_source()
    assert len(launch_names(src)) == 20
    assert not ledger_problems(src, TABLES), ledger_problems(src, TABLES)


def test_ledger_fails_on_a_new_launch_site_or_a_lost_row():
    src = simt_source()
    assert ledger_problems(src + '\nvoid f() { PV_LAUNCH_OK("new_kernel"); }\n', TABLES)
    assert ledger_problems(src + '\nextern "C" int pv_new_entry(void* stream) { return 0; }\n', TABLES)
    for key in TABLES:
        name = TABLES[key][0][0]
        fewer = {k: [r for r in t if r[0] != name] for k, t in TABLES.items()}
        assert ledger_problems(src, fewer), name
