"""Kernel-instance matrix: every compiled instance of the hot kernels against a float64 reference.

Each row of a table names a shape and the kernel instance the library is expected to launch for it; the test runs
the op, compares with the same operation in float64 on the f16-grid operands (testing.assert_close_to_f64) and asserts
from the library's per-instance launch counts that the expected instance ran.  CPU tests below check the comparator
(it must reject known kernel bugs), the instance ledger (every compiled instance is some row's expected instance or
is listed as unreachable) and the attention routing (pv_attention_kernel_for).

Measured on an NVIDIA H100 80GB HBM3 (132 SMs, 400 W power limit), per kernel family: the largest err / tol, and in
brackets the largest share of the accumulation term a result used beyond its own f16 rounding (the margin of the
accumulation constant; a correctly rounded f16 result may use nearly all of the rounding term):
  igemm 0.992 (0.017), window-mode igemm 0.920 (0.011), gather 0.989 (0.011), stem rows incl. the factored temporal
  stem 0.990 (0.133), depthwise 0.995 (0.020), attention wgmma 0.196 (0.097), attention mma 0.180 (0.092),
  attention CUDA-core f16 0.142.
The f32 rows are held to fp32 bounds: the fp32 rounding term, and for attention_kernel<float, D> the fp32 attention
bound (testing.ACC_EPS_ATTN_F32 over Nk, testing.attn_score_extra64).  Measured on an NVIDIA H100 80GB HBM3 (700 W
power limit): attention CUDA-core f32 0.0087 (0.033), depthwise f32 0.133 (0.099), conv3d_direct_kernel<float>
(DIRECT_F32_ROWS) 0.097 (0.084).

The fused bottleneck block keeps its intermediates a and b in f16, so its bound also carries their rounding error
propagated to y (fused_block_ref64).  Measured on an NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit) over every
FUSED_ROWS and poison row: largest err / tol 0.583, largest share of the propagated term used 0.310 (charging all
error beyond y's own rounding to it).  The accumulation share is not meaningful there: the f16 intermediates, not
the fp32 sums, make up nearly all of the error.
"""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.testing import ACC_EPS_ATTN, attn_ref64, conv_ref64, fused_block_ref64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorchvideo_b200", "csrc")

def _dev():
    return torch.device("cuda:0")


def _bn(c, seed):
    g = torch.Generator().manual_seed(seed)
    bn = torch.nn.BatchNorm3d(c).eval()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.rand(c, generator=g) - 0.5)
        bn.running_mean.copy_(torch.rand(c, generator=g) - 0.5)
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn


# ---- convolution rows --------------------------------------------------------------------------------------------
# (expected instance, N, Ci, T, H, W, Co, kernel, stride, padding, dilation, act, residual, depthwise se_sums)
# Block N of the TMA-fed kernel comes from a cost model over the SM count (pv_igemm.cu): C_out <= 16 / 32 / 64 gives
# 16 / 32 / 64; wider outputs take 64 when there are only a few dozen 128-row tiles and 128 from about a hundred on.
# Shapes sit far from that boundary so 132-SM (SXM) and 114-SM (PCIe) parts choose the same instance.  k-block bytes:
# C_in = 16 -> 32, C_in = 32 -> 64 (narrow TMA, one tap per k-block), C_in >= 64 -> 128.
IGEMM_ROWS = [
    # C_in 16: a stage holds 4 taps; 9, 7 and 27 taps leave the last stage short (zero-filled boxes)
    ("conv3d_igemm_kernel<16,32>", 1, 16, 4, 9, 9, 16, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), "relu", True),
    ("conv3d_igemm_kernel<32,32>", 2, 16, 9, 6, 6, 24, (7, 1, 1), (1, 1, 1), (3, 0, 0), (1, 1, 1), "swish", False),
    ("conv3d_igemm_kernel<64,32>", 1, 16, 7, 11, 11, 40, (3, 3, 3), (2, 2, 2), (1, 1, 1), (1, 1, 1), "gelu", False),
    ("conv3d_igemm_kernel<128,32>", 2, 16, 8, 40, 40, 200, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), "sigmoid", True),
    # C_in 32: a stage holds 2 taps; odd tap counts leave the last stage short
    ("conv3d_igemm_kernel<16,64>", 2, 32, 6, 10, 10, 8, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1), "relu", False),
    ("conv3d_igemm_kernel<32,64>", 1, 32, 7, 8, 8, 32, (5, 1, 1), (1, 1, 1), (2, 0, 0), (1, 1, 1), None, False),
    ("conv3d_igemm_kernel<64,64>", 2, 32, 3, 15, 15, 56, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), "swish", True),
    ("conv3d_igemm_kernel<128,64>", 2, 32, 8, 36, 36, 432, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), "gelu", True),
    # C_in >= 64 (80 and 216 are padded to 128 / 256 in the packed weights)
    ("conv3d_igemm_kernel<16,128>", 1, 80, 4, 12, 12, 16, (3, 3, 3), (1, 1, 1), (1, 2, 2), (1, 2, 2), "relu", False),
    ("conv3d_igemm_kernel<32,128>", 2, 64, 4, 9, 9, 24, (1, 1, 1), (2, 2, 2), (0, 0, 0), (1, 1, 1), None, True),
    ("conv3d_igemm_kernel<64,128>", 1, 216, 2, 14, 14, 200, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), "sigmoid", True),
    ("conv3d_igemm_kernel<128,128>", 4, 128, 8, 28, 28, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), "relu", True),
    # 63 taps (IG_MAX_TAPS = 64), several N tiles of a C_out that is not a multiple of 64, dilation as in res5
    ("conv3d_igemm_kernel<64,128>", 1, 64, 3, 9, 11, 64, (1, 7, 9), (1, 1, 1), (0, 3, 4), (1, 1, 1), None, False),
    ("conv3d_igemm_kernel<64,128>", 1, 64, 2, 14, 14, 432, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), "relu", False),
    ("conv3d_igemm_kernel<64,128>", 1, 128, 2, 7, 7, 128, (1, 3, 3), (1, 1, 1), (0, 2, 2), (1, 2, 2), "relu", True),
]

GATHER_ROWS = [
    # C_in < 64 other than 16 / 32: cp.async gather.  Block N halves from 128 to 64 only below ~2 waves of tiles.
    ("conv3d_igemm_gather_kernel<16>", 2, 8, 4, 12, 12, 16, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), "relu", True),
    ("conv3d_igemm_gather_kernel<32>", 1, 3, 4, 12, 12, 24, (3, 3, 3), (1, 1, 1), (1, 1, 1), (1, 1, 1), "relu", False),
    ("conv3d_igemm_gather_kernel<64>", 1, 40, 6, 11, 11, 48, (3, 3, 3), (2, 2, 2), (1, 1, 1), (1, 1, 1), "swish", True),
    ("conv3d_igemm_gather_kernel<128>", 2, 8, 4, 72, 72, 96, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), None, False),
    ("conv3d_igemm_gather_kernel<64>", 1, 24, 5, 10, 10, 56, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1), "gelu", True),
    ("conv3d_igemm_gather_kernel<64>", 2, 48, 3, 14, 14, 48, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), "relu", True),
    ("conv3d_igemm_gather_kernel<64>", 1, 56, 3, 9, 9, 56, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), "sigmoid", True),
]

# stem rows: 3-channel input (padded to 4), stride 2 along W; window 16 / 32 / 64 elements for kw = 3 / 7 / >= 9
STEM_ROWS = [
    ("conv3d_stem_rows_kernel<16,1>", 2, 3, 2, 20, 20, 16, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), "relu", False),
    ("conv3d_stem_rows_kernel<32,1>", 1, 3, 1, 12, 312, 24, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), None, False),
    ("conv3d_stem_rows_kernel<64,1>", 1, 3, 2, 18, 30, 48, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), "relu", False),
    ("conv3d_stem_rows_kernel<128,1>", 1, 3, 6, 16, 16, 96, (3, 3, 3), (2, 2, 2), (1, 1, 1), (1, 1, 1), "relu", False),
    ("conv3d_stem_rows_kernel<16,2>", 1, 3, 2, 22, 22, 8, (1, 7, 7), (1, 2, 2), (0, 3, 3), (1, 1, 1), "relu", False),
    ("conv3d_stem_rows_kernel<32,2>", 1, 3, 2, 22, 22, 32, (1, 7, 7), (1, 2, 2), (0, 3, 3), (1, 1, 1), None, False),
    ("conv3d_stem_rows_kernel<64,2>", 1, 3, 2, 32, 32, 64, (1, 7, 7), (1, 2, 2), (0, 3, 3), (1, 1, 1), "relu", False),
    ("conv3d_stem_rows_kernel<128,2>", 1, 3, 1, 20, 280, 128, (1, 7, 7), (1, 2, 2), (0, 3, 3), (1, 1, 1), "relu", False),
    ("conv3d_stem_rows_kernel<16,4>", 1, 3, 2, 20, 20, 16, (1, 9, 9), (1, 2, 2), (0, 4, 4), (1, 1, 1), "relu", False),
    ("conv3d_stem_rows_kernel<32,4>", 1, 3, 2, 20, 20, 32, (1, 9, 9), (1, 2, 2), (0, 4, 4), (1, 1, 1), None, False),
    ("conv3d_stem_rows_kernel<64,4>", 1, 3, 2, 20, 20, 64, (1, 9, 9), (1, 2, 2), (0, 4, 4), (1, 1, 1), "relu", False),
    ("conv3d_stem_rows_kernel<128,4>", 1, 3, 2, 14, 20, 128, (1, 5, 9), (1, 2, 2), (0, 2, 4), (1, 1, 1), "relu", False),
    # factored temporal stem (SlowFast Fast stem): (1,7,7) with kt * Co channels on stem rows + pv_temporal_tap_sum
    ("temporal_tap_sum_kernel", 1, 3, 6, 18, 18, 8, (5, 7, 7), (1, 2, 2), (2, 3, 3), (1, 1, 1), "relu", False),
]

WINDOW_ROWS = [
    # I3D's (5,7,7) stem: 5*7 filter rows of 64 channels exceed the stem-rows weight budget -> window-mode igemm
    ("conv3d_igemm_kernel<64,64>", 1, 3, 6, 20, 20, 64, (5, 7, 7), (1, 2, 2), (2, 3, 3), (1, 1, 1), "relu", False),
    # MViT patch embedding: stride 4 along W (stem rows need stride 2)
    ("conv3d_igemm_kernel<64,64>", 1, 3, 8, 32, 32, 96, (3, 7, 7), (2, 4, 4), (1, 3, 3), (1, 1, 1), None, False),
]

# depthwise: (expected instance, N, C, T, H, W, kernel, stride, padding, dtype, se_sums)
DW_ROWS = [
    # lane-per-channel-pair 3x3x3 kernel: 4x4 patches, or 2x7 on planes a multiple of 7 wide (template arguments
    # <stride, patch h, patch w>)
    ("dwconv3d_lane_kernel<1,4,4>", 2, 56, 4, 20, 20, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f16", True),
    ("dwconv3d_lane_kernel<1,2,7>", 1, 216, 4, 14, 14, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f16", False),
    ("dwconv3d_lane_kernel<1,2,7>", 1, 48, 3, 7, 7, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f16", True),
    ("dwconv3d_lane_kernel<2,4,4>", 2, 56, 5, 21, 19, (3, 3, 3), (1, 2, 2), (1, 1, 1), "f16", True),
    ("dwconv3d_lane_kernel<2,2,7>", 1, 216, 3, 28, 28, (3, 3, 3), (1, 2, 2), (1, 1, 1), "f16", False),
    ("dwconv3d_lane_kernel<2,2,7>", 1, 48, 3, 14, 14, (3, 3, 3), (1, 2, 2), (1, 1, 1), "f16", True),
    ("dwconv3d_lane_kernel<2,4,4>", 1, 64, 6, 15, 15, (3, 3, 3), (2, 2, 2), (1, 1, 1), "f16", True),
    ("dwconv3d_lane_kernel<1,4,4>", 1, 24, 1, 8, 8, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f16", False),
    # streaming temporal kernel (no SE sums): prefetch ring longer than the clip, T = 1, the X3D stem conv_t
    ("dwconv_temporal_kernel<3>", 1, 40, 5, 9, 9, (3, 1, 1), (1, 1, 1), (1, 0, 0), "f16", False),
    ("dwconv_temporal_kernel<5>", 1, 16, 1, 6, 6, (5, 1, 1), (1, 1, 1), (2, 0, 0), "f16", False),
    ("dwconv_temporal_kernel<5>", 2, 24, 16, 28, 28, (5, 1, 1), (1, 1, 1), (2, 0, 0), "f16", False),
    ("dwconv_temporal_kernel<5>", 1, 24, 3, 10, 10, (5, 1, 1), (1, 1, 1), (2, 0, 0), "f16", False),
    # TMA tile kernel: everything else with kw in {1, 3}, with and without SE sums
    ("dwconv3d_tile_kernel<3,1>", 1, 128, 2, 7, 7, (1, 3, 3), (1, 1, 1), (0, 1, 1), "f16", True),
    ("dwconv3d_tile_kernel<3,1>", 1, 96, 3, 9, 9, (1, 3, 3), (1, 1, 1), (0, 1, 1), "f16", False),
    ("dwconv3d_tile_kernel<3,2>", 1, 96, 4, 14, 14, (1, 3, 3), (1, 2, 2), (0, 1, 1), "f16", True),
    ("dwconv3d_tile_kernel<3,2>", 1, 64, 3, 12, 12, (3, 3, 3), (1, 1, 2), (1, 1, 1), "f16", False),
    ("dwconv3d_tile_kernel<1,1>", 2, 24, 8, 12, 12, (5, 1, 1), (1, 1, 1), (2, 0, 0), "f16", True),
    ("dwconv3d_tile_kernel<1,1>", 1, 40, 5, 9, 9, (3, 1, 1), (1, 1, 1), (1, 0, 0), "f16", True),
    ("dwconv3d_tile_kernel<1,1>", 1, 40, 8, 9, 9, (3, 1, 1), (2, 1, 1), (1, 0, 0), "f16", False),   # st 2: not temporal
    ("dwconv3d_tile_kernel<1,2>", 1, 32, 4, 10, 10, (3, 1, 1), (1, 2, 2), (1, 0, 0), "f16", True),
    ("dwconv3d_tile_kernel<1,2>", 1, 48, 4, 10, 10, (3, 1, 1), (1, 2, 2), (1, 0, 0), "f16", False),
    # generic CUDA-core stencil: f16 shapes no TMA kernel takes (kw = 5), and f32
    ("dwconv3d_kernel<__half>", 1, 32, 3, 10, 10, (1, 5, 5), (1, 1, 1), (0, 2, 2), "f16", True),
    ("dwconv3d_kernel<__half>", 1, 16, 3, 10, 10, (1, 5, 5), (1, 2, 2), (0, 2, 2), "f16", False),
    ("dwconv3d_w4_kernel<float,3,1>", 1, 56, 4, 9, 9, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f32", True),
    ("dwconv3d_w4_kernel<float,3,2>", 1, 16, 4, 9, 9, (3, 3, 3), (2, 2, 2), (1, 1, 1), "f32", False),
    ("dwconv3d_w4_kernel<float,1,1>", 1, 24, 6, 9, 9, (5, 1, 1), (1, 1, 1), (2, 0, 0), "f32", True),
    ("dwconv3d_kernel<float>", 1, 8, 3, 3, 3, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f32", False),
]


def _row_id(row):
    return "%s-%s" % (row[0], "x".join(str(v) for v in row[1:7]))


def _f16_operands(g, N, Ci, T, H, W, Co, k, groups=1):
    x = TS.f16_exact(torch.randn(N, Ci, T, H, W, generator=g))
    fan = Ci // groups * int(np.prod(k))
    w = TS.f16_exact(torch.randn(Co, Ci // groups, *k, generator=g) * (2.0 / fan) ** 0.5)
    return x, w


def _scale_bias(bn, Co):
    from pytorchvideo_b200.engine import packing as PK
    s, b = PK.fold_bn(None, bn, Co, Co)       # exactly the fp32 values the kernel multiplies by
    return s, b


def _run_conv_row(row, family, acc_eps=TS.ACC_EPS):
    from pytorchvideo_b200 import ops
    name, N, Ci, T, H, W, Co, k, s, p, dil, act, use_res = row
    g = torch.Generator().manual_seed(N * 1000 + Ci * 7 + Co + T + H)
    x, w = _f16_operands(g, N, Ci, T, H, W, Co, k)
    bn = _bn(Co, Co + Ci)
    scale, bias = _scale_bias(bn, Co)
    res = None
    if use_res:
        with torch.no_grad():
            shape = F.conv3d(x[:, :, :, :, :], w, None, s, p, dil).shape
        res = TS.f16_exact(torch.randn(shape, generator=g))
    ref, absref = conv_ref64(x, w, scale, bias, s, p, dil, 1, act, res)
    (got, stats), launched = TS.launched_kernels(
        ops.conv3d_bn_act, x.to(_dev()), w, None, bn, s, p, dil, 1, act, None if res is None else res.to(_dev()), "f16")
    assert name in launched, "expected %s, launched %s" % (name, launched)
    ratio = TS.assert_close_to_f64(got, ref, absref, Ci * int(np.prod(k)), acc_eps=acc_eps, what=name)
    print("RATIO %s %s %.4f %.4f %s" % (family, _row_id(row), ratio[0], ratio[1], sorted(launched)))
    return launched


@pytest.mark.gpu
@pytest.mark.parametrize("row", IGEMM_ROWS, ids=[_row_id(r) for r in IGEMM_ROWS])
def test_igemm_instance(row):
    launched = _run_conv_row(row, "igemm")
    assert not any(k.startswith("conv3d_direct_kernel") for k in launched)


@pytest.mark.gpu
@pytest.mark.parametrize("row", GATHER_ROWS, ids=[_row_id(r) for r in GATHER_ROWS])
def test_gather_instance(row):
    _run_conv_row(row, "gather")


@pytest.mark.gpu
@pytest.mark.parametrize("row", STEM_ROWS, ids=[_row_id(r) for r in STEM_ROWS])
def test_stem_rows_instance(row):
    # the factored temporal stem rounds each temporal tap's partial sum to f16 before pv_temporal_tap_sum adds them:
    # allow one f16 rounding of absref instead of the accumulation term
    K = row[2] * int(np.prod(row[7]))
    acc_eps = TS.F16_EPS / (1 + K / 64.0) if row[0] == "temporal_tap_sum_kernel" else TS.ACC_EPS
    launched = _run_conv_row(row, "stem_rows", acc_eps)
    assert any(k.startswith("conv3d_stem_rows_kernel<") for k in launched), launched


@pytest.mark.gpu
@pytest.mark.parametrize("row", WINDOW_ROWS, ids=[_row_id(r) for r in WINDOW_ROWS])
def test_window_igemm_instance(row):
    launched = _run_conv_row(row, "window")
    assert not any(k.startswith("conv3d_stem_rows_kernel") for k in launched), launched
    # window mode reads the W-padded stem layout: the input went through the padded-row conversion
    assert any("ndhwc4_padw" in k or "ndhwc_padw" in k for k in launched), launched


@pytest.mark.gpu
@pytest.mark.parametrize("row", DW_ROWS, ids=[_row_id(r) for r in DW_ROWS])
def test_depthwise_instance(row):
    from pytorchvideo_b200 import ops
    name, N, Cc, T, H, W, k, s, p, dtype, se = row
    g = torch.Generator().manual_seed(Cc + T + H + W)
    x, w = _f16_operands(g, N, Cc, T, H, W, Cc, k, groups=Cc)
    bn = _bn(Cc, Cc)
    scale, bias = _scale_bias(bn, Cc)
    ref, absref = conv_ref64(x, w, scale, bias, s, p, (1, 1, 1), Cc, None, None)
    (got, stats), launched = TS.launched_kernels(
        ops.conv3d_bn_act, x.to(_dev()), w, None, bn, s, p, (1, 1, 1), Cc, None, None, dtype, None, se_sums=se)
    assert name in launched, "expected %s, launched %s" % (name, launched)
    ntaps = int(np.prod(k))
    ratio = TS.assert_close_to_f64(got, ref, absref, ntaps, what=name,
                                   rnd_eps=TS.F32_EPS if dtype == "f32" else TS.F16_EPS)
    print("RATIO depthwise %s %.4f %.4f %s" % (_row_id(row), ratio[0], ratio[1], sorted(launched)))
    if se:
        # fp32 sums of the pre-rounding outputs, quantised to 2^-24 per add: bounded by the per-element bound times
        # the number of positions
        sums = stats["se_sums"].double().cpu()
        npos = ref[0, 0].numel()
        ref_s = ref.sum(dim=(2, 3, 4))
        tol = (2.0 ** -20 * (1 + ntaps / 64.0) * absref.sum(dim=(2, 3, 4)) + npos * 2.0 ** -23
               + 2.0 ** -22 * ref_s.abs())
        if name.startswith(("dwconv3d_kernel<", "dwconv3d_w4_kernel<")):
            # the generic path sums the STORED outputs (pv_channel_sum after the stencil): one rounding per element
            tol = tol + (TS.F16_EPS if dtype == "f16" else 2.0 ** -24) * ref.abs().sum(dim=(2, 3, 4))
        assert bool(((sums - ref_s).abs() <= tol).all()), float(((sums - ref_s).abs() / tol).max())


# ---- the fp32 dense convolution (f32 parity mode: every dense convolution) ------------------------------------------
# (N, Ci, T, H, W, Co, kernel, stride, padding, dilation, act, residual, addend): conv3d_direct_kernel<float> at its
# edges - M (output rows) not a multiple of 64, Co not a multiple of 64, K = Ci * taps not a multiple of 16, strides,
# dilations, paddings, a residual, and an addend per output frame (T' = To) or per clip (T' = 1) added after the
# activation from a channel offset of a wider tensor.
DIRECT_F32_ROWS = [
    (1, 3, 4, 9, 11, 20, (3, 3, 3), (1, 1, 1), (1, 1, 1), (1, 1, 1), "relu", False, None),
    (2, 24, 3, 10, 10, 72, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), "swish", True, None),
    (1, 40, 5, 9, 9, 64, (3, 1, 1), (2, 1, 1), (2, 0, 0), (2, 1, 1), None, False, "frame"),
    (2, 16, 2, 7, 13, 130, (1, 3, 3), (1, 1, 1), (0, 2, 2), (1, 2, 2), "gelu", True, "clip"),
    (1, 8, 1, 5, 5, 8, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), "sigmoid", False, None),
    (1, 200, 2, 6, 6, 96, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), "hswish", True, "clip"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("row", DIRECT_F32_ROWS,
                         ids=["x".join(str(v) for v in r[:6]) + "-%s" % r[12] for r in DIRECT_F32_ROWS])
def test_direct_f32_instance(row):
    from pytorchvideo_b200 import _lib as L
    from pytorchvideo_b200.engine import packing as PK
    from pytorchvideo_b200.engine.plan import Plan
    N, Ci, T, H, W, Co, k, s, p, dil, act, use_res, addend = row
    g = torch.Generator().manual_seed(N + Ci + Co + T)
    x = torch.randn(N, Ci, T, H, W, generator=g)
    w = torch.randn(Co, Ci, *k, generator=g) * (2.0 / (Ci * int(np.prod(k)))) ** 0.5
    bn = _bn(Co, Co + 1)
    scale, bias = PK.fold_bn(None, bn, Co, Co)
    To, Ho, Wo = F.conv3d(x[:1, :1], w[:1, :1], None, s, p, dil).shape[2:]
    res = torch.randn(N, Co, To, Ho, Wo, generator=g) if use_res else None
    off, ca = 8, Co + 16
    add = torch.randn(N, ca, To if addend == "frame" else 1, 1, 1, generator=g) if addend else None
    plan = Plan(_dev(), L.PV_F32)
    xr = plan.emit_input_ncdhw(x.to(_dev()), Ci, PK.pad8(Ci))
    rr = plan.materialize_input(plan.emit_input_ncdhw(res.to(_dev()), Co, PK.pad8(Co))) if use_res else None
    ar = plan.materialize_input(plan.emit_input_ncdhw(add.to(_dev()), ca, PK.pad8(ca))) if addend else None
    acts = {None: L.ACT_NONE, "relu": L.ACT_RELU, "swish": L.ACT_SWISH, "gelu": L.ACT_GELU, "sigmoid": L.ACT_SIGMOID,
            "hswish": L.ACT_HSWISH}
    y = plan.emit_conv(xr, w, None, bn, s, p, dil, 1, acts[act], rr, "conv", addend=(ar, off) if addend else None)
    out, shape = plan.emit_to_ncdhw(y)
    plan.finalize()
    got, launched = TS.launched_kernels(lambda: (plan.run(torch.cuda.current_stream().cuda_stream),
                                                 torch.cuda.synchronize()))
    assert launched.get("conv3d_direct_kernel<float>") == 1, launched
    got = out.tensor[:int(np.prod(shape))].view(*shape).cpu()
    ref, absref = conv_ref64(x, w, scale, bias, s, p, dil, 1, act, res)
    if addend:
        a64 = add[:, off:off + Co].double()
        ref, absref = ref + a64, absref + a64.abs()
    ratio = TS.assert_close_to_f64(got, ref, absref, Ci * int(np.prod(k)), what="direct f32", rnd_eps=TS.F32_EPS)
    print("RATIO direct-f32 %s %.4f %.4f" % ("x".join(str(v) for v in row[:6]), ratio[0], ratio[1]))


# ---- attention -----------------------------------------------------------------------------------------------------
ATTN_NK = [1, 63, 64, 65, 393, 1569]


def _attn_rows():
    rows = []
    for D, kern in ((32, "attention_wgmma_kernel<32>"), (64, "attention_wgmma_kernel<64>"),
                    (96, "attention_wgmma_kernel<96>"), (128, "attention_mma_kernel<128>")):
        for Nq, Nk in ((1, 1), (63, 64), (64, 65), (65, 63), (393, 393), (1569, 65), (64, 1569)):
            rows.append((kern, "f16", D, Nq, Nk, (Nq + Nk) % 2 == 1))
    for D in (32, 64, 96, 128):
        for Nq, Nk in ((1, 1), (65, 63), (393, 393)):
            rows.append(("attention_kernel<float,%d>" % D, "f32", D, Nq, Nk, Nq % 2 == 1))
            rows.append(("attention_kernel<__half,%d>" % D, "unaligned", D, Nq, Nk, Nq % 2 == 0))
    return rows


ATTN_ROWS = _attn_rows()

def _attention_call(q, k, v, scale, resid, mode):
    """ops.attention; mode "unaligned": the f16 problem through the raw ABI with o 2 bytes off the 4-byte alignment the
    tensor-core kernels store with, which routes it to the CUDA-core kernel."""
    from pytorchvideo_b200 import _lib as L
    from pytorchvideo_b200 import ops
    if mode != "unaligned":
        return ops.attention(q.to(_dev()), k.to(_dev()), v.to(_dev()), scale, resid, mode)
    B, H, Nq, D = q.shape
    Nk = k.shape[2]
    qs, ks, vs = (t.permute(0, 2, 1, 3).contiguous().half().to(_dev()) for t in (q, k, v))     # [B][N][H][D]
    o = torch.empty(1 + B * Nq * H * D, dtype=torch.float16, device=_dev())
    d = _attn_desc(L.PV_F16, B, H, Nq, Nk, D, H * D, (Nq * H * D, Nk * H * D, Nk * H * D), H * D, Nq * H * D,
                   resid=1 if resid else 0)
    d.scale = scale
    ptrs = (qs.data_ptr(), ks.data_ptr(), vs.data_ptr(), o.data_ptr() + 2)
    assert L.load().pv_attention_kernel_for(C.byref(d), *ptrs) == L.ATTN_SIMT
    L.check(L.load().pv_attention_fwd(C.byref(d), *ptrs, torch.cuda.current_stream().cuda_stream), "pv_attention_fwd")
    torch.cuda.synchronize()
    return o[1:].view(B, Nq, H, D).permute(0, 2, 1, 3).float()


@pytest.mark.gpu
@pytest.mark.parametrize("row", ATTN_ROWS, ids=["%s-%s-%dx%d" % (r[0], r[1], r[3], r[4]) for r in ATTN_ROWS])
def test_attention_instance(row):
    name, mode, D, Nq, Nk, resid = row
    B, H = 2, 3
    g = torch.Generator().manual_seed(D + Nq * 3 + Nk)
    q, k, v = (TS.f16_exact(torch.randn(B, H, n, D, generator=g)) for n in (Nq, Nk, Nk))
    scale = D ** -0.5
    ref, absref = attn_ref64(q, k, v, scale, resid)
    got, launched = TS.launched_kernels(_attention_call, q, k, v, scale, resid, mode)
    assert name in launched, "expected %s, launched %s" % (name, launched)
    if Nk == 1:
        # one key: softmax is exactly 1, so o = v (+ q) after ONE f16 rounding, bit for bit
        want = (v.float() + (q.float() if resid else 0)).expand(B, H, Nq, D)     # the kernels' one fp32 add
        want = want if mode == "f32" else want.half().float()
        assert torch.equal(got.cpu(), want), float((got.cpu() - want).abs().max())
    if mode == "f32":
        # fp32 probabilities: the fp32 attention bound (ACC_EPS_ATTN_F32 over Nk, attn_score_extra64), fp32 rounding
        ratio = TS.assert_close_to_f64(got, ref, absref, Nk, acc_eps=TS.ACC_EPS_ATTN_F32, what=name,
                                       extra64=TS.attn_score_extra64(q, k, v, scale), rnd_eps=TS.F32_EPS)
    else:
        ratio = TS.assert_close_to_f64(got, ref, absref, 0, acc_eps=ACC_EPS_ATTN, what=name)
    print("RATIO attention %s-%s-%dx%d-D%d %.4f %.4f" % (name, mode, Nq, Nk, D, ratio[0], ratio[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("D", [32, 64, 96, 128])
def test_attention_large_logits_and_late_maximum(D):
    """max |scaled q.k| ~ 50; the largest key of every query sits in the last, partial key tile and the first tiles
    score far below it, so the running-max correction factor underflows to 0 when that tile arrives."""
    B, H, Nq, Nk = 1, 2, 70, 200
    g = torch.Generator().manual_seed(D)
    scale = D ** -0.5
    u = torch.randn(D, generator=g)
    q = TS.f16_exact(2 * u + 0.5 * torch.randn(B, H, Nq, D, generator=g))
    k = TS.f16_exact(torch.randn(B, H, Nk, D, generator=g) * 0.05)
    v = TS.f16_exact(torch.randn(B, H, Nk, D, generator=g))
    c = 50.0 / (scale * 2 * float(u @ u))             # q . (c u) * scale ~ 50 for every query
    k[:, :, 197] = TS.f16_exact(c * u)                # the maximum: key 197, in the last (partial) tile of 64 keys
    k[:, :, :192] = TS.f16_exact(-c * u)              # every earlier tile scores ~ -50: the running max is ~ -50
    # until the last tile, whose correction factor exp(-50 - 50) is below the fp32 range and flushes to 0
    ref, absref = attn_ref64(q, k, v, scale, True)
    logits = (q.double() * scale) @ k.double().transpose(-2, -1)
    assert float(logits.max()) > 35 and bool((logits.argmax(-1) == 197).all())
    assert float((logits[..., :192].max(-1).values - logits[..., 197]).max()) < -88     # exp underflows in fp32
    kern = "attention_mma_kernel<128>" if D == 128 else "attention_wgmma_kernel<%d>" % D
    got, launched = TS.launched_kernels(_attention_call, q, k, v, scale, True, "f16")
    assert kern in launched, launched
    ratio = TS.assert_close_to_f64(got, ref, absref, 0, acc_eps=ACC_EPS_ATTN, what=kern)
    print("RATIO attention-late-max D%d %.4f %.4f" % (D, ratio[0], ratio[1]))


def _attn_desc(dtype, B, H, Nq, Nk, D, rs, bs, o_rs, o_bs, resid=0):
    from pytorchvideo_b200 import _lib as L
    d = L.AttentionDesc()
    d.dtype, d.B, d.H, d.Nq, d.Nk, d.D = dtype, B, H, Nq, Nk, D
    d.q_row_stride = d.k_row_stride = d.v_row_stride = rs
    d.o_row_stride = o_rs
    d.q_batch_stride, d.k_batch_stride, d.v_batch_stride = bs
    d.o_batch_stride = o_bs
    d.scale, d.add_q_residual = (D ** -0.5 if D > 0 else 1.0), resid
    return d


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["model_layout", "odd_batch_stride", "o_offset_2_bytes"])
def test_attention_qkv_slices(case):
    """MViT's own layout: q / k / v are channel slices of one [B][1 + N][3 H D] qkv buffer (row stride 3 H D; the
    batch stride includes the cls row), o is a slice of a wider buffer.  The two unusual-stride cases must route to
    the CUDA-core kernel (the tensor-core kernels need 16-byte aligned q/k/v and 4-byte aligned o) and be right."""
    from pytorchvideo_b200 import _lib as L
    lib = L.load()
    B, H, D, N = 2, 2, 64, 50
    rows = 1 + N
    rs = 3 * H * D
    bs = rows * rs + (1 if case == "odd_batch_stride" else 0)
    g = torch.Generator().manual_seed(11)
    flat = TS.f16_exact(torch.randn(B * bs + rs, generator=g)).half()
    buf = flat.to(_dev())
    o_off = 1 if case == "o_offset_2_bytes" else 0
    o_rs = H * D + 8
    obuf = torch.full((B * rows * o_rs + 8,), 7.0, dtype=torch.float16, device=_dev())
    d = _attn_desc(L.PV_F16, B, H, rows, rows, D, rs, (bs, bs, bs), o_rs, rows * o_rs, resid=1)
    esz = 2
    qp, kp, vp = (buf.data_ptr() + off * esz for off in (0, H * D, 2 * H * D))
    op = obuf.data_ptr() + o_off * esz
    want_kernel = L.ATTN_WGMMA if case == "model_layout" else L.ATTN_SIMT
    assert lib.pv_attention_kernel_for(C.byref(d), qp, kp, vp, op) == want_kernel
    before = TS.kernel_counts()
    L.check(lib.pv_attention_fwd(C.byref(d), qp, kp, vp, op, torch.cuda.current_stream().cuda_stream), "attention")
    torch.cuda.synchronize()
    launched = TS.kernel_count_diff(before, TS.kernel_counts())
    assert ("attention_wgmma_kernel<64>" if case == "model_layout" else "attention_kernel<__half,64>") in launched
    host = flat.float()

    def view(off):
        t = torch.stack([host[b * bs + off: b * bs + off + rows * rs].view(rows, rs) for b in range(B)])
        return t[:, :, :H * D].reshape(B, rows, H, D).permute(0, 2, 1, 3)
    q, k, v = view(0), view(H * D), view(2 * H * D)
    ref, absref = attn_ref64(q, k, v, D ** -0.5, True)
    o = obuf.float().cpu()
    got = torch.stack([o[o_off + b * rows * o_rs: o_off + (b + 1) * rows * o_rs].view(rows, o_rs) for b in range(B)])
    assert bool((got[:, :, H * D:] == 7.0).all())            # the gap columns of the wider o rows are untouched
    got = got[:, :, :H * D].reshape(B, rows, H, D).permute(0, 2, 1, 3)
    TS.assert_close_to_f64(got, ref, absref, 0, acc_eps=ACC_EPS_ATTN, what=case)


# ---- output invariants: a channel slice of a wider, sentinel-filled NDHWC buffer ----------------------------------
SENTINEL = 0x5A5A          # an f16 bit pattern (203.25) no kernel writes by accident

INVARIANT_ROWS = [
    # (path, Ci, Co, kernel, stride, padding, residual); every C_out is padded (to 48 / 24 / 56 / 24) so there are
    # pad lanes to check
    ("tma", 64, 44, (1, 3, 3), (1, 1, 1), (0, 1, 1), True),
    ("tma", 32, 20, (3, 1, 1), (1, 1, 1), (1, 0, 0), False),
    ("gather", 24, 52, (1, 3, 3), (1, 2, 2), (0, 1, 1), True),
    ("direct", 24, 20, (1, 3, 3), (1, 1, 1), (0, 1, 1), True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("row", INVARIANT_ROWS, ids=["%s-%d-%d" % r[:3] for r in INVARIANT_ROWS])
def test_output_slice_invariants(row):
    """pv_conv3d_fwd writing channels [off, off + Co_pad) of a wider NDHWC buffer: everything outside the slice keeps
    its sentinel bits, the pad lanes [Co, Co_pad) are exactly zero, the slice matches float64."""
    from pytorchvideo_b200 import _lib as L
    from pytorchvideo_b200.engine import packing as PK
    lib = L.load()
    path, Ci, Co, k, s, p, use_res = row
    N, T, H, W = 2, 3, 10, 12
    g = torch.Generator().manual_seed(Ci * Co)
    x, w = _f16_operands(g, N, Ci, T, H, W, Co, k)
    bn = _bn(Co, 3)
    co_pad, ci_pad = PK.pad8(Co), PK.pad8(Ci)
    assert co_pad > Co
    scale, bias = PK.fold_bn(None, bn, Co, co_pad)
    To, Ho, Wo = ((T + 2 * p[0] - k[0]) // s[0] + 1, (H + 2 * p[1] - k[1]) // s[1] + 1, (W + 2 * p[2] - k[2]) // s[2] + 1)
    M = N * To * Ho * Wo
    res = TS.f16_exact(torch.randn(N, Co, To, Ho, Wo, generator=g)) if use_res else None
    ref, absref = conv_ref64(x, w, scale[:Co], bias[:Co], s, p, (1, 1, 1), 1, "relu", res)
    xd = torch.zeros(N, T, H, W, ci_pad, dtype=torch.float16)
    xd[..., :Ci] = x.permute(0, 2, 3, 4, 1).half()
    wide, off = co_pad + 40, 16
    y = torch.full((M, wide), 0, dtype=torch.int16)
    y.fill_(SENTINEL)
    y = y.view(torch.float16).to(_dev())
    rd = None
    if use_res:
        rd = torch.zeros(M, co_pad, dtype=torch.float16)
        rd[:, :Co] = res.permute(0, 2, 3, 4, 1).reshape(M, Co).half()
        rd = rd.to(_dev())
    d = L.Conv3dDesc()
    d.dtype = L.PV_F16
    d.N, d.Ti, d.Hi, d.Wi, d.Ci = N, T, H, W, ci_pad
    d.To, d.Ho, d.Wo, d.Co = To, Ho, Wo, co_pad
    d.kt, d.kh, d.kw = k
    d.st, d.sh, d.sw = s
    d.pt, d.ph, d.pw = p
    d.dt = d.dh = d.dw = 1
    d.groups, d.act, d.has_residual = 1, L.ACT_RELU, 1 if use_res else 0
    d.x_row_stride, d.y_row_stride, d.res_row_stride = ci_pad, wide, co_pad if use_res else 0
    d.ci_pad64 = ci_pad if ci_pad < 64 else PK.pad_to(ci_pad, 64)
    if path == "direct":
        algo, wp = L.ALGO_DIRECT, PK.pack_dense_direct(w, ci_pad, co_pad, torch.float16)
        want = "conv3d_direct_kernel<__half>"
    else:
        algo, wp = L.ALGO_TCGEN05, PK.pack_dense_tcgen05(w, d.ci_pad64, co_pad)
        want = "conv3d_igemm_gather_kernel<" if path == "gather" else "conv3d_igemm_kernel<"
    xg, wg, sg, bg = xd.to(_dev()), wp.to(_dev()), scale.to(_dev()), bias.to(_dev())
    before = TS.kernel_counts()
    L.check(lib.pv_conv3d_fwd(C.byref(d), algo, xg.data_ptr(), wg.data_ptr(), sg.data_ptr(), bg.data_ptr(),
                              rd.data_ptr() if rd is not None else None, y.data_ptr() + off * 2,
                              torch.cuda.current_stream().cuda_stream), "pv_conv3d_fwd")
    torch.cuda.synchronize()
    launched = TS.kernel_count_diff(before, TS.kernel_counts())
    assert any(kname.startswith(want) for kname in launched), launched
    _check_slice(y, M, wide, off, Co, co_pad)
    got = y.cpu()[:, off:off + Co].float().view(N, To, Ho, Wo, Co).permute(0, 4, 1, 2, 3)
    TS.assert_close_to_f64(got, ref, absref, Ci * int(np.prod(k)), what=path)


def _check_slice(y, M, wide, off, Co, co_pad):
    """Sentinel bits outside [off, off + co_pad), exact zeros in the pad lanes [off + Co, off + co_pad)."""
    yb = y.cpu().view(torch.int16).view(M, wide)
    outside = torch.ones(M, wide, dtype=torch.bool)
    outside[:, off:off + co_pad] = False
    assert bool((yb[outside] == SENTINEL).all()), "a kernel wrote outside its channel slice"
    assert bool((yb[:, off + Co:off + co_pad] == 0).all()), "pad lanes are not exactly zero"


@pytest.mark.gpu
@pytest.mark.parametrize("Co,k", [(20, (1, 3, 3)), (60, (1, 7, 7))])
def test_stem_rows_output_slice_invariants(Co, k):
    """pv_conv3d_stem_rows_fwd (its own output tensor map) writing a channel slice of a wider sentinel-filled buffer,
    C_out padded to a multiple of 8: same invariants as test_output_slice_invariants."""
    from pytorchvideo_b200 import _lib as L
    from pytorchvideo_b200.engine import packing as PK
    lib = L.load()
    N, T, H, W = 2, 2, 14, 150          # W_out = 75 (one partial W tile)
    kt, kh, kw = k
    s, p = (1, 2, 2), (0, kh // 2, kw // 2)
    g = torch.Generator().manual_seed(Co)
    x, w = _f16_operands(g, N, 3, T, H, W, Co, k)
    bn = _bn(Co, 4)
    co_pad = PK.pad8(Co)
    assert co_pad > Co
    scale, bias = PK.fold_bn(None, bn, Co, co_pad)
    To, Ho, Wo = T, (H + 2 * p[1] - kh) // 2 + 1, (W + 2 * p[2] - kw) // 2 + 1
    M = N * To * Ho * Wo
    ref, absref = conv_ref64(x, w, scale[:Co], bias[:Co], s, p, (1, 1, 1), 1, "relu", None)
    # the W-padded 4-channel stem layout, as engine/plan.py builds it for a window-mode stem
    wp = (p[2] + 3) // 4 * 4
    lead = PK.window_lead(wp, p[2], 4)
    win = PK.window_elems(kw, 4, lead)
    need = wp - p[2] + max(W + 2 * p[2], (Wo - 1) * 2 + (win + 3) // 4)
    w_phys = (need + 3) // 4 * 4
    xs = torch.zeros(N * T * H * w_phys * 4 + 64 * 4, dtype=torch.float16, device=_dev())
    xin = x.contiguous().to(_dev())
    L.check(lib.pv_ncdhw_to_ndhwc_padw(xin.data_ptr(), L.PV_F32, xs.data_ptr(), L.PV_F16, N, 3, T, H, W, 4, wp, w_phys,
                                       torch.cuda.current_stream().cuda_stream), "pv_ncdhw_to_ndhwc_padw")
    d = L.Conv3dDesc()
    d.dtype = L.PV_F16
    d.N, d.Ti, d.Hi, d.Wi, d.Ci = N, T, H, W, 4
    d.To, d.Ho, d.Wo, d.Co = To, Ho, Wo, co_pad
    d.kt, d.kh, d.kw = k
    d.st, d.sh, d.sw = s
    d.pt, d.ph, d.pw = p
    d.dt = d.dh = d.dw = 1
    d.groups, d.act, d.has_residual = 1, L.ACT_RELU, 0
    wide, off = co_pad + 40, 16
    d.x_row_stride, d.y_row_stride = 4, wide
    d.ci_pad64, d.x_w_pad, d.x_w_phys = win, wp, w_phys
    assert lib.pv_conv3d_stem_rows_supported(C.byref(d))
    wg = PK.pack_stem_rows(w, 4, co_pad, lead).to(_dev())
    sg, bg = scale.to(_dev()), bias.to(_dev())
    zero_row = torch.zeros(4096, dtype=torch.float16, device=_dev())
    y = torch.full((M * wide,), SENTINEL, dtype=torch.int16).view(torch.float16).to(_dev())
    before = TS.kernel_counts()
    L.check(lib.pv_conv3d_stem_rows_fwd(C.byref(d), xs.data_ptr(), wg.data_ptr(), sg.data_ptr(), bg.data_ptr(),
                                        zero_row.data_ptr(), y.data_ptr() + off * 2,
                                        torch.cuda.current_stream().cuda_stream), "pv_conv3d_stem_rows_fwd")
    torch.cuda.synchronize()
    launched = TS.kernel_count_diff(before, TS.kernel_counts())
    assert any(kname.startswith("conv3d_stem_rows_kernel<") for kname in launched), launched
    _check_slice(y, M, wide, off, Co, co_pad)
    got = y.cpu().view(M, wide)[:, off:off + Co].float().view(N, To, Ho, Wo, Co).permute(0, 4, 1, 2, 3)
    TS.assert_close_to_f64(got, ref, absref, 3 * int(np.prod(k)), what="stem rows slice")


@pytest.mark.gpu
@pytest.mark.parametrize("k,s,se", [((3, 3, 3), (1, 2, 2), False), ((3, 3, 3), (1, 1, 1), True),
                                    ((1, 3, 3), (1, 1, 1), True), ((3, 1, 1), (1, 1, 1), False)])
def test_depthwise_cls_row_batch_stride(k, s, se):
    """MViT's pooling convs: every sample of x and y is [1 + T*H*W][C] with a cls row in front of the patch tokens, so
    x_batch_stride / y_batch_stride step over it.  The kernels must read and write only the patch rows (the cls rows
    and the gap columns keep their sentinel bits) and match float64."""
    from pytorchvideo_b200 import _lib as L
    from pytorchvideo_b200.engine import packing as PK
    lib = L.load()
    N, Cc, T, H, W = 2, 96, 4, 8, 8
    p = tuple(kk // 2 for kk in k)
    g = torch.Generator().manual_seed(Cc + sum(k) + s[1])
    x, w = _f16_operands(g, N, Cc, T, H, W, Cc, k, groups=Cc)
    bn = _bn(Cc, 9)
    scale, bias = PK.fold_bn(None, bn, Cc, Cc)
    ref, absref = conv_ref64(x, w, scale, bias, s, p, (1, 1, 1), Cc, None, None)
    To, Ho, Wo = ref.shape[2:]
    xrows, yrows = 1 + T * H * W, 1 + To * Ho * Wo
    xrs, yrs = Cc + 8, Cc + 16                        # rows wider than C as well
    xb = torch.full((N, xrows, xrs), SENTINEL, dtype=torch.int16).view(torch.float16)
    xb[:, 1:, :Cc] = x.permute(0, 2, 3, 4, 1).reshape(N, T * H * W, Cc).half()
    xg = xb.to(_dev())
    y = torch.full((N, yrows, yrs), SENTINEL, dtype=torch.int16).view(torch.float16).to(_dev())
    d = L.Conv3dDesc()
    d.dtype = L.PV_F16
    d.N, d.Ti, d.Hi, d.Wi, d.Ci = N, T, H, W, Cc
    d.To, d.Ho, d.Wo, d.Co = To, Ho, Wo, Cc
    d.kt, d.kh, d.kw = k
    d.st, d.sh, d.sw = s
    d.pt, d.ph, d.pw = p
    d.dt = d.dh = d.dw = 1
    d.groups, d.act, d.has_residual = Cc, L.ACT_NONE, 0
    d.x_row_stride, d.y_row_stride = xrs, yrs
    d.x_batch_stride, d.y_batch_stride = xrows * xrs, yrows * yrs
    wg = PK.pack_depthwise(w, Cc, torch.float16).to(_dev())
    sg, bg = scale.to(_dev()), bias.to(_dev())
    sums = torch.zeros(2 * N * Cc, dtype=torch.float32, device=_dev()) if se else None
    before = TS.kernel_counts()
    L.check(lib.pv_dwconv3d_fwd(C.byref(d), xg.data_ptr() + xrs * 2, wg.data_ptr(), sg.data_ptr(), bg.data_ptr(),
                                y.data_ptr() + yrs * 2, sums.data_ptr() if se else None,
                                torch.cuda.current_stream().cuda_stream), "pv_dwconv3d_fwd")
    torch.cuda.synchronize()
    launched = TS.kernel_count_diff(before, TS.kernel_counts())
    assert any(kname.startswith(("dwconv3d_lane_kernel<", "dwconv3d_tile_kernel<", "dwconv_temporal_kernel<"))
               for kname in launched), launched
    yb = y.cpu().view(torch.int16)
    assert bool((yb[:, 0] == SENTINEL).all()), "cls row overwritten"
    assert bool((yb[:, :, Cc:] == SENTINEL).all()), "gap columns overwritten"
    got = y.cpu()[:, 1:, :Cc].float().view(N, To, Ho, Wo, Cc).permute(0, 4, 1, 2, 3)
    ratio = TS.assert_close_to_f64(got, ref, absref, int(np.prod(k)), what="cls-row depthwise")
    print("RATIO depthwise cls-row %s %s %.4f %.4f %s" % (k, s, ratio[0], ratio[1], sorted(launched)))
    if se:
        got_s = (sums.cpu().view(torch.int64).view(N, Cc).double() / 2 ** 24)
        ref_s = ref.sum(dim=(2, 3, 4))
        tol = 2.0 ** -20 * (1 + int(np.prod(k)) / 64.0) * absref.sum(dim=(2, 3, 4)) + To * Ho * Wo * 2.0 ** -23
        assert bool(((got_s - ref_s).abs() <= tol + 2.0 ** -22 * ref_s.abs()).all())


# ---- fused bottleneck block (csrc/pv_fastblock.cu) -----------------------------------------------------------------
# One launch per ResBlock: a = relu(bn_a(conv_a(x))) (kt,1,1); b = relu(bn_b(conv_b(a))) (1,3,3) stride (1,s,s);
# y = act(bn_c(conv_c(b)) + shortcut).  The instance is bottleneck_fused_kernel<Cin,Cmid,kt,s,projection>.  Tile
# (TH x TW outputs) and frame chunk (TC frames per CTA) come from a cost model over the SM count
# (pv_bottleneck_fused_tiling); each row claims the tiling properties it is there for, and the test checks them with
# the query at the device's SM count (test_fused_row_claims_hold checks them for 132- and 114-SM parts on the CPU):
#   partial_h / partial_w  the last tile row / column of the plane is cut by the image edge
#   chunks                 a clip is split over several CTAs, each of which reloads its halo frame
#   short_chunk            ... and the last chunk holds fewer frames than the others
#   single_tile            the whole plane is one tile (its halo is image border on every side)
def _fb(cin, cmid, kt, s, proj):
    return "bottleneck_fused_kernel<%d,%d,%d,%d,%d>" % (cin, cmid, kt, s, proj)


FB_RES2_0, FB_RES2, FB_PW = _fb(8, 8, 3, 1, 1), _fb(32, 8, 3, 1, 0), _fb(32, 8, 1, 1, 0)
FB_RES3_0, FB_PROJ16, FB_RES3 = _fb(32, 16, 3, 2, 1), _fb(32, 16, 3, 1, 1), _fb(64, 16, 3, 1, 0)
PH, PW, CH, SC, ST = "partial_h", "partial_w", "chunks", "short_chunk", "single_tile"

# (expected instance, N, T, H, W, act, extra x row elements, extra y row elements, claimed tiling properties)
FUSED_ROWS = [
    # partial tiles in both directions, several frame chunks and a short last chunk
    (FB_RES2_0, 1, 9, 10, 9, "relu", 0, 0, (PH, PW, CH, SC)),
    (FB_RES2, 1, 9, 10, 9, None, 8, 0, (PH, PW, CH, SC)),
    (FB_PW, 1, 9, 9, 11, "relu", 0, 8, (PH, PW, CH, SC)),
    (FB_RES3_0, 1, 9, 9, 11, None, 0, 0, (PH, PW, CH, SC)),
    (FB_PROJ16, 1, 9, 10, 9, "relu", 16, 8, (PH, PW, CH, SC)),
    (FB_RES3, 1, 9, 10, 11, "relu", 0, 0, (PH, PW, CH, SC)),
    # clips of 1 and 2 frames: both temporal neighbours of conv_a are padding
    (FB_RES2_0, 2, 1, 1, 1, "relu", 0, 0, (ST,)),
    (FB_RES2_0, 1, 2, 2, 3, None, 8, 8, (ST,)),
    (FB_RES2, 1, 1, 1, 9, None, 0, 0, ()),
    (FB_RES2, 2, 2, 5, 6, "relu", 0, 0, ()),
    (FB_RES3_0, 1, 1, 1, 1, "relu", 0, 0, (ST,)),
    (FB_RES3_0, 2, 2, 2, 3, None, 8, 0, (ST,)),
    (FB_PROJ16, 1, 1, 2, 3, None, 0, 0, (ST,)),
    (FB_PROJ16, 2, 2, 1, 9, "relu", 0, 16, ()),
    (FB_RES3, 1, 1, 1, 9, "relu", 0, 0, ()),
    (FB_RES3, 1, 2, 1, 1, None, 16, 0, (ST,)),
    # tiny planes; stride 2 with odd and even H and W
    (FB_PW, 1, 3, 1, 1, None, 0, 0, (ST,)),
    (FB_PW, 2, 4, 2, 3, "relu", 8, 8, (ST,)),
    (FB_RES3_0, 1, 3, 4, 6, "relu", 0, 8, ()),
    (FB_RES3_0, 1, 3, 5, 7, None, 0, 0, ()),
    (FB_RES3_0, 1, 4, 6, 5, "relu", 8, 0, ()),
    # SlowFast-R50 Fast pathway at batch 8 (32 frames): res2 block 0, res2 blocks 1-2, res3 block 0, res3 blocks 1-3
    (FB_RES2_0, 8, 32, 56, 56, "relu", 0, 0, (CH, SC)),
    (FB_RES2, 8, 32, 56, 56, "relu", 0, 0, (CH,)),
    (FB_RES3_0, 8, 32, 56, 56, "relu", 0, 0, (PW, CH)),
    (FB_RES3, 8, 32, 28, 28, "relu", 0, 0, (CH,)),
]


def _fused_row_id(row):
    return "%s-%s-%s-x%d-y%d" % (row[0], "x".join(str(v) for v in row[1:5]), row[5] or "none", row[6], row[7])


def _fused_shape(inst):
    cin, cmid, kt, s, proj = (int(v) for v in re.match(r"bottleneck_fused_kernel<(\d+),(\d+),(\d+),(\d+),(\d+)>$",
                                                       inst).groups())
    return cin, cmid, 4 * cmid, kt, s, proj


def _fused_desc(inst, N, T, H, W, act="relu", xrs=None, yrs=None):
    from pytorchvideo_b200 import _lib as L
    cin, cmid, cout, kt, s, proj = _fused_shape(inst)
    d = L.BottleneckDesc()
    d.N, d.T, d.H, d.W = N, T, H, W
    d.Cin, d.Cmid, d.Cout, d.kt, d.sb, d.has_shortcut = cin, cmid, cout, kt, s, proj
    d.act = L.ACT_RELU if act == "relu" else L.ACT_NONE
    d.x_row_stride, d.y_row_stride = xrs or cin, yrs or cout
    return d


def fused_tiling(d, sm_count):
    """(tile_h, tile_w, frames per CTA, shared-memory bytes) that pv_bottleneck_fused_fwd would use on sm_count SMs."""
    from pytorchvideo_b200 import _lib as L
    th, tw, tc, smem = C.c_int(), C.c_int(), C.c_int(), C.c_longlong()
    L.check(L.load().pv_bottleneck_fused_tiling(C.byref(d), sm_count, C.byref(th), C.byref(tw), C.byref(tc),
                                                C.byref(smem)), "pv_bottleneck_fused_tiling")
    return th.value, tw.value, tc.value, smem.value


def fused_tiling_properties(d, sm_count):
    th, tw, tc, _ = fused_tiling(d, sm_count)
    Ho, Wo = (d.H - 1) // d.sb + 1, (d.W - 1) // d.sb + 1
    chunks = -(-d.T // tc)
    props = set()
    if Ho % th:
        props.add(PH)
    if Wo % tw:
        props.add(PW)
    if chunks > 1:
        props.add(CH)
        if d.T % tc:
            props.add(SC)
    if Ho <= th and Wo <= tw:
        props.add(ST)
    return props


def _fused_operands(inst, N, T, H, W, seed):
    """f16-grid x and weights, and the folded fp32 BatchNorm (scale, bias) of each convolution."""
    cin, cmid, cout, kt, s, proj = _fused_shape(inst)
    g = torch.Generator().manual_seed(seed)
    x = TS.f16_exact(torch.randn(N, cin, T, H, W, generator=g))

    def w(co, ci, k):
        return TS.f16_exact(torch.randn(co, ci, *k, generator=g) * (2.0 / (ci * int(np.prod(k)))) ** 0.5)
    wa, wb, wc = w(cmid, cin, (kt, 1, 1)), w(cmid, cmid, (1, 3, 3)), w(cout, cmid, (1, 1, 1))
    ws = w(cout, cin, (1, 1, 1)) if proj else None
    folds = []
    for i, c in enumerate((cmid, cmid, cout, cout if proj else 0)):
        folds += list(_scale_bias(_bn(c, seed + i), c)) if c else [None, None]
    return x, wa, wb, wc, ws, tuple(folds)


def _fused_k(inst):
    cin, cmid, cout, kt, s, proj = _fused_shape(inst)
    return cmid + (cin if proj else 0)


def _fused_call(d, x_ptr, y_ptr, dev_ops):
    """pv_bottleneck_fused_fwd on raw device pointers; returns {instance: launches}."""
    from pytorchvideo_b200 import _lib as L
    wa, wb, wc, ws, sa, ba, sbn, bbn, sc, bc, ssc, bsc = dev_ops
    p = lambda t: None if t is None else t.data_ptr()
    before = TS.kernel_counts()
    L.check(L.load().pv_bottleneck_fused_fwd(C.byref(d), x_ptr, p(wa), p(wb), p(wc), p(ws), p(sa), p(ba), p(sbn),
                                             p(bbn), p(sc), p(bc), p(ssc), p(bsc), y_ptr,
                                             torch.cuda.current_stream().cuda_stream), "pv_bottleneck_fused_fwd")
    torch.cuda.synchronize()
    return TS.kernel_count_diff(before, TS.kernel_counts())


def _fused_device_operands(inst, wa, wb, wc, ws, folds):
    from pytorchvideo_b200.engine import packing as PK
    cin, cmid, cout, kt, s, proj = _fused_shape(inst)
    packed = [PK.pack_rows_k16(wa, cin, cmid), PK.pack_rows_k16(wb, cmid, cmid), PK.pack_rows_k16(wc, cmid, cout),
              PK.pack_rows_k16(ws, cin, cout) if ws is not None else None]
    return tuple(None if t is None else t.to(_dev()) for t in packed + list(folds))


def _fused_run(inst, x, dev_ops, act, xrs, yrs):
    """x (NCDHW, f16 grid) -> (y NCDHW float on the device, launched); x and y in NDHWC buffers with the given rows."""
    N, cin, T, H, W = x.shape
    _, _, cout, _, s, _ = _fused_shape(inst)
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    xd = torch.zeros(N, T, H, W, xrs, dtype=torch.float16, device=_dev())
    xd[..., :cin] = x.to(_dev()).permute(0, 2, 3, 4, 1).half()
    yd = torch.zeros(N, T, Ho, Wo, yrs, dtype=torch.float16, device=_dev())
    d = _fused_desc(inst, N, T, H, W, act, xrs, yrs)
    launched = _fused_call(d, xd.data_ptr(), yd.data_ptr(), dev_ops)
    return yd[..., :cout].permute(0, 4, 1, 2, 3).float(), launched


@pytest.mark.gpu
@pytest.mark.parametrize("row", FUSED_ROWS, ids=[_fused_row_id(r) for r in FUSED_ROWS])
def test_fused_instance(row):
    from pytorchvideo_b200 import _lib as L
    inst, N, T, H, W, act, xe, ye, claims = row
    cin, cmid, cout, kt, s, proj = _fused_shape(inst)
    sm, _ = L.require_device()
    d = _fused_desc(inst, N, T, H, W, act, cin + xe, cout + ye)
    props = fused_tiling_properties(d, sm)
    assert set(claims) <= props, "row claims %s, tiling %s on %d SMs gives %s" % (claims, fused_tiling(d, sm), sm, props)
    x, wa, wb, wc, ws, folds = _fused_operands(inst, N, T, H, W, seed=N + T * 3 + H * 5 + W * 7 + cin)
    dev_ops = _fused_device_operands(inst, wa, wb, wc, ws, folds)
    got, launched = _fused_run(inst, x, dev_ops, act, cin + xe, cout + ye)
    assert launched == {inst: 1}, "expected %s, launched %s" % (inst, launched)
    big = N * T * H * W > 100000
    y, _, _, Y, prop = fused_block_ref64(x.to(_dev()) if big else x, wa, wb, wc, ws, folds, kt, s, act)
    ratio = TS.assert_close_to_f64(got, y, Y, _fused_k(inst), what=inst, extra64=prop)
    print("RATIO fused %s %.4f %.4f %.4f tiling=%s" % (_fused_row_id(row), ratio[0], ratio[1], ratio[2],
                                                      fused_tiling(d, sm)[:3]))


FUSED_POISON_ROWS = [
    (FB_RES2_0, 2, 5, 9, 10, "relu"),
    (FB_RES2, 1, 9, 10, 9, None),
    (FB_RES3_0, 2, 4, 9, 11, "relu"),
    (FB_RES3, 1, 6, 7, 13, None),
]
NAN16 = 0x7E00             # an f16 quiet NaN


@pytest.mark.gpu
@pytest.mark.parametrize("row", FUSED_POISON_ROWS, ids=["%s-%s" % (r[0], "x".join(map(str, r[1:5]))) for r in FUSED_POISON_ROWS])
def test_fused_poison_and_sentinel(row):
    """x is a channel slice of wider rows between guard rows, and everything around it is f16 NaN: the kernel must
    not read it (a NaN times a zero weight is still NaN).  y is a channel slice of a sentinel-filled buffer with
    wider rows and guard rows: every byte outside the slice keeps its sentinel, and the slice matches float64."""
    inst, N, T, H, W, act = row
    cin, cmid, cout, kt, s, proj = _fused_shape(inst)
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    xrs, yrs, guard = cin + 8, cout + 16, 37
    mx, my = N * T * H * W, N * T * Ho * Wo
    x, wa, wb, wc, ws, folds = _fused_operands(inst, N, T, H, W, seed=101 + cin + H)
    dev_ops = _fused_device_operands(inst, wa, wb, wc, ws, folds)
    xb = torch.full((guard + mx + guard, xrs), NAN16, dtype=torch.int16).view(torch.float16)
    xb[guard:guard + mx, :cin] = x.permute(0, 2, 3, 4, 1).reshape(mx, cin).half()
    xg = xb.to(_dev())
    yg = torch.full((guard + my + guard, yrs), SENTINEL, dtype=torch.int16).view(torch.float16).to(_dev())
    d = _fused_desc(inst, N, T, H, W, act, xrs, yrs)
    launched = _fused_call(d, xg.data_ptr() + guard * xrs * 2, yg.data_ptr() + guard * yrs * 2, dev_ops)
    assert launched == {inst: 1}, launched
    yb = yg.cpu().view(torch.int16)
    inside = torch.zeros_like(yb, dtype=torch.bool)
    inside[guard:guard + my, :cout] = True
    assert bool((yb[~inside] == SENTINEL).all()), "the kernel wrote outside y's slice"
    got16 = yg.cpu()[guard:guard + my, :cout]
    assert not bool(torch.isnan(got16).any()), "NaN in y: the kernel read poisoned x bytes"
    got = got16.float().view(N, T, Ho, Wo, cout).permute(0, 4, 1, 2, 3)
    y, _, _, Y, prop = fused_block_ref64(x, wa, wb, wc, ws, folds, kt, s, act)
    ratio = TS.assert_close_to_f64(got, y, Y, _fused_k(inst), what=inst, extra64=prop)
    print("RATIO fused poison %s %.4f %.4f %.4f" % (inst, ratio[0], ratio[1], ratio[2]))


# Rows where a batch of 8 clips and one clip alone choose different (TH, TW, TC): every output element's arithmetic
# (mma K order, roundings of a and b) does not depend on which tile or frame chunk computes it, so clip i of the batch
# must equal the clip run alone bit for bit; a difference is a tile, halo or chunk bug.
FUSED_BATCH_ROWS = [
    (FB_RES2_0, 32, 56, 56),
    (FB_RES2, 32, 56, 56),
    (FB_PW, 32, 56, 56),
    (FB_RES3_0, 32, 56, 56),
    (FB_PROJ16, 32, 56, 56),
    (FB_RES3, 32, 28, 28),
    (FB_RES3, 12, 17, 14),
]


@pytest.mark.gpu
@pytest.mark.parametrize("row", FUSED_BATCH_ROWS, ids=["%s-%s" % (r[0], "x".join(map(str, r[1:]))) for r in FUSED_BATCH_ROWS])
def test_fused_batch_invariance(row):
    from pytorchvideo_b200 import _lib as L
    inst, T, H, W = row
    cin, cmid, cout, kt, s, proj = _fused_shape(inst)
    sm, _ = L.require_device()
    t8, t1 = fused_tiling(_fused_desc(inst, 8, T, H, W), sm)[:3], fused_tiling(_fused_desc(inst, 1, T, H, W), sm)[:3]
    assert t8 != t1, (t8, t1)
    x, wa, wb, wc, ws, folds = _fused_operands(inst, 8, T, H, W, seed=7 + cin + H)
    dev_ops = _fused_device_operands(inst, wa, wb, wc, ws, folds)
    y8, launched = _fused_run(inst, x, dev_ops, "relu", cin, cout)
    assert launched == {inst: 1}, launched
    for i in range(8):
        y1, _ = _fused_run(inst, x[i:i + 1], dev_ops, "relu", cin, cout)
        assert torch.equal(y8[i:i + 1], y1), "clip %d: batch tiling %s and single-clip tiling %s disagree at %d elements" % (
            i, t8, t1, int((y8[i:i + 1] != y1).sum()))


# ---- CPU: the instance ledger --------------------------------------------------------------------------------------
def compiled_instances():
    """The kernel instances the launch sites in csrc/ can name, parsed from their instantiation lines."""
    def src(f):
        return open(os.path.join(CSRC, f)).read()
    out = set()
    for bn, kb in re.findall(r"PV_IG_LAUNCH\((\d+), (\d+)\)", src("pv_igemm.cu")):
        out.add("conv3d_igemm_kernel<%s,%s>" % (bn, kb))
    for bn, ks in re.findall(r"PV_ST_LAUNCH\((\d+), (\d+)\)", src("pv_stem.cu")):
        out.add("conv3d_stem_rows_kernel<%s,%s>" % (bn, ks))
    for bn in re.findall(r"PV_GG_LAUNCH\((\d+)\)", src("pv_igemm_gather.cu")):
        out.add("conv3d_igemm_gather_kernel<%s>" % bn)
    for kw, sw in re.findall(r"PV_DWT\((\d+), (\d+)\)", src("pv_dwconv.cu")):
        out.add("dwconv3d_tile_kernel<%s,%s>" % (kw, sw))
    for kt in re.findall(r"dwconv_temporal_kernel<(\d+)><<<", src("pv_dwconv.cu")):
        out.add("dwconv_temporal_kernel<%s>" % kt)
    for s, ph, pw in re.findall(r"PV_DWL\((\d+), (\d+), (\d+)\);", src("pv_dwlane.cu")):
        out.add("dwconv3d_lane_kernel<%s,%s,%s>" % (s, ph, pw))
    for dd in re.findall(r"PV_AW\((\d+)\)", src("pv_attention_wgmma.cu")):
        out.add("attention_wgmma_kernel<%s>" % dd)
    for dd in re.findall(r"PV_AM\((\d+)\)", src("pv_attention_mma.cu")):
        out.add("attention_mma_kernel<%s>" % dd)
    for dd in re.findall(r"PV_ATT\((\d+)\)", src("pv_attention.cu")):
        out.update({"attention_kernel<__half,%s>" % dd, "attention_kernel<float,%s>" % dd})
    for args in re.findall(r"PV_FB\((\d+), (\d+), (\d+), (\d+), (\d+)\)", src("pv_fastblock.cu")):
        out.add("bottleneck_fused_kernel<%s>" % ",".join(args))
    return out


EXPECTED_INSTANCES = {r[0] for r in IGEMM_ROWS + GATHER_ROWS + STEM_ROWS + WINDOW_ROWS + DW_ROWS + ATTN_ROWS + FUSED_ROWS}


def test_instance_ledger_covers_every_compiled_instance():
    compiled = compiled_instances()
    assert len([n for n in compiled if n.startswith("conv3d_igemm_kernel<")]) == 12
    assert len([n for n in compiled if n.startswith("conv3d_stem_rows_kernel<")]) == 12
    assert len([n for n in compiled if n.startswith("conv3d_igemm_gather_kernel<")]) == 4
    assert len([n for n in compiled if n.startswith("dwconv3d_tile_kernel<")]) == 4
    assert len([n for n in compiled if n.startswith("dwconv3d_lane_kernel<")]) == 4
    assert len([n for n in compiled if n.startswith("bottleneck_fused_kernel<")]) == 6
    # the rows also cover kernels whose instances are parsed elsewhere (pv_simt.cu): compare this ledger's families
    families = {n.split("<")[0] for n in compiled}
    expected = {n for n in EXPECTED_INSTANCES if n.split("<")[0] in families}
    assert compiled == expected, ("compiled instances no matrix row reaches: %s" % sorted(compiled - expected),
                                  "matrix rows naming no compiled instance: %s" % sorted(expected - compiled))


def test_launch_sites_name_their_instances():
    """Every launch site of the matrix's kernels passes a name with its template arguments to the launch counter."""
    for f, pat in (("pv_igemm.cu", r'"conv3d_igemm_kernel<" #BN "," #KB ">"'),
                   ("pv_stem.cu", r'"conv3d_stem_rows_kernel<" #BN "," #KS ">"'),
                   ("pv_igemm_gather.cu", r'"conv3d_igemm_gather_kernel<" #BN ">"'),
                   ("pv_dwconv.cu", r'"dwconv3d_tile_kernel<" #KW_ "," #SW_ ">"'),
                   ("pv_dwlane.cu", r'PV_PRE_NAME("dwconv3d_lane_kernel<" #S_ "," #PH_ "," #PW_, PRE_)'),
                   ("pv_attention_wgmma.cu", r'"attention_wgmma_kernel<" #DD ">"'),
                   ("pv_fastblock.cu", r'"bottleneck_fused_kernel<" #CI "," #CM "," #KT_ "," #SB_ "," #SC_ ">"')):
        assert pat in open(os.path.join(CSRC, f)).read(), f


def test_kernel_counts_read_back():
    """pv_kernel_counts is callable without a GPU and parses into a dict (empty before any launch)."""
    from pytorchvideo_b200 import _lib as L
    counts = L.kernel_counts()
    assert isinstance(counts, dict)
    assert all(isinstance(v, int) and v > 0 for v in counts.values())
    assert TS.kernel_count_diff({"a<1>": 2}, {"a<1>": 5, "b": 1}) == {"a<1>": 3, "b": 1}


# ---- CPU: attention routing ----------------------------------------------------------------------------------------
def _route(dtype="f16", D=64, rs=192, bs=(51 * 192,) * 3, o_rs=128, o_bs=51 * 128, q=0x10000, k=0x20000, v=0x30000,
           o=0x40000):
    from pytorchvideo_b200 import _lib as L
    d = _attn_desc(L.PV_F16 if dtype == "f16" else L.PV_F32, 2, 2, 51, 51, D, rs, bs, o_rs, o_bs)
    return L.load().pv_attention_kernel_for(C.byref(d), q, k, v, o)


def test_attention_routing_aligned():
    from pytorchvideo_b200 import _lib as L
    for D in (32, 64, 96):
        assert _route(D=D, rs=3 * 2 * D, o_rs=2 * D, bs=(51 * 6 * D,) * 3, o_bs=51 * 2 * D) == L.ATTN_WGMMA
    assert _route(D=128, rs=768, o_rs=256, bs=(51 * 768,) * 3, o_bs=51 * 256) == L.ATTN_MMA
    assert _route(dtype="f32", D=64) == L.ATTN_SIMT
    assert _route(D=48) < 0 and _route(D=0) < 0


@pytest.mark.parametrize("D", [64, 128])
def test_attention_routing_misaligned_goes_to_cuda_cores(D):
    """Strides and pointers the tensor-core kernels would read or write misaligned route to the CUDA-core kernel."""
    from pytorchvideo_b200 import _lib as L
    base = dict(D=D, rs=6 * D, o_rs=2 * D, bs=(51 * 6 * D,) * 3, o_bs=51 * 2 * D)
    assert _route(**base) != L.ATTN_SIMT
    odd = 51 * 6 * D + 1
    for bad in (dict(bs=(odd, 51 * 6 * D, 51 * 6 * D)), dict(bs=(51 * 6 * D, odd, 51 * 6 * D)),
                dict(bs=(51 * 6 * D, 51 * 6 * D, odd)), dict(bs=(51 * 6 * D + 4,) * 3),
                dict(o_bs=51 * 2 * D + 1), dict(o=0x40002), dict(o=0x40001), dict(q=0x10008), dict(k=0x20002),
                dict(rs=6 * D + 4), dict(o_rs=2 * D + 1)):
        args = dict(base)
        args.update(bad)
        assert _route(**args) == L.ATTN_SIMT, bad


def test_attention_routing_only_admits_encodable_strides():
    """The tensor-core kernels' rule also covers what their tensor maps need: no zero / overlapping / >= 2^40-byte
    strides.  A single sample's batch stride is never used and is not checked."""
    from pytorchvideo_b200 import _lib as L
    base = dict(D=64, rs=384, o_rs=128, bs=(51 * 384,) * 3, o_bs=51 * 128)
    assert _route(**base) == L.ATTN_WGMMA
    for bad in (dict(bs=(0, 51 * 384, 51 * 384)), dict(bs=(51 * 384, 0, 0)),      # broadcast k / v over the batch
                dict(bs=(50 * 384, 51 * 384, 51 * 384)),                          # samples overlap
                dict(rs=64), dict(rs=0),                                          # rows narrower than H*D
                dict(bs=(1 << 39,) * 3), dict(rs=1 << 39)):                       # >= 2^40 bytes
        args = dict(base)
        args.update(bad)
        assert _route(**args) == L.ATTN_SIMT, bad
    d = _attn_desc(L.PV_F16, 1, 2, 51, 51, 64, 384, (0, 0, 7), 128, 1)
    assert L.load().pv_attention_kernel_for(C.byref(d), 0x10000, 0x20000, 0x30000, 0x40000) == L.ATTN_WGMMA


def test_attention_routing_rejects_bad_arguments():
    from pytorchvideo_b200 import _lib as L
    assert _route(q=0) == -1
    d = _attn_desc(L.PV_F16, 0, 2, 51, 51, 64, 384, (1,) * 3, 128, 1)
    assert L.load().pv_attention_kernel_for(C.byref(d), 16, 16, 16, 16) == -1


# ---- CPU: the comparator has teeth ---------------------------------------------------------------------------------
def _mutation_case(seed=3):
    """A conv with residual whose output has 2 x 128-row M tiles and 2 N tiles of 64 channels."""
    g = torch.Generator().manual_seed(seed)
    N, Ci, T, H, W, Co, k = 1, 32, 2, 12, 12, 128, (1, 3, 3)
    x, w = _f16_operands(g, N, Ci, T, H, W, Co, k)
    scale = torch.rand(Co, generator=g) + 0.5
    bias = torch.rand(Co, generator=g) - 0.5
    res = TS.f16_exact(torch.randn(N, Co, T, H, W, generator=g))
    ref, absref = conv_ref64(x, w, scale, bias, (1, 1, 1), (0, 1, 1), (1, 1, 1), 1, None, res)
    return x, w, scale, bias, res, ref, absref, Ci * 9


def _rows(t):      # NCDHW -> [M, C] (the kernel's output rows)
    return t.permute(0, 2, 3, 4, 1).reshape(-1, t.shape[1])


def _unrows(r, like):
    N, Co, T, H, W = like.shape
    return r.reshape(N, T, H, W, Co).permute(0, 4, 1, 2, 3)


def test_comparator_accepts_the_f16_rounded_reference():
    *_, ref, absref, K = _mutation_case()
    TS.assert_close_to_f64(ref.half().double(), ref, absref, K)
    TS.assert_close_to_f64(ref.float().half().double(), ref, absref, K)


@pytest.mark.parametrize("mutation", ["drop_tap", "shift_channel", "zero_tile_last_row", "stale_n_tile",
                                      "round_toward_zero", "skip_residual_tile"])
def test_comparator_rejects_kernel_bugs(mutation):
    x, w, scale, bias, res, ref, absref, K = _mutation_case()
    if mutation == "drop_tap":
        w2 = w.clone()
        w2[:, :, :, 2, 1] = 0
        got = conv_ref64(x, w2, scale, bias, (1, 1, 1), (0, 1, 1), (1, 1, 1), 1, None, res)[0]
    elif mutation == "shift_channel":
        got = torch.roll(ref, 1, dims=1)
    elif mutation == "zero_tile_last_row":
        r = _rows(ref).clone()
        r[127] = 0
        got = _unrows(r, ref)
    elif mutation == "stale_n_tile":
        other = conv_ref64(_mutation_case(seed=4)[0], w, scale, bias, (1, 1, 1), (0, 1, 1), (1, 1, 1), 1, None, res)[0]
        got = ref.clone()
        got[:, 64:128] = other[:, 64:128]
    elif mutation == "round_toward_zero":
        h = ref.half().double()
        away = (h.abs() > ref.abs())                     # round-to-nearest went up in magnitude: step back one ulp
        bits = ref.half().view(torch.int16)
        got = torch.where(away, (bits - 1).view(torch.float16).double(), h)
    elif mutation == "skip_residual_tile":
        r = _rows(ref).clone()
        r[128:256] -= _rows(res.double())[128:256]
        got = _unrows(r, ref)
    with pytest.raises(AssertionError):
        TS.assert_close_to_f64(got.half().double() if mutation != "round_toward_zero" else got, ref, absref, K)


# ---- CPU: the fused block's comparator has teeth -------------------------------------------------------------------
# Two small cases with partial tiles and T = 5, each with thousands of normal-range outputs (so the bias check applies):
# stride 1 with the identity shortcut, and stride 2 with a projection shortcut.
FUSED_CPU_CASES = {
    "identity": (FB_RES2, 1, 5, 7, 9),
    "stride2_projection": (FB_RES3_0, 1, 5, 9, 7),
}
FUSED_CPU_CHUNK = 2          # frames per CTA of the emulated chunk-boundary bug
FUSED_CPU_TILE_H = 4         # tile rows of the emulated edge-tile bug (H_out = 7 / 5: the last tile row is partial)


def _h16(t):
    return t.half().float()


def fused_block_emulate(x, wa, wb, wc, ws, folds, kt, sb, act, mutation=None):
    """The kernel's rounding points on the CPU: fp32 accumulation and BatchNorm, a and b stored as f16, y rounded to
    f16.  `mutation` plants one kernel-specific bug (see test_fused_comparator_rejects_kernel_bugs)."""
    sa, ba, sbn, bbn, sc, bc, ssc, bsc = folds
    v = lambda t: t.view(1, -1, 1, 1, 1)
    pa = kt // 2
    x = x.float()
    T = x.shape[2]
    pad_b = (0, 1, 1)
    if mutation == "edge_frame_replicated":              # conv_a repeats the first / last frame instead of zeros
        a_pre = F.conv3d(F.pad(x, (0, 0, 0, 0, pa, pa), mode="replicate"), wa)
    elif mutation == "halo_a_bn0":                        # a = relu(bn_a(0)) outside the image instead of 0
        a_pre, pad_b = F.conv3d(F.pad(x, (1, 1, 1, 1)), wa, padding=(pa, 0, 0)), (0, 0, 0)
    else:
        a_pre = F.conv3d(x, wa, padding=(pa, 0, 0))
    a = _h16((a_pre * v(sa) + v(ba)).clamp_min(0))
    if mutation == "chunk_halo_zero":                    # a chunk's leading halo frame read as zeros
        for t0 in range(FUSED_CPU_CHUNK, T, FUSED_CPU_CHUNK):
            x2 = x.clone()
            x2[:, :, t0 - 1] = 0
            a[:, :, t0] = _h16((F.conv3d(x2, wa, padding=(pa, 0, 0)) * v(sa) + v(ba)).clamp_min(0))[:, :, t0]
    if mutation == "drop_conv_b_tap":                    # the last (dh, dw) = (2, 2) tap of conv_b skipped
        wb = wb.clone()
        wb[:, :, :, 2, 2] = 0
    b32 = (F.conv3d(a, wb, None, (1, sb, sb), pad_b) * v(sbn) + v(bbn)).clamp_min(0)
    b = _h16(b32)
    if mutation == "b_truncated":                        # b rounded toward zero instead of to nearest (b >= 0)
        bits = b32.half().view(torch.int16)
        b = torch.where(b > b32, (bits - 1).view(torch.float16), bits.view(torch.float16)).float()
    xs = x
    if mutation == "shortcut_prev_frame":                # the shortcut reads frame t-1 (ring slot off by one)
        xs = torch.cat([torch.zeros_like(x[:, :, :1]), x[:, :, :-1]], 2)
    if mutation == "stride2_shortcut_odd":               # the stride-2 shortcut samples 2i+1 instead of 2i
        xs = F.pad(x[:, :, :, 1:, 1:], (0, 1, 0, 1))
    xs = xs[:, :, :, ::sb, ::sb]
    short = xs if ws is None else F.conv3d(xs, ws) * v(ssc) + v(bsc)
    y = F.conv3d(b, wc) * v(sc) + v(bc) + short
    y = _h16(y.clamp_min(0) if act == "relu" else y)
    if mutation == "edge_tile_last_row":                 # the last row of the partial bottom tiles is not stored
        assert y.shape[3] % FUSED_CPU_TILE_H
        y[:, :, :, -1] = 0
    return y


def _fused_cpu_case(name, act):
    inst, N, T, H, W = FUSED_CPU_CASES[name]
    cin, cmid, cout, kt, s, proj = _fused_shape(inst)
    x, wa, wb, wc, ws, folds = _fused_operands(inst, N, T, H, W, seed=5)
    y, _, _, Y, prop = fused_block_ref64(x, wa, wb, wc, ws, folds, kt, s, act)
    assert int((y.abs() >= 2.0 ** -14).sum()) >= 256
    return inst, (x, wa, wb, wc, ws, folds, kt, s, act), y, Y, prop


@pytest.mark.parametrize("act", ["relu", None])
@pytest.mark.parametrize("case", sorted(FUSED_CPU_CASES))
def test_fused_comparator_accepts_the_kernel_rounding(case, act):
    inst, args, y, Y, prop = _fused_cpu_case(case, act)
    got = fused_block_emulate(*args)
    ratio = TS.assert_close_to_f64(got, y, Y, _fused_k(inst), what=case, extra64=prop)
    print("RATIO fused emulation %s %s %.4f %.4f %.4f" % (case, act, *ratio))


FUSED_MUTATIONS = ["halo_a_bn0", "edge_frame_replicated", "chunk_halo_zero", "shortcut_prev_frame",
                   "stride2_shortcut_odd", "drop_conv_b_tap", "b_truncated", "edge_tile_last_row"]


@pytest.mark.parametrize("case,mutation", [(c, m) for c in sorted(FUSED_CPU_CASES) for m in FUSED_MUTATIONS
                                           if not (c == "identity" and m == "stride2_shortcut_odd")])
def test_fused_comparator_rejects_kernel_bugs(case, mutation):
    inst, args, y, Y, prop = _fused_cpu_case(case, "relu")
    got = fused_block_emulate(*args, mutation=mutation)
    with pytest.raises(AssertionError):
        TS.assert_close_to_f64(got, y, Y, _fused_k(inst), what=case, extra64=prop)


# ---- CPU: the fused block's host checks and tile search ------------------------------------------------------------
def test_fused_supported_rejects_32_bit_output_offsets():
    """In-frame y offsets live in a 32-bit table: H_out * W_out * y_row_stride must stay below 2^31 even when the
    input frame (8 channels) is 4x smaller."""
    from pytorchvideo_b200 import _lib as L
    lib = L.load()
    big = _fused_desc(FB_RES2_0, 1, 4, 8192, 8192, xrs=8, yrs=32)
    assert 8192 * 8192 * 8 < 2 ** 31 <= 8192 * 8192 * 32
    assert lib.pv_bottleneck_fused_supported(C.byref(big)) == 0
    half = _fused_desc(FB_RES2_0, 1, 4, 8192, 4096, xrs=8, yrs=32)
    assert lib.pv_bottleneck_fused_supported(C.byref(half)) == 1
    wide = _fused_desc(FB_RES2_0, 1, 4, 4096, 4096, xrs=8, yrs=128)
    assert lib.pv_bottleneck_fused_supported(C.byref(wide)) == 0


@pytest.mark.parametrize("inst", [FB_RES2_0, FB_RES2])
@pytest.mark.parametrize("which", ["x", "y", "wa", "wb", "wc", "wsc"])
def test_fused_rejects_misaligned_pointers(inst, which):
    """Every pointer the kernel reads or writes 16 bytes at a time must be 16-byte aligned: PV_ERR_INVALID, decided
    before any CUDA call.  N = 0, so no call here can launch a kernel whatever the library decides."""
    from pytorchvideo_b200 import _lib as L
    lib = L.load()
    cin, cmid, cout, kt, s, proj = _fused_shape(inst)
    d = _fused_desc(inst, 0, 4, 8, 8)
    assert lib.pv_bottleneck_fused_supported(C.byref(d)) == 1
    ptrs = dict(x=0x10000, y=0x20000, wa=0x30000, wb=0x40000, wc=0x50000, wsc=0x60000 if proj else None)
    f32 = 0x70000

    def call(**kw):
        p = dict(ptrs, **kw)
        return lib.pv_bottleneck_fused_fwd(C.byref(d), p["x"], p["wa"], p["wb"], p["wc"], p["wsc"], f32, f32, f32,
                                           f32, f32, f32, f32 if proj else None, f32 if proj else None, p["y"], None)
    assert call() != -1, L.last_error()             # aligned: past the argument checks (no device, or N = 0: no launch)
    if which == "wsc" and not proj:
        assert call(wsc=0x60008) != -1               # the identity shortcut has no weights to check
        return
    for off in (8, 2):
        assert call(**{which: ptrs[which] + off}) == -1, (which, off)
        assert "aligned" in L.last_error()


# (TH, TW, TC) of the parent commit's tile search at 132 SMs (H100 SXM) for SlowFast-R50's Fast pathway at batch 8
FUSED_BENCH_TILINGS = {
    (FB_RES2_0, 56): (8, 14, 7),
    (FB_RES2, 56): (14, 14, 7),
    (FB_RES3_0, 56): (4, 8, 11),
    (FB_RES3, 28): (10, 14, 6),
}


def test_fused_tiling_pinned_bench_geometry():
    for (inst, hw), want in FUSED_BENCH_TILINGS.items():
        cin, cmid, cout, kt, s, proj = _fused_shape(inst)
        th, tw, tc, smem = fused_tiling(_fused_desc(inst, 8, 32, hw, hw), 132)
        assert (th, tw, tc) == want, (inst, hw, (th, tw, tc))
        assert 0 < smem <= 200 * 1024


def test_fused_tiling_rejects_bad_arguments():
    from pytorchvideo_b200 import _lib as L
    lib = L.load()
    th, tw, tc, smem = C.c_int(), C.c_int(), C.c_int(), C.c_longlong()
    d = _fused_desc(FB_RES2, 1, 4, 8, 8)
    assert lib.pv_bottleneck_fused_tiling(C.byref(d), 0, C.byref(th), C.byref(tw), C.byref(tc), C.byref(smem)) == -1
    bad = _fused_desc(FB_RES2, 1, 4, 8, 8, xrs=36)
    assert lib.pv_bottleneck_fused_tiling(C.byref(bad), 132, C.byref(th), C.byref(tw), C.byref(tc), C.byref(smem)) == -3


@pytest.mark.parametrize("sm_count", [132, 114])
def test_fused_row_claims_hold(sm_count):
    """On an H100 SXM (132 SMs) and PCIe (114 SMs) every fused row's claimed tiling property holds, and every
    batch-invariance row tiles a batch of 8 differently from one clip."""
    for row in FUSED_ROWS:
        inst, N, T, H, W, act, xe, ye, claims = row
        cin, cmid, cout, kt, s, proj = _fused_shape(inst)
        d = _fused_desc(inst, N, T, H, W, act, cin + xe, cout + ye)
        props = fused_tiling_properties(d, sm_count)
        assert set(claims) <= props, (_fused_row_id(row), claims, props, fused_tiling(d, sm_count))
    for inst in {r[0] for r in FUSED_ROWS}:
        for claim in (PH, PW, CH, SC):
            assert any(r[0] == inst and claim in r[8] for r in FUSED_ROWS), (inst, claim)
    for inst, T, H, W in FUSED_BATCH_ROWS:
        t8 = fused_tiling(_fused_desc(inst, 8, T, H, W), sm_count)[:3]
        t1 = fused_tiling(_fused_desc(inst, 1, T, H, W), sm_count)[:3]
        assert t8 != t1, (inst, T, H, W, t8)
