"""Grouped 3-D convolutions (ResNeXt-style conv_b group counts, CSN with several channels per group).

Grouped mode of the TMA-fed implicit GEMM (csrc/pv_igemm.cu): the output channels form group spans of
S = 64 / gcd(Cg, 64) groups whose input channels fill whole 64-channel boxes; each N tile reads only its own span and
multiplies it by block-diagonal weights.  Shapes grouped mode does not take run as the dense convolution with
block-diagonal weights (packing.expand_grouped_dense).

CPU: a float64 emulation of grouped mode (im2col + pack_grouped_tcgen05 + the span origin rule) equals F.conv3d, the
span / routing table of the C library, the host lowering of every grouped model case and the instance ledger.
GPU: kernel rows against float64 with the instance each must launch, a span-isolation test, and the grouped model
cases against the reference goldens.

Measured on an NVIDIA H100 80GB HBM3 (132 SMs, 400 W power limit): largest err / tol 0.987 over the grouped-mode rows,
the channel-slice row and the span-isolation rows, 0.988 over the f16 expansion rows, 0.074 for the f32 expansion row.
"""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.engine import packing as PK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorchvideo_b200", "csrc")
GOLD = os.path.join(ROOT, "tests", "golden")


def _dev():
    return torch.device("cuda:0")


def _out(i, k, s, p, d):
    return (i + 2 * p - d * (k - 1) - 1) // s + 1


def _desc(N, Ci, Co, groups, T, H, W, k=(1, 3, 3), s=(1, 1, 1), p=(0, 1, 1), dil=(1, 1, 1), dtype=L.PV_F16,
          ci_pad64=0, xrs=None):
    d = L.Conv3dDesc()
    d.dtype, d.N, d.Ti, d.Hi, d.Wi, d.Ci = dtype, N, T, H, W, Ci
    d.To, d.Ho, d.Wo = (_out(i, kk, ss, pp, dd) for i, kk, ss, pp, dd in zip((T, H, W), k, s, p, dil))
    d.Co = Co
    d.kt, d.kh, d.kw = k
    d.st, d.sh, d.sw = s
    d.pt, d.ph, d.pw = p
    d.dt, d.dh, d.dw = dil
    d.groups, d.act, d.has_residual = groups, L.ACT_RELU, 0
    d.x_row_stride, d.y_row_stride, d.ci_pad64 = xrs or Ci, Co, ci_pad64
    return d


# ---- CPU: float64 emulation of grouped mode -------------------------------------------------------------------------
def emulate_grouped(x, w, groups, stride, padding, dilation, block_n=64):
    """Grouped mode in float64: im2col of the input, the packed weights of pack_grouped_tcgen05, and every block_n-wide
    N tile reading K_span input channels from c0 = (n0 // N_span) * K_span, where (S, K_span, N_span) come from
    pv_conv3d_group_span.  Input channels past C_in read as zeros (TMA out-of-bounds fill of the last span)."""
    N, Ci, T, H, W = x.shape
    Co = w.shape[0]
    kt, kh, kw = w.shape[2:]
    taken, S, K, NS = L.group_span(_desc(N, Ci, Co, groups, T, H, W, (kt, kh, kw), stride, padding, dilation))
    assert K % 64 == 0 and NS % block_n == 0
    spans = -(-groups // S)
    xp = torch.zeros(N, spans * K, T, H, W, dtype=torch.float64)
    xp[:, :Ci] = x.double()
    xp = F.pad(xp, (padding[2], padding[2], padding[1], padding[1], padding[0], padding[0]))
    To, Ho, Wo = (_out(i, kk, s, p, d) for i, kk, s, p, d in zip((T, H, W), (kt, kh, kw), stride, padding, dilation))
    cols = []
    for it in range(kt):
        for ih in range(kh):
            for iw in range(kw):
                t0, h0, w0 = it * dilation[0], ih * dilation[1], iw * dilation[2]
                cols.append(xp[:, :, t0:t0 + (To - 1) * stride[0] + 1:stride[0], h0:h0 + (Ho - 1) * stride[1] + 1:stride[1],
                               w0:w0 + (Wo - 1) * stride[2] + 1:stride[2]])
    A = torch.stack(cols, 1).permute(0, 3, 4, 5, 1, 2).reshape(N * To * Ho * Wo, kt * kh * kw, spans * K)
    B = PK.pack_grouped_tcgen05(w, groups, S, K).double().view(Co, kt * kh * kw, K)
    y = torch.zeros(N * To * Ho * Wo, Co, dtype=torch.float64)
    for n0 in range(0, Co, block_n):
        c0 = (n0 // NS) * K
        a = A[:, :, c0:c0 + K].reshape(A.shape[0], -1)
        y[:, n0:n0 + block_n] = a @ B[n0:n0 + block_n].reshape(min(block_n, Co - n0), -1).t()
    return y.view(N, To, Ho, Wo, Co).permute(0, 4, 1, 2, 3), taken


EMU_CASES = [
    # (C, Cg, kernel, stride, padding, dilation, block_n)
    (128, 2, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), 64),
    (128, 4, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), 64),
    (256, 8, (3, 3, 3), (2, 2, 2), (1, 1, 1), (1, 1, 1), 64),
    (256, 16, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1), 64),
    (384, 24, (1, 3, 3), (1, 1, 1), (0, 2, 2), (1, 2, 2), 64),     # S = 8, span width 192: three boxes per span
    (256, 32, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), 64),
    (256, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 64),
    (256, 128, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), 128),
    (512, 128, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 64),    # two N tiles per span
    (96, 8, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), 64),       # partial last span: 4 of 8 groups
    (320, 16, (3, 3, 3), (1, 1, 1), (1, 1, 1), (1, 1, 1), 64),     # 5 spans
]


@pytest.mark.parametrize("case", EMU_CASES, ids=["C%d-Cg%d-k%s" % (c[0], c[1], "".join(map(str, c[2]))) for c in EMU_CASES])
def test_grouped_mode_emulation_matches_conv3d(case):
    Cc, cg, k, s, p, dil, bn = case
    g = torch.Generator().manual_seed(Cc + cg)
    x = TS.f16_exact(torch.randn(2, Cc, 3, 7, 6, generator=g))
    w = TS.f16_exact(torch.randn(Cc, cg, *k, generator=g))
    ref = F.conv3d(x.double(), w.double(), None, s, p, dil, Cc // cg)
    got, taken = emulate_grouped(x, w, Cc // cg, s, p, dil, bn)
    assert taken
    assert torch.allclose(got, ref, rtol=0, atol=1e-9 * float(ref.abs().max())), float((got - ref).abs().max())


def test_grouped_mode_emulation_detects_a_wrong_span_origin():
    """The emulation is not vacuous: reading the first span for every tile (c0 = 0) disagrees with F.conv3d."""
    g = torch.Generator().manual_seed(3)
    x = TS.f16_exact(torch.randn(1, 128, 2, 5, 5, generator=g))
    w = TS.f16_exact(torch.randn(128, 8, 1, 3, 3, generator=g))
    ref = F.conv3d(x.double(), w.double(), None, 1, (0, 1, 1), 1, 16)
    x_bad = x.clone()
    x_bad[:, 64:] = x[:, :64]            # what a tile of span 1 would see with c0 = 0
    bad, _ = emulate_grouped(x_bad, w, 16, (1, 1, 1), (0, 1, 1), (1, 1, 1))
    assert not torch.allclose(bad[:, 64:], ref[:, 64:], atol=1e-3)


def test_grouped_packing_layout():
    w = torch.randn(96, 8, 1, 3, 3)
    t = PK.pack_grouped_tcgen05(w, 12, 8, 64)
    assert t.shape == (96, 9 * 64) and t.dtype == torch.float16
    # group 9 (channels 72..79) is the 2nd group of span 1: input offset 8
    assert t[75, 4 * 64 + 8 + 3] == w[75, 3, 0, 1, 1].half()
    row = t[75].view(9, 64)
    assert float(row[:, :8].abs().sum()) == 0 and float(row[:, 16:].abs().sum()) == 0
    dense = PK.expand_grouped_dense(w, 12)
    assert dense.shape == (96, 96, 1, 3, 3)
    x = torch.randn(1, 96, 2, 5, 5)
    assert torch.allclose(F.conv3d(x, dense, padding=(0, 1, 1)), F.conv3d(x, w, padding=(0, 1, 1), groups=12), atol=1e-5)


# ---- CPU: span and routing table ------------------------------------------------------------------------------------
SPAN_TABLE = [
    # (Ci, Co, groups, dtype, taken, span_groups, span_k, span_n)
    (128, 128, 32, L.PV_F16, True, 16, 64, 64),       # slow_r50 res3, 4 channels per group: 2 spans
    (256, 256, 32, L.PV_F16, True, 8, 64, 64),
    (512, 512, 32, L.PV_F16, True, 4, 64, 64),
    (128, 128, 16, L.PV_F16, True, 8, 64, 64),        # CSN width 8
    (384, 384, 16, L.PV_F16, True, 8, 192, 192),      # Cg 24
    (256, 256, 2, L.PV_F16, True, 1, 128, 128),       # Cg 128
    (96, 96, 12, L.PV_F16, True, 8, 64, 64),          # partial last span
    (64, 64, 32, L.PV_F16, False, 32, 64, 64),        # one span: dense expansion
    (64, 64, 8, L.PV_F16, False, 8, 64, 64),
    (128, 128, 1, L.PV_F16, False, 0, 0, 0),          # dense: no span
    (128, 128, 128, L.PV_F16, False, 64, 64, 64),     # depthwise
    (128, 256, 16, L.PV_F16, False, 8, 64, 128),      # non-square groups
    (256, 128, 16, L.PV_F16, False, 4, 64, 32),
    (128, 128, 32, L.PV_F32, False, 16, 64, 64),      # f32
    (120, 120, 10, L.PV_F16, False, 16, 192, 192),    # Cg 12: one span of 120 channels
    (132, 132, 12, L.PV_F16, False, 64, 704, 704),    # C % 8 != 0
    (128, 128, 3, L.PV_F16, False, 0, 0, 0),          # groups does not divide C
]


@pytest.mark.parametrize("row", SPAN_TABLE, ids=["%d-%d-g%d-%s" % (r[0], r[1], r[2], "f16" if r[3] == 0 else "f32")
                                                 for r in SPAN_TABLE])
def test_group_span_and_routing_table(row):
    ci, co, groups, dtype, taken, sg, sk, sn = row
    lib = L.load()
    d = _desc(2, ci, co, groups, 4, 14, 14, dtype=dtype)
    got = L.group_span(d)
    assert got == (taken, sg, sk, sn), got
    d.ci_pad64 = sk
    expect = 1 if taken else 0
    assert lib.pv_conv3d_tcgen05_supported(C.byref(d)) == expect
    if taken:
        # the packed-weight width must be the span width; stems, odd strides and too many taps are declined as in
        # dense mode
        d.ci_pad64 = sk + 64
        assert lib.pv_conv3d_tcgen05_supported(C.byref(d)) == 0 and L.group_span(d)[0]
        for kw_ in ({"xrs": ci + 4}, {"k": (5, 5, 5), "p": (2, 2, 2)}, {"s": (3, 3, 1)}):
            assert not L.group_span(_desc(2, ci, co, groups, 8, 14, 14, **kw_))[0], kw_


def test_depthwise_descriptors_stay_off_the_tensor_cores():
    lib = L.load()
    for c in (24, 64, 128, 432):
        for pad in (c, 64 * ((c + 63) // 64)):
            d = _desc(1, c, c, c, 4, 9, 9, ci_pad64=pad)
            assert lib.pv_conv3d_tcgen05_supported(C.byref(d)) == 0
            assert L.group_span(d)[0] is False


def test_direct_algo_refuses_grouped_descriptors():
    """PV_ALGO_DIRECT on a grouped, non-depthwise descriptor returns PV_ERR_UNSUPPORTED before any CUDA call (the
    pointers are never touched); groups that do not divide the channels are PV_ERR_INVALID."""
    lib = L.load()
    fake = [0x10000 * (i + 1) for i in range(5)]
    for ci, co, groups in ((128, 128, 32), (64, 64, 8), (128, 256, 16)):
        d = _desc(1, ci, co, groups, 4, 9, 9)
        rc = lib.pv_conv3d_fwd(C.byref(d), L.ALGO_DIRECT, fake[0], fake[1], fake[2], fake[3], None, fake[4], None)
        assert rc == -3, (ci, co, groups, rc, L.last_error())
    d = _desc(1, 128, 128, 3, 4, 9, 9)
    assert lib.pv_conv3d_fwd(C.byref(d), L.ALGO_DIRECT, fake[0], fake[1], fake[2], fake[3], None, fake[4], None) == -1


# ---- CPU: host lowering of the grouped model cases ------------------------------------------------------------------
# (grouped-mode convolutions, convolutions expanded to dense)
GROUPED_LOWERING = {
    "slow_r50_g32": (13, 3),        # res2 (64 channels, 2 per group) is one span
    "csn_r101_w8": (30, 3),
    "slowfast_r50_g": (13, 3 + 16),  # + every Fast-pathway conv_b (8-64 channels, one span)
    "slow_r50_g32_f16w": (13, 3),
}


@pytest.mark.parametrize("case", sorted(TS.GROUPED_MODEL_CASES))
def test_grouped_model_case_lowers_on_the_host(case):
    import pytorchvideo_b200.models.hub as PH
    from pytorchvideo_b200.engine.lower import lower_only
    hub, kw, B, T, H, W, is_sf, _ = TS.GROUPED_MODEL_CASES[case]
    m = getattr(PH, hub)(**kw).eval()
    clip = torch.zeros(B, 3, T, H, W)
    plan, out_shape = lower_only(m, TS.slowfast_inputs(clip) if is_sf else clip)
    assert out_shape == (B, 400)
    n_grouped, n_expanded = GROUPED_LOWERING[case]
    mods = [mod for mod in m.modules() if isinstance(mod, torch.nn.Conv3d) and mod.groups > 1]
    assert len(mods) == n_grouped + n_expanded
    assert plan.stats.get("grouped", 0) == n_grouped
    assert plan.stats["depthwise"] == 0
    assert plan.stats["direct"] <= 1
    assert plan.stats.get("fused_block", 0) == 0    # the fused Fast-pathway block kernel is dense only


def test_grouped_convs_expand_in_f32_mode():
    import pytorchvideo_b200.models.hub as PH
    from pytorchvideo_b200.engine.lower import lower_only
    m = PH.slow_r50(stage_conv_b_num_groups=(32,) * 4).eval()
    plan, out_shape = lower_only(m, torch.zeros(1, 3, 8, 224, 224), dtype="f32")
    assert out_shape == (1, 400) and plan.stats.get("grouped", 0) == 0 and plan.stats["tcgen05"] == 0


# ---- CPU: instance ledger -------------------------------------------------------------------------------------------
def grouped_instances():
    src = open(os.path.join(CSRC, "pv_igemm.cu")).read()
    return {"conv3d_igemm_grouped_kernel<%s,%s>" % a for a in re.findall(r"PV_IG_GROUPED_LAUNCH\((\d+), (\d+)\)", src)}


def test_grouped_instance_ledger():
    src = open(os.path.join(CSRC, "pv_igemm.cu")).read()
    assert '"conv3d_igemm_grouped_kernel<" #BN "," #KB ">"' in src
    assert grouped_instances() == {"conv3d_igemm_grouped_kernel<64,128>", "conv3d_igemm_grouped_kernel<128,128>"}
    assert grouped_instances() <= {r[0] for r in GROUPED_ROWS}


# ---- GPU: kernel rows -----------------------------------------------------------------------------------------------
def _act64(y, act):
    if act in (None, "none"):
        return y
    if act == "relu":
        return y.clamp_min(0)
    if act == "swish":
        return y * torch.sigmoid(y)
    if act == "gelu":
        return 0.5 * y * (1 + torch.erf(y / math.sqrt(2.0)))
    if act == "sigmoid":
        return torch.sigmoid(y)
    raise ValueError(act)


def _bn(c, seed):
    g = torch.Generator().manual_seed(seed)
    bn = torch.nn.BatchNorm3d(c).eval()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.rand(c, generator=g) - 0.5)
        bn.running_mean.copy_(torch.rand(c, generator=g) - 0.5)
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn


def conv_ref64(x, w, scale, bias, stride, padding, dilation, groups, act, res):
    x64, w64 = x.double(), w.double()
    sc, bi = scale.double().view(1, -1, 1, 1, 1), bias.double().view(1, -1, 1, 1, 1)
    y = F.conv3d(x64, w64, None, stride, padding, dilation, groups) * sc + bi
    a = F.conv3d(x64.abs(), w64.abs(), None, stride, padding, dilation, groups) * sc.abs() + bi.abs()
    if res is not None:
        y = y + res.double()
        a = a + res.double().abs()
    return _act64(y, act), a


# (expected instance, N, C_in, C_out, groups, T, H, W, kernel, stride, padding, dilation, act, residual)
# Grouped mode picks BLOCK_N from {64, 128} dividing the span width by the dense cost model: spans of 64 channels
# always take 64; 128-channel spans take 128 from a few hundred 128-row tiles on (on 114 and 132 SMs alike).
GROUPED_ROWS = [
    ("conv3d_igemm_grouped_kernel<64,128>", 1, 128, 128, 32, 4, 14, 14, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), "relu", False),
    ("conv3d_igemm_grouped_kernel<64,128>", 2, 256, 256, 32, 3, 15, 13, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), "swish", True),
    ("conv3d_igemm_grouped_kernel<64,128>", 1, 128, 128, 16, 5, 9, 9, (3, 3, 3), (2, 2, 2), (1, 1, 1), (1, 1, 1), "gelu", False),
    ("conv3d_igemm_grouped_kernel<64,128>", 1, 512, 512, 32, 1, 7, 7, (1, 3, 3), (1, 1, 1), (0, 2, 2), (1, 2, 2), "sigmoid", False),
    ("conv3d_igemm_grouped_kernel<64,128>", 2, 96, 96, 12, 4, 6, 6, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1), None, True),
    # tiles that cross samples: 5x5 planes, T = 2, N = 4 -> a 128-row box holds several clips
    ("conv3d_igemm_grouped_kernel<64,128>", 4, 256, 256, 16, 2, 5, 5, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), "relu", True),
    ("conv3d_igemm_grouped_kernel<64,128>", 1, 384, 384, 16, 2, 8, 8, (3, 3, 3), (1, 1, 1), (1, 1, 1), (1, 1, 1), "relu", False),
    ("conv3d_igemm_grouped_kernel<64,128>", 2, 512, 512, 2, 4, 14, 14, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), None, False),
    ("conv3d_igemm_grouped_kernel<128,128>", 4, 256, 256, 2, 8, 28, 28, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), "relu", True),
    ("conv3d_igemm_grouped_kernel<128,128>", 2, 512, 512, 2, 8, 28, 28, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), "swish", False),
]

# what grouped mode does not take runs as the dense convolution of the block-diagonal weights
EXPANDED_ROWS = [
    # one span (slow_r50 res2, SlowFast Fast pathway)
    ("conv3d_igemm_kernel<64,128>", 1, 64, 64, 32, 4, 14, 14, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), "relu", False, "f16"),
    # non-square groups
    ("conv3d_igemm_kernel<", 1, 128, 256, 16, 2, 9, 9, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), None, False, "f16"),
    # f32 storage
    ("conv3d_direct_kernel<float>", 1, 128, 128, 32, 2, 9, 9, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), "relu", True, "f32"),
]


def _gid(r):
    return "%s-%s" % (r[0], "x".join(str(v) for v in r[1:8]))


def _grouped_operands(row, seed):
    _, N, ci, co, groups, T, H, W, k = row[:9]
    g = torch.Generator().manual_seed(seed)
    x = TS.f16_exact(torch.randn(N, ci, T, H, W, generator=g))
    fan = ci // groups * int(np.prod(k))
    w = TS.f16_exact(torch.randn(co, ci // groups, *k, generator=g) * (2.0 / fan) ** 0.5)
    return x, w, g


def _check_row(row, got, ref, absref, launched, family):
    name, ci, groups, k = row[0], row[2], row[4], row[8]
    assert any(n.startswith(name) for n in launched), "expected %s, launched %s" % (name, launched)
    ratio = TS.assert_close_to_f64(got, ref, absref, ci // groups * int(np.prod(k)), what=name)
    print("RATIO %s %s %.4f %.4f %s" % (family, _gid(row), ratio[0], ratio[1], sorted(launched)))


@pytest.mark.gpu
@pytest.mark.parametrize("row", GROUPED_ROWS, ids=[_gid(r) for r in GROUPED_ROWS])
def test_grouped_instance(row):
    from pytorchvideo_b200 import ops
    name, N, ci, co, groups, T, H, W, k, s, p, dil, act, use_res = row
    x, w, g = _grouped_operands(row, N * 1000 + ci + groups + T + H)
    bn = _bn(co, co + groups)
    scale, bias = PK.fold_bn(None, bn, co, co)
    res = None
    if use_res:
        shape = F.conv3d(x, w, None, s, p, dil, groups).shape
        res = TS.f16_exact(torch.randn(shape, generator=g))
    ref, absref = conv_ref64(x, w, scale, bias, s, p, dil, groups, act, res)
    (got, stats), launched = TS.launched_kernels(
        ops.conv3d_bn_act, x.to(_dev()), w, None, bn, s, p, dil, groups, act, None if res is None else res.to(_dev()), "f16")
    assert stats.get("grouped") == 1 and launched.get(name) == 1, (stats, launched)
    assert not any(n.startswith(("conv3d_igemm_kernel<", "conv3d_direct_kernel")) for n in launched), launched
    _check_row(row, got, ref, absref, launched, "grouped")


@pytest.mark.gpu
@pytest.mark.parametrize("row", EXPANDED_ROWS, ids=[_gid(r) + "-" + r[-1] for r in EXPANDED_ROWS])
def test_grouped_expansion_instance(row):
    from pytorchvideo_b200 import ops
    name, N, ci, co, groups, T, H, W, k, s, p, dil, act, use_res, dtype = row
    x, w, g = _grouped_operands(row, 77 + ci + co)
    bn = _bn(co, co)
    scale, bias = PK.fold_bn(None, bn, co, co)
    res = None
    if use_res:
        res = TS.f16_exact(torch.randn(F.conv3d(x, w, None, s, p, dil, groups).shape, generator=g))
    ref, absref = conv_ref64(x, w, scale, bias, s, p, dil, groups, act, res)
    (got, stats), launched = TS.launched_kernels(
        ops.conv3d_bn_act, x.to(_dev()), w, None, bn, s, p, dil, groups, act, None if res is None else res.to(_dev()), dtype)
    assert "grouped" not in stats and not any("grouped" in n for n in launched), (stats, launched)
    if dtype == "f32":
        # f32 storage: one fp32 rounding of the result plus the accumulation term of assert_close_to_f64
        assert any(n.startswith(name) for n in launched), launched
        ratio = TS.assert_close_to_f64(got, ref, absref, ci // groups * int(np.prod(k)), what=name, rnd_eps=TS.F32_EPS)
        print("RATIO expanded %s-f32 %.4f %s" % (_gid(row), ratio[0], sorted(launched)))
        return
    _check_row(row, got, ref, absref, launched, "expanded")


@pytest.mark.gpu
def test_grouped_input_channel_slice():
    """The input is a channel slice (offset 16) of a wider buffer: the span origin is relative to the slice."""
    from pytorchvideo_b200.engine.plan import Plan, channel_slice
    row = ("conv3d_igemm_grouped_kernel<64,128>", 2, 256, 256, 16, 3, 10, 10, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1),
           "relu", False)
    _, N, ci, co, groups, T, H, W, k, s, p, dil, act, _ = row
    x, w, g = _grouped_operands(row, 5)
    wide = TS.f16_exact(torch.randn(N, ci + 48, T, H, W, generator=g))
    wide[:, 16:16 + ci] = x
    bn = _bn(co, 3)
    scale, bias = PK.fold_bn(None, bn, co, co)
    ref, absref = conv_ref64(x, w, scale, bias, s, p, dil, groups, act, None)

    def run():
        plan = Plan(_dev(), L.PV_F16)
        src = wide.to(_dev()).contiguous()
        xr = plan.emit_input_ncdhw(src, ci + 48, ci + 48)
        plan.materialize_input(xr)
        xs = channel_slice(xr, 16, ci)
        y = plan.emit_conv(xs, w, None, bn, s, p, dil, groups, L.ACT_RELU, None, "conv")
        out, shape = plan.emit_to_ncdhw(y)
        plan.finalize()
        plan.run(torch.cuda.current_stream(_dev()).cuda_stream)
        torch.cuda.synchronize(_dev())
        assert plan.stats.get("grouped") == 1, plan.stats
        return out.tensor[: int(np.prod(shape))].view(*shape).clone()
    got, launched = TS.launched_kernels(run)
    _check_row(row, got, ref, absref, launched, "grouped")


@pytest.mark.gpu
@pytest.mark.parametrize("poison_span", [0, 1, 3])
def test_grouped_span_isolation(poison_span):
    """Fill the input channels of one span with +-inf: every output channel of the other spans stays finite and
    matches float64.  A tile reading from the wrong span origin would multiply those infinities (even by a zero
    weight, giving NaN).  224 channels in 28 groups of 8 make 4 spans of 64 channels; the last holds 4 of its 8
    groups."""
    from pytorchvideo_b200 import ops
    ci = co = 224
    groups = 28                          # Cg 8: spans of 64 channels, the 4th holds 32 channels
    k, s, p, dil = (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1)
    g = torch.Generator().manual_seed(11 + poison_span)
    x = TS.f16_exact(torch.randn(2, ci, 3, 9, 9, generator=g))
    w = TS.f16_exact(torch.randn(co, ci // groups, *k, generator=g) * (2.0 / 72) ** 0.5)
    lo, hi = 64 * poison_span, min(64 * (poison_span + 1), ci)
    sign = torch.where(torch.rand(x[:, lo:hi].shape, generator=g) < 0.5, -1.0, 1.0)
    x[:, lo:hi] = sign * float("inf")
    bn = _bn(co, 9)
    scale, bias = PK.fold_bn(None, bn, co, co)
    keep = [c for c in range(co) if not lo <= c < hi]
    clean = x.clone()
    clean[:, lo:hi] = 0
    ref, absref = conv_ref64(clean, w, scale, bias, s, p, dil, groups, "relu", None)
    (got, stats), launched = TS.launched_kernels(ops.conv3d_bn_act, x.to(_dev()), w, None, bn, s, p, dil, groups, "relu",
                                                 None, "f16")
    assert launched.get("conv3d_igemm_grouped_kernel<64,128>") == 1, launched
    got = got.cpu()
    assert bool(torch.isfinite(got[:, keep]).all()), "non-finite outputs outside the poisoned span"
    ratio = TS.assert_close_to_f64(got[:, keep], ref[:, keep], absref[:, keep], 8 * 9, what="span isolation")
    print("RATIO span_isolation %d %.4f %.4f" % (poison_span, ratio[0], ratio[1]))


# ---- GPU: model cases -----------------------------------------------------------------------------------------------
# (min fraction of logits inside rtol 1e-3 / atol 1e-4 * max(1, max|ref|), max |d| / max|ref|), in the shape of
# test_gpu_models.F16_BOUNDS.  Measured on an NVIDIA H100 80GB HBM3 (132 SMs, 400 W power limit): slow_r50_g32 0.873 /
# 7.8e-4, csn_r101_w8 0.882 / 5.2e-4, slowfast_r50_g 0.882 / 6.1e-4, slow_r50_g32_f16w 0.985 / 4.5e-4; the bounds keep a
# small margin.  Arbitrary fp32 weights lose their f16 rounding in the engine; the f16w case multiplies identical
# operands on both sides and has the tight bound.
GROUPED_F16_BOUNDS = {
    "slow_r50_g32": (0.85, 1.0e-3),
    "csn_r101_w8": (0.86, 7e-4),
    "slowfast_r50_g": (0.86, 8e-4),
    "slow_r50_g32_f16w": (0.97, 6e-4),
}


def _setup_grouped(case):
    import pytorchvideo_b200.models.hub as PH
    g = torch.load(os.path.join(GOLD, "model_grouped_%s.pt" % case), weights_only=False)
    model, inp, is_sf = TS.build_grouped_case(case, PH, weight_seed=g["weight_seed"], input_seed=g["input_seed"])
    assert abs(TS.state_checksum(model) - g["state_checksum"]) <= 1e-6 * abs(g["state_checksum"]), "weights differ"
    return g, model, inp


def _to_dev(inp):
    return [t.cuda() for t in inp] if isinstance(inp, list) else inp.cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GROUPED_F16_BOUNDS))
def test_grouped_model_f16(case):
    g, model, inp = _setup_grouped(case)
    ref = g["output"]
    model.cuda()
    try:
        out, launched = TS.launched_kernels(lambda: model(_to_dev(inp)).float().cpu())
        out2 = model(_to_dev(inp)).float().cpu()
    finally:
        model.cpu()
    assert torch.equal(out, out2)
    assert out.shape == ref.shape
    assert any(n.startswith("conv3d_igemm_grouped_kernel<") for n in launched), launched
    scale = float(ref.abs().max())
    err = (out - ref).abs()
    inside = float((err <= 1e-3 * ref.abs() + 1e-4 * max(1.0, scale)).float().mean())
    rel = float(err.max()) / scale
    print("PARITY grouped %s f16: max|d|/max|ref| = %.3e, fraction within rtol1e-3/atol1e-4 = %.3f" % (case, rel, inside))
    lo, hi = GROUPED_F16_BOUNDS[case]
    assert rel <= hi, "max|d|/max|ref| = %.3e > %.1e" % (rel, hi)
    assert inside >= lo, "only %.3f of the logits inside the band (floor %.2f)" % (inside, lo)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GROUPED_F16_BOUNDS))
def test_grouped_model_f32_parity_mode(case):
    from pytorchvideo_b200 import config
    g, model, inp = _setup_grouped(case)
    ref = g["output"]
    config.set_precision("f32")
    try:
        model.cuda()
        out = model(_to_dev(inp)).float().cpu()
    finally:
        config.set_precision("f16")
        model.cpu()
    scale = max(1.0, float(ref.abs().max()))
    err = (out - ref).abs()
    print("PARITY grouped %s f32: max|d|/scale = %.3e" % (case, float(err.max()) / scale))
    assert out.shape == ref.shape
    assert bool((err <= 1e-3 * ref.abs() + 1e-4 * scale).all()), "max err %.3e (scale %.3g)" % (float(err.max()), scale)


@pytest.mark.gpu
def test_grouped_model_batch_split():
    """f(batch)[i] == f(batch[i:i+1]) on slow_r50_g32_f16w: the batch-2 and batch-1 plans tile differently."""
    _, model, inp = _setup_grouped("slow_r50_g32_f16w")
    model.cuda()
    try:
        full = model(inp.cuda()).float().cpu()
        for i in range(inp.shape[0]):
            one = model(inp[i:i + 1].cuda()).float().cpu()
            assert torch.equal(one, full[i:i + 1]), float((one - full[i:i + 1]).abs().max())
    finally:
        model.cpu()
