"""Temporal-streaming stem (csrc/pv_stem_stream.cu): float64 reference per instance, edge cases of the frame walk and
the W tiles through direct library calls, channel-slice output, batch invariance, routing and the instance ledger.

The kernel sums the five temporal taps in fp32 and rounds once, so on its own (direct calls, BN and activation in
its epilogue) it is held to the unrelaxed accumulation bound (testing.ACC_EPS).  Through the plan it writes the pre-BN
sum and pv_temporal_tap_sum applies BN and the activation: one f16 rounding more, the allowance of the factored row of
the kernel matrix.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pytorchvideo_b200 import testing as TS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorchvideo_b200", "csrc")
INSTANCE = "conv3d_stem_stream_kernel<5,2>"
K, S, P = (5, 7, 7), (1, 2, 2), (2, 3, 3)      # the SlowFast Fast stem


def _ref64(x, w, scale, bias, act):
    x64, w64 = x.double(), w.double()
    sc, bi = scale.double().view(1, -1, 1, 1, 1), bias.double().view(1, -1, 1, 1, 1)
    y = F.conv3d(x64, w64, None, S, P) * sc + bi
    a = F.conv3d(x64.abs(), w64.abs(), None, S, P) * sc.abs() + bi.abs()
    return (y.clamp_min(0) if act == "relu" else y), a


def _operands(N, T, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = TS.f16_exact(torch.randn(N, 3, T, H, W, generator=g))
    w = TS.f16_exact(torch.randn(8, 3, *K, generator=g) * (2.0 / (3 * 245)) ** 0.5)
    scale = (torch.rand(8, generator=g) + 0.5).float()
    bias = (torch.rand(8, generator=g) - 0.5).float()
    return x, w, scale, bias


def _stream_direct(x, w, scale, bias, act, y_row_stride=8, y_ch_off=0):
    """One pv_conv3d_stem_stream_fwd call on x [N, 3, T, H, W] -> (NDHWC f16 output buffer of row stride
    ``y_row_stride`` (sentinel-filled, the result at channel ``y_ch_off``), NCDHW fp32 result, launched instances)."""
    from pytorchvideo_b200 import _lib as L
    from pytorchvideo_b200.engine import packing as PK
    from pytorchvideo_b200.engine.plan import Plan, TRef, _conv_out
    dev = torch.device("cuda:0")
    N, _, T, H, W = x.shape
    To, Ho, Wo = (_conv_out(i, k, s, p, 1) for i, k, s, p in zip((T, H, W), K, S, P))
    plan = Plan(dev)
    xr = TRef(None, N, T, H, W, 3, Cp=4)
    wp, w_phys, lead, win = Plan._stem_window(xr, K[2], S[2], P[2], Wo)
    d = plan._conv_desc(xr, (To, Ho, Wo), 8, K, S, P, (1, 1, 1), 1, L.ACT_RELU if act == "relu" else L.ACT_NONE,
                        None, y_row_stride, win)
    d.x_w_pad, d.x_w_phys = wp, w_phys
    assert L.load().pv_conv3d_stem_stream_supported(C.byref(d)), (N, T, H, W)
    xp = torch.zeros(N * T * H * w_phys * 4 + 64 * 4, dtype=torch.float16)
    xp[: N * T * H * w_phys * 4].view(N, T, H, w_phys, 4)[:, :, :, wp:wp + W, :3] = x.permute(0, 2, 3, 4, 1).half()
    xp = xp.to(dev)
    wd = PK.pack_stem_stream(w, 4, 8, lead).to(dev)
    sd, bd = scale.to(dev), bias.to(dev)
    zero_row = torch.zeros(4096, dtype=torch.float16, device=dev)
    y = torch.full((N * To * Ho * Wo, y_row_stride), 7.0, dtype=torch.float16, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    before = TS.kernel_counts()
    L.check(L.load().pv_conv3d_stem_stream_fwd(C.byref(d), xp.data_ptr(), wd.data_ptr(), sd.data_ptr(), bd.data_ptr(),
                                               zero_row.data_ptr(), y.data_ptr() + 2 * y_ch_off, stream),
            "pv_conv3d_stem_stream_fwd")
    torch.cuda.synchronize(dev)
    launched = TS.kernel_count_diff(before, TS.kernel_counts())
    out = y[:, y_ch_off:y_ch_off + 8].float().view(N, To, Ho, Wo, 8).permute(0, 4, 1, 2, 3).cpu()
    return y.cpu(), out, launched


# (N, T, H, W, act): fewer frames than the 5 taps, exactly 5, just over; Wo < 128 and two W tiles (W = 300);
# a single unit and fewer units than SMs; and more rows than SMs, so a CTA walks several units in turn
DIRECT_ROWS = [
    (1, 1, 10, 20, "relu"),
    (1, 2, 12, 300, None),
    (2, 4, 16, 40, "relu"),
    (1, 5, 9, 64, None),
    (3, 6, 14, 30, "relu"),
    (2, 6, 160, 60, None),
]


@pytest.mark.gpu
@pytest.mark.parametrize("row", DIRECT_ROWS, ids=["x".join(str(v) for v in r) for r in DIRECT_ROWS])
def test_stem_stream_direct(row):
    N, T, H, W, act = row
    x, w, scale, bias = _operands(N, T, H, W, seed=N * 100 + T * 10 + H + W)
    ref, absref = _ref64(x, w, scale, bias, act)
    _, got, launched = _stream_direct(x, w, scale, bias, act)
    assert launched == {INSTANCE: 1}, launched
    ratio = TS.assert_close_to_f64(got, ref, absref, 3 * int(np.prod(K)), acc_eps=TS.ACC_EPS, what=INSTANCE)
    print("RATIO stem_stream %s %.4f %.4f" % (row, ratio[0], ratio[1]))


@pytest.mark.gpu
def test_stem_stream_writes_only_its_channel_slice():
    x, w, scale, bias = _operands(2, 6, 12, 36, seed=3)
    ref, absref = _ref64(x, w, scale, bias, "relu")
    y, got, launched = _stream_direct(x, w, scale, bias, "relu", y_row_stride=24, y_ch_off=8)
    assert launched == {INSTANCE: 1}, launched
    TS.assert_close_to_f64(got, ref, absref, 3 * int(np.prod(K)), acc_eps=TS.ACC_EPS, what=INSTANCE)
    outside = torch.cat([y[:, :8], y[:, 16:]], 1)
    assert bool((outside == 7.0).all()), "stem stream kernel wrote outside its channel slice"


@pytest.mark.gpu
def test_stem_stream_batch_invariance():
    x, w, scale, bias = _operands(8, 6, 32, 48, seed=11)
    _, full, _ = _stream_direct(x, w, scale, bias, "relu")
    for i in (0, 5, 7):
        _, one, _ = _stream_direct(x[i:i + 1].contiguous(), w, scale, bias, "relu")
        assert torch.equal(full[i:i + 1], one), i


@pytest.mark.gpu
def test_stem_stream_through_the_plan():
    """A Fast-stem shape with a full wave of output rows (N = 2, 224^2: 224 rows) takes the stream route: the stream
    kernel, then the BN / activation pass of pv_temporal_tap_sum over its pre-BN sum."""
    from pytorchvideo_b200 import ops
    x, w, _, _ = _operands(2, 8, 224, 224, seed=5)
    bn = torch.nn.BatchNorm3d(8).eval()
    g = torch.Generator().manual_seed(6)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(8, generator=g) + 0.5)
        bn.bias.copy_(torch.rand(8, generator=g) - 0.5)
        bn.running_mean.copy_(torch.rand(8, generator=g) - 0.5)
        bn.running_var.copy_(torch.rand(8, generator=g) + 0.5)
    from pytorchvideo_b200.engine import packing as PK
    scale, bias = PK.fold_bn(None, bn, 8, 8)
    ref, absref = _ref64(x, w, scale, bias, "relu")
    (got, stats), launched = TS.launched_kernels(ops.conv3d_bn_act, x.cuda(), w, None, bn, S, P, (1, 1, 1), 1, "relu",
                                                 None, "f16")
    assert launched.get(INSTANCE) == 1 and launched.get("temporal_tap_sum_kernel") == 1, launched
    assert not any(k.startswith("conv3d_stem_rows_kernel") for k in launched), launched
    assert stats.get("stem_stream") == 1
    k_len = 3 * int(np.prod(K))
    TS.assert_close_to_f64(got, ref, absref, k_len, acc_eps=TS.F16_EPS / (1 + k_len / 64.0), what=INSTANCE)


# ---- CPU: routing -------------------------------------------------------------------------------------------------
def _fast_stem_ops(batch):
    import pytorchvideo_b200.models.hub as PH
    from pytorchvideo_b200.engine.lower import lower_only
    plan, _ = lower_only(PH.slowfast_r50().eval(), TS.slowfast_inputs(torch.zeros(batch, 3, 32, 224, 224)))
    stem = "blocks.0.multipathway_blocks.1.conv"
    return [m for m in plan.meta if m["name"].startswith(stem)], plan.stats


PAIR = [("blocks.0.multipathway_blocks.1.conv.taps", "tcgen05"), ("blocks.0.multipathway_blocks.1.conv.tapsum", "other")]


def test_slowfast_fast_stem_route_by_batch(monkeypatch):
    """Batch 8: the stream kernel as `.taps`; `.tapsum` then reads one tap (its Co = 8 channels of the pre-BN sum),
    not the kt * Co channels of the factored partials.  The op list is the factored route's either way."""
    ops8, stats = _fast_stem_ops(8)
    assert [(m["name"], m["kind"]) for m in ops8] == PAIR, ops8
    assert stats["stem_stream"] == 1
    n_out = 8 * 32 * 112 * 112 * 8
    assert ops8[1]["bytes"] == 2 * n_out * 2
    from pytorchvideo_b200.engine import plan as PL
    monkeypatch.setattr(PL, "H100_SXM_SMS", 1 << 30)      # no batch fills the machine: the factored route
    off, stats_off = _fast_stem_ops(8)
    monkeypatch.undo()
    assert [(m["name"], m["kind"]) for m in off] == PAIR, off
    assert "stem_stream" not in stats_off
    assert off[1]["bytes"] == (5 + 1) * n_out * 2
    # batch 1: 112 output rows, less than a wave - the factored pair (pinned by tests/golden/reference_lowering.json)
    one, stats1 = _fast_stem_ops(1)
    assert [(m["name"], m["kind"]) for m in one] == PAIR
    assert "stem_stream" not in stats1


# ---- CPU: the instance ledger --------------------------------------------------------------------------------------
def test_every_stream_instance_is_reached():
    src = open(os.path.join(CSRC, "pv_stem_stream.cu")).read()
    compiled = {"conv3d_stem_stream_kernel<%s,%s>" % a for a in re.findall(r"PV_SS_LAUNCH\((\d+), (\d+)\)", src)}
    assert compiled == {INSTANCE}
    assert '"conv3d_stem_stream_kernel<" #KT "," #KS ">"' in src
