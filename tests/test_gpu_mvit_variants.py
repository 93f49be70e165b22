"""GPU: the MViT builder variants (norm="batchnorm" before / after fuse_bn(), pool_first, average pooling, token input,
headless, a stand-alone BatchNorm MultiScaleBlock) against the reference's outputs (tests/golden/mvit_variants.pt), and
every depthwise kernel instance with the pre-activation prologue (pv_conv3d_desc.pre_*) against float64."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

import pytorchvideo_b200.layers.attention as PA
import pytorchvideo_b200.models.hub as PH
import pytorchvideo_b200.models.vision_transformers as PV
from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200 import config
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.engine import compile_model

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CASES = sorted(TS.MVIT_VARIANT_CASES)
# (min in-band fraction, max |d|/max|ref|) of the f16 engine.  Measured on an H100 80GB HBM3 (400 W power limit), each
# bound is the measured value less 0.03 in-band and times 1.25 in max error; the comment holds the measurement
# (max |d| / max |ref|, fraction within rtol 1e-3 / atol 1e-4).  The BatchNorm models without any LayerNorm (bn_small,
# pool_first_bn) carry |logit| up to 67 / 23 through f16 activations and f16-rounded folded weights: fewer logits
# inside the band, while their f32 parity-mode outputs are within it everywhere.
F16_BOUNDS = {
    "avg": (0.77, 8.3e-4),                  # 6.641e-04, 0.803
    "bn_mvit_b": (0.91, 7.5e-4),            # 6.004e-04, 0.942
    "bn_mvit_b_fused": (0.85, 7.4e-4),      # 5.923e-04, 0.885
    "bn_small": (0.38, 3.0e-3),             # 2.423e-03, 0.411
    "head_none": (0.75, 1.4e-3),            # 1.088e-03, 0.784
    "pool_first_bn": (0.38, 4.9e-3),        # 3.887e-03, 0.417
    "pool_first_bn_avg": (0.57, 1.6e-3),    # 1.246e-03, 0.601
    "pool_first_ln": (0.64, 1.2e-3),        # 9.074e-04, 0.670
    "tokens": (0.80, 7.6e-4),               # 6.098e-04, 0.837
    "tokens_no_cls": (0.89, 7.1e-4),        # 5.685e-04, 0.921
    "bn_block": (0.88, 9.3e-4),             # 7.430e-04, 0.917
}
PRE_INSTANCES = ("dwconv3d_lane_kernel", "dwconv3d_tile_kernel", "dwconv3d_kernel", "dwconv3d_w4_kernel",
                 "dwconv_plane_kernel")


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(HERE, "golden", "mvit_variants.pt"), weights_only=False)


def _case(gold, case):
    g = gold[case]
    model, x, extra = TS.build_mvit_variant_case(case, PV.create_multiscale_vision_transformers, PA.MultiScaleBlock,
                                                 weight_seed=g["weight_seed"], input_seed=g["input_seed"])
    assert abs(TS.state_checksum(model) - g["state_checksum"]) <= 1e-6 * abs(g["state_checksum"])
    return g, model, x, extra


def _forward(model, x, extra):
    model.cuda()
    try:
        out = model(x.cuda(), *extra)
        out = out[0] if isinstance(out, tuple) else out
        return out.float().cpu()
    finally:
        model.cpu()


@pytest.mark.parametrize("case", CASES)
def test_mvit_variant_f32_parity_mode(gold, case):
    g, model, x, extra = _case(gold, case)
    ref = g["output"]
    config.set_precision("f32")
    try:
        out = _forward(model, x, extra)
    finally:
        config.set_precision("f16")
    assert out.shape == ref.shape
    scale = max(1.0, float(ref.abs().max()))
    err = (out - ref).abs()
    print("PARITY %s f32: max|d| = %.3e (scale %.3g)" % (case, float(err.max()), scale))
    assert bool((err <= 1e-3 * ref.abs() + 1e-4 * scale).all()), float(err.max())


@pytest.mark.parametrize("case", CASES)
def test_mvit_variant_f16(gold, case):
    g, model, x, extra = _case(gold, case)
    ref = g["output"]
    out = _forward(model, x, extra)
    out2 = _forward(model, x, extra)
    assert torch.equal(out, out2)
    assert out.shape == ref.shape
    scale = float(ref.abs().max())
    err = (out - ref).abs()
    inside = float((err <= 1e-3 * ref.abs() + 1e-4 * max(1.0, scale)).float().mean())
    rel = float(err.max()) / scale
    print("PARITY %s f16: max|d|/max|ref| = %.3e, fraction within rtol1e-3/atol1e-4 = %.3f" % (case, rel, inside))
    lo, hi = F16_BOUNDS[case]
    assert rel <= hi and inside >= lo, (rel, inside)


def _plan_kernels(model, x, extra):
    model.cuda()
    try:
        xd = x.cuda()
        cm = compile_model(model, xd, dtype="f16", use_graph=False, extra=tuple(tuple(e) for e in extra))
        _, ran = TS.launched_kernels(cm, xd)
    finally:
        model.cpu()
    return cm, ran


@pytest.mark.parametrize("case", ["bn_mvit_b", "bn_small", "pool_first_bn", "bn_block"])
def test_batchnorm_pools_run_prologue_instances(gold, case):
    _, model, x, extra = _case(gold, case)
    cm, ran = _plan_kernels(model, x, extra)
    print("%s kernels:" % case, ran)
    pre = sum(n for k, n in ran.items() if k.endswith(",pre>"))
    assert pre == cm.plan.stats["pool_prologue"] > 0


# The kernel ledger of the LayerNorm MViT-B-16x4 plan below (batch 1, 16x224x224) as the engine ran it before the
# prologue existed (recorded on an H100 from the parent tree): the LayerNorm model must run exactly these launches.
MVIT_B_16X4_LEDGER = {
    "add_layernorm_kernel": 33, "add_pos_cls_kernel": 1, "attention_wgmma_kernel<96>": 16,
    "conv3d_igemm_kernel<128,128>": 42, "conv3d_igemm_kernel<128,64>": 1, "conv3d_igemm_kernel<64,128>": 26,
    "copy_rows_kernel": 3, "dwconv3d_kernel<__half>": 3, "dwconv3d_lane_kernel<1,2,7>": 2,
    "dwconv3d_lane_kernel<2,2,7>": 13, "dwconv3d_lane_kernel<2,4,4>": 1, "head_reduce_kernel": 1,
    "layernorm_reg_kernel": 19, "ncdhw_f32_to_ndhwc4_padw_kernel": 1, "pool3d_kernel": 3,
}


def test_layernorm_mvit_b_runs_no_prologue_instance():
    """MViT-B-16x4: no prologue instance runs, and the plan's kernel ledger is the one it had before the prologue."""
    model = TS.randomize_model(PH.mvit_base_16x4(), seed=3).eval()
    x = TS.synthetic_clip(1, 16, 224, 224, seed=4)
    cm, ran = _plan_kernels(model, x, ())
    print("MViT-B-16x4 kernels:", ran)
    assert not [k for k in ran if k.endswith(",pre>")]
    assert "pool_prologue" not in cm.plan.stats
    pools = sum(n.endswith(".dwconv") for n, _ in cm.plan.ops)
    assert pools == 19
    assert sum(n for k, n in ran.items() if k.startswith(PRE_INSTANCES)) == pools
    assert ran == MVIT_B_16X4_LEDGER


# ---- every prologue instance against float64 ------------------------------------------------------------------------
# (dtype, T, H, kernel, stride, C, batch, entry): the pool strides of the video MViT, the image MViT's plane strides,
# and the route each takes: lane (3x3x3, W stride 1 / 2), TMA tile (kt = 1, T > 1), generic stencil (W stride 4 / 8),
# 4-wide stencil (f32 parity mode, and f16 when neither TMA kernel takes the shape: a temporal stride of 3 rules out the
# lane kernel, and a 5x5 output plane gives no tile-kernel box enough work), plane (one frame).
PRE_CASES = [
    ("f16", 4, 16, (3, 3, 3), (1, 1, 1), 96, 2, "dw"),
    ("f16", 4, 16, (3, 3, 3), (1, 2, 2), 192, 2, "dw"),
    ("f16", 4, 14, (3, 3, 3), (1, 2, 2), 40, 3, "dw"),
    ("f16", 4, 16, (1, 3, 3), (1, 2, 2), 96, 2, "dw"),
    ("f16", 4, 16, (3, 3, 3), (1, 4, 4), 96, 2, "dw"),
    ("f16", 8, 24, (3, 3, 3), (1, 8, 8), 96, 2, "dw"),
    ("f16", 4, 5, (3, 3, 3), (3, 1, 1), 96, 2, "dw"),
    ("f32", 4, 16, (3, 3, 3), (1, 1, 1), 96, 2, "dw"),
    ("f32", 4, 16, (3, 3, 3), (1, 2, 2), 96, 2, "dw"),
    ("f32", 4, 16, (3, 3, 3), (1, 4, 4), 96, 2, "dw"),
    ("f32", 8, 24, (3, 3, 3), (1, 8, 8), 96, 2, "dw"),
    ("f16", 1, 28, (1, 3, 3), (1, 1, 1), 96, 2, "plane"),
    ("f16", 1, 28, (1, 3, 3), (1, 2, 2), 96, 2, "plane"),
    ("f16", 1, 30, (1, 3, 3), (1, 2, 2), 200, 3, "plane"),
    ("f16", 1, 56, (1, 3, 3), (1, 4, 4), 192, 2, "plane"),
]


def _run_pre(dtype, T, H, k, s, C, N, entry, seed):
    g = torch.Generator().manual_seed(seed)
    tdt = torch.float16 if dtype == "f16" else torch.float32
    pad = tuple(v // 2 for v in k)
    To, Ho = [(n + 2 * p_ - kk) // st + 1 for n, p_, kk, st in ((T, pad[0], k[0], s[0]), (H, pad[1], k[1], s[1]))]
    rs = C + 8                                           # a token row carries more channels than the pool reads
    x = torch.randn(N, 1 + T * H * H, rs, generator=g).to(tdt).cuda()
    w = (torch.randn(C, 1, *k, generator=g) * 0.3).to(tdt)
    scale = torch.rand(C, generator=g) + 0.5
    bias = torch.rand(C, generator=g) - 0.5
    pre_s = torch.rand(C, generator=g) + 0.5
    pre_b = torch.rand(C, generator=g) * 4.0 - 1.0       # up to GELU(3) ~ 3: a leak into a padded tap shows
    y = torch.full((N, 1 + To * Ho * Ho, C), 7.0, dtype=tdt, device="cuda")
    d = L.Conv3dDesc()
    d.dtype = L.PV_F16 if dtype == "f16" else L.PV_F32
    d.N, d.Ti, d.Hi, d.Wi, d.Ci = N, T, H, H, C
    d.To, d.Ho, d.Wo, d.Co = To, Ho, Ho, C
    d.kt, d.kh, d.kw = k
    d.st, d.sh, d.sw = s
    d.pt, d.ph, d.pw = pad
    d.dt, d.dh, d.dw = 1, 1, 1
    d.groups = C
    d.x_row_stride, d.y_row_stride = rs, C
    d.x_batch_stride, d.y_batch_stride = (1 + T * H * H) * rs, (1 + To * Ho * Ho) * C
    wd = w.reshape(C, -1).t().contiguous().cuda()
    sd, bd, psd, pbd = scale.cuda(), bias.cuda(), pre_s.cuda(), pre_b.cuda()
    d.pre_scale, d.pre_bias, d.pre_act = psd.data_ptr(), pbd.data_ptr(), L.ACT_GELU
    lib = L.load()
    esz = x.element_size()
    st = torch.cuda.current_stream().cuda_stream

    def launch():
        xp, yp = x.data_ptr() + rs * esz, y.data_ptr() + C * esz           # step over the cls row of sample 0
        if entry == "plane":
            rc = lib.pv_dwplane_fwd(ctypes.byref(d), xp, wd.data_ptr(), sd.data_ptr(), bd.data_ptr(), yp, st)
        else:
            rc = lib.pv_dwconv3d_fwd(ctypes.byref(d), xp, wd.data_ptr(), sd.data_ptr(), bd.data_ptr(), yp, None, st)
        L.check(rc, "depthwise prologue")
        torch.cuda.synchronize()
    _, ran = TS.launched_kernels(launch)
    xin = x[:, 1:, :C].double().cpu().reshape(N, T, H, H, C).permute(0, 4, 1, 2, 3)
    w64 = w.double()
    ref, absref, u, _ = TS.prologue_conv_ref64(xin, pre_s, pre_b, w64, scale, bias, s, pad)
    sc = scale.double().view(1, C, 1, 1, 1)
    got = y[:, 1:].float().cpu().reshape(N, To, Ho, Ho, C).permute(0, 4, 1, 2, 3)
    return got, ref, absref, y, ran, u, w64, sc, pad


@pytest.mark.parametrize("case", PRE_CASES, ids=["%s_t%d_h%d_k%s_s%s_c%d_%s" % (c[0], c[1], c[2], "".join(map(str, c[3])),
                                                                                 "".join(map(str, c[4])), c[5], c[7])
                                                 for c in PRE_CASES])
def test_prologue_instance_against_float64(case):
    dtype, T, H, k, s, C, N, entry = case
    got, ref, absref, y, ran, u, w64, sc, pad = _run_pre(*case, seed=T * 131 + H * 31 + s[2] * 7 + C)
    print("prologue %s: %s" % (case, ran))
    assert len(ran) == 1 and next(iter(ran)).endswith(",pre>") and next(iter(ran)).startswith(PRE_INSTANCES), ran
    if dtype == "f16":
        # the TMA kernels round u(x) to f16 once in shared memory: one f16 rounding of every u, carried by the stencil
        extra = F.conv3d(u.abs(), w64.abs(), stride=s, padding=pad, groups=C) * sc.abs() * TS.F16_EPS
        TS.assert_close_to_f64(got, ref, absref, k[0] * k[1] * k[2], what="prologue %s %s" % (case, ran), extra64=extra)
    else:
        err = (got.double() - ref).abs()
        assert bool((err <= 2.0 ** -20 * absref + 1e-6).all()), float((err / (absref + 1e-6)).max())
    assert bool((y[:, 0] == 7.0).all())            # the cls rows are not written


def test_prologue_cases_reach_every_route_by_shape():
    reached = set()
    for i, case in enumerate(PRE_CASES):
        reached.update(_run_pre(*case, seed=i)[4])
    print("prologue instances:", sorted(reached))
    for base in PRE_INSTANCES:
        assert any(r.startswith(base + "<") for r in reached), base
    assert {"dwconv3d_w4_kernel<float,3,1,pre>", "dwconv3d_w4_kernel<__half,3,1,pre>", "dwconv3d_kernel<float,pre>",
            "dwconv3d_kernel<__half,pre>", "dwconv_plane_kernel<4,1,2,pre>"} <= reached


def test_dense_and_stem_entry_points_refuse_a_prologue():
    d = L.Conv3dDesc()
    d.dtype, d.N, d.Ti, d.Hi, d.Wi, d.Ci = L.PV_F16, 1, 2, 8, 8, 16
    d.To, d.Ho, d.Wo, d.Co = 2, 8, 8, 16
    d.kt = d.kh = d.kw = d.st = d.sh = d.sw = d.dt = d.dh = d.dw = d.groups = 1
    d.x_row_stride = d.y_row_stride = 16
    buf = torch.zeros(4096, dtype=torch.float32, device="cuda")
    d.pre_scale, d.pre_bias, d.pre_act = buf.data_ptr(), buf.data_ptr(), L.ACT_GELU
    lib = L.load()
    p = buf.data_ptr()
    assert lib.pv_conv3d_fwd(ctypes.byref(d), 0, p, p, p, p, None, p, None) == -3   # PV_ERR_UNSUPPORTED
    assert lib.pv_conv3d_tcgen05_supported(ctypes.byref(d)) == 0
    assert lib.pv_conv3d_stem_rows_supported(ctypes.byref(d)) == 0
    assert lib.pv_conv3d_stem_stream_supported(ctypes.byref(d)) == 0
