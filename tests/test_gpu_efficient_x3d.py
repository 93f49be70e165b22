"""Efficient X3D and the mobile efficient blocks on the engine, and HardSwish (PV_ACT_HSWISH) in every kernel family that
takes an activation.

CPU: builder parity with tests/golden/efficient_x3d.pt, the oracle against the goldens, the launch lists, the same
launches as models.x3d for the same network, error types.
GPU: HardSwish against float64 per kernel family, every golden case in f32 parity mode and in f16, the x3d cross-check
(bitwise), and the accelerator routes."""
import copy
import ctypes
import os
import sys

import pytest
import torch
import torch.nn as nn

from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.engine.lower import lower_only
from pytorchvideo_b200.engine.packing import fold_bn
from pytorchvideo_b200.engine.plan import Plan
from pytorchvideo_b200.models import hub as H

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "efficient_x3d.pt")
SEED = 31
NS = TS.efficient_namespace()


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


def _case(name):
    return TS.build_efficient_case(name, NS, seed=SEED)


def _mapped(x3d_builder, eff_builder, seed=5):
    """(x3d model, efficient model with the x3d weights) of the same network."""
    x3 = TS.randomize_model(x3d_builder(), seed=seed).eval()
    return x3, TS.map_x3d_to_efficient(x3, eff_builder().eval())


# ------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", sorted(TS.EFFICIENT_CASES))
def test_builders_match_the_reference(gold, name):
    m, x = _case(name)
    g = gold[name]
    assert TS.tree_digests(m) == g["tree_digests"]       # repr and state_dict keys of the reference's tree
    assert TS.state_checksum(m) == pytest.approx(g["state_checksum"], rel=1e-12)
    assert TS.tensor_checksum(x) == g["input_checksum"]


@pytest.mark.parametrize("name", sorted(TS.EFFICIENT_CASES))
def test_lowering_of_this_package_equals_the_reference_tree(gold, name):
    m, x = _case(name)
    plan, _ = lower_only(m, x)
    assert [(md["name"], md["kind"]) for md in plan.meta] == [tuple(v) for v in gold["launch_lists"][gold[name]["launches"]]]


def test_oracle_matches_the_goldens(gold):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    try:
        from oracle.efficient_ref import efficient_forward
    finally:
        sys.path.remove(root)
    for name in ("xs_no_head", "xs_head_hswish", "block_hswish_se", "block_bias_no_bn", "conv_5x1x1_dw_hswish",
                 "conv_3x1x1_hswish"):
        m, x = _case(name)
        assert torch.equal(efficient_forward(m, x), gold[name]["output"]), name


def test_xs_size_and_hub():
    m = H.efficient_x3d_xs()
    assert sum(p.numel() for p in m.parameters()) == 3794322 and len(m.state_dict()) == 568
    assert type(H.efficient_x3d_s()).__name__ == "EfficientX3d"
    with pytest.raises(RuntimeError):
        H.efficient_x3d_xs(pretrained=True)


@pytest.mark.parametrize("size", ["xs", "s"])
def test_same_launches_as_x3d(size):
    x3, eff = _mapped(getattr(H, "x3d_" + size), getattr(H, "efficient_x3d_" + size))
    T = {"xs": 4, "s": 13}[size]
    x = torch.empty(2, 3, T, 160, 160)
    pa, sa = lower_only(x3, x)
    pb, sb = lower_only(eff, x)
    assert sa == sb == (2, 400)
    assert [md["kind"] for md in pa.meta] == [md["kind"] for md in pb.meta]
    assert [md["flops"] for md in pa.meta] == [md["flops"] for md in pb.meta]
    # the stride-only shortcut's identity BatchNorm folds to exactly (1, 0)
    bn = eff.s2.pathway0_res0._res_proj.kernel.bn
    s, b = fold_bn(None, bn, 24, 24)
    assert bool((s == 1).all()) and bool((b == 0).all())


def test_routing_of_the_block():
    m, x = _case("block_hswish_se")
    plan, _ = lower_only(m, x)
    kinds = {md["name"]: md["kind"] for md in plan.meta}
    assert kinds["block._res_proj"] == kinds["block.layers.conv_0"] == kinds["block.layers.conv_2"] == "tcgen05"
    assert kinds["block.layers.conv_1"] == "depthwise"
    assert "block.layers.se.apply" in kinds and "block.layers.se.sum" not in kinds     # sums fused into conv_1
    m, x = _case("block_no_residual")
    names = [md["name"] for md in lower_only(m, x)[0].meta]
    assert not any("_res_proj" in n for n in names)


def test_convert_errors():
    m, _ = _case("block_hswish")
    with pytest.raises(NotImplementedError):
        m.convert((2, 24, 4, 14, 14), convert_for_quantize=True)
    m.convert_flag = True
    with pytest.raises(AssertionError, match="already converted"):
        m.convert((2, 24, 4, 14, 14))
    c = NS.Conv3dPwBnAct(8, 8)
    c.convert_flag = True
    with pytest.raises(AssertionError, match="already converted"):
        c.convert((1, 8, 1, 2, 2))


def test_deployable_form_is_refused():
    m, x = _case("xs_no_head")
    # what the reference's convert() leaves behind: a Conv2d-decomposed kernel
    m.s2.pathway0_res0.layers.conv_0.kernel = nn.Sequential(nn.Identity(), nn.Conv2d(24, 54, 1), nn.Identity())
    with pytest.raises(NotImplementedError, match="s2.pathway0_res0.layers.conv_0"):
        lower_only(m, x)
    m, x = _case("block_hswish_se")
    m.layers.se.se = nn.Sequential(nn.AdaptiveAvgPool3d(1))        # _SkipConnectMul-like SE
    with pytest.raises(NotImplementedError, match="layers.se"):
        lower_only(m, x)


def test_2d_pools_are_refused():
    from pytorchvideo_b200.layers.accelerator.mobile_cpu.pool import AdaptiveAvgPool2d, AdaptiveAvgPool2dOutSize1
    for p in (AdaptiveAvgPool2d(1), AdaptiveAvgPool2dOutSize1()):
        with pytest.raises(NotImplementedError):
            lower_only(p, torch.empty(1, 8, 2, 4, 4))


def test_torch_adaptive_pool_and_hardswish_still_lower():
    plan, shp = lower_only(nn.AdaptiveAvgPool3d(1), torch.empty(2, 8, 2, 4, 4))
    assert shp == (2, 8, 1, 1, 1)
    plan, _ = lower_only(nn.Hardswish(), torch.empty(2, 8, 2, 4, 4))
    assert plan.meta[-2]["name"] == "hswish"


def test_unknown_activation_codes_are_rejected():
    lib = L.load()
    p = Plan("cpu", L.PV_F16)
    x = p.new_tensor(1, 2, 8, 8, 64)
    for act in (L.ACT_HSWISH + 1, -1):
        d = p._conv_desc(x, (2, 8, 8), 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 1, act, None, 64, 64)
        assert not lib.pv_conv3d_tcgen05_supported(ctypes.byref(d))
        assert lib.pv_conv3d_fwd(ctypes.byref(d), L.ALGO_DIRECT, 16, 16, 16, 16, None, 16, None) == -1
        assert "activation" in L.last_error()
        assert lib.pv_scale_act(16, 16, L.PV_F16, 64, 64, 1, 1, 64, None, act, None) == -1
        assert lib.pv_temporal_tap_sum(16, 16, L.PV_F16, 1, 1, 1, 1, 8, 1, 1, 0, 1, 16, 16, act, 8, 8, None) == -1
    d = p._conv_desc(x, (2, 8, 8), 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 1, L.ACT_HSWISH, None, 64, 64)
    assert lib.pv_conv3d_tcgen05_supported(ctypes.byref(d))
    # the fused Fast-pathway bottleneck takes ReLU / none only
    bd = p.fused_bottleneck_desc(p.new_tensor(1, 4, 8, 8, 8), 8, 8, 32, 3, 1, True, L.ACT_HSWISH)
    assert not lib.pv_bottleneck_fused_supported(ctypes.byref(bd))


def test_hardswish_bottleneck_routes_around_the_fused_kernel():
    from pytorchvideo_b200.models.resnet import create_res_block, create_bottleneck_block
    blk = create_res_block(dim_in=8, dim_inner=8, dim_out=32, bottleneck=create_bottleneck_block,
                           conv_a_kernel_size=(3, 1, 1), conv_a_padding=(1, 0, 0), activation_block=nn.Hardswish).eval()
    plan, _ = lower_only(blk, torch.empty(1, 8, 4, 8, 8))
    assert "fused_block" not in [md["kind"] for md in plan.meta]


# ------------------------------------------------------------------------------------------------- GPU
def _hswish64(t):
    return t * (t + 3).clamp(0, 6) / 6


def _conv_case(dt, N, T, H, W, Ci, Co, k, stride, pad, groups=1, stem=False, seed=0):
    """One convolution with BN and HardSwish through the engine's Plan, and its float64 reference."""
    g = torch.Generator().manual_seed(seed)
    plan = Plan("cuda", dt)
    xv = torch.randn(N, T, H, W, Ci, generator=g) * 2.0
    xv = TS.f16_exact(xv) if dt == L.PV_F16 else xv
    if stem:
        x = plan.emit_input_ncdhw(xv.permute(0, 4, 1, 2, 3).contiguous().cuda(), Ci, 4)
    else:
        x = plan.new_tensor(N, T, H, W, Ci)
    w = torch.randn(Co, Ci // groups, *k, generator=g) * (6.0 / (Ci // groups * k[0] * k[1] * k[2])) ** 0.5
    w = TS.f16_exact(w) if dt == L.PV_F16 else w
    bn = nn.BatchNorm3d(Co).eval()
    TS.randomize_model(bn, seed=seed)
    y = plan.emit_conv(x, w, None, bn, stride, pad, (1, 1, 1), groups, L.ACT_HSWISH, None, "conv")
    plan.finalize()
    if not stem:
        x.buf.tensor.view(N, T, H, W, x.Cp)[..., :Ci].copy_(xv)
    _, ran = TS.launched_kernels(lambda: (plan.run(torch.cuda.current_stream().cuda_stream), torch.cuda.synchronize()))
    got = y.buf.tensor.view(N, y.T, y.H, y.W, y.row_stride)[..., y.ch_off:y.ch_off + Co].float().cpu()
    s, b = (t[:Co].double() for t in fold_bn(None, bn, Co, Co))
    xd = xv.permute(0, 4, 1, 2, 3).double()
    pre = torch.nn.functional.conv3d(xd, w.double(), stride=stride, padding=pad, groups=groups)
    apre = torch.nn.functional.conv3d(xd.abs(), w.double().abs(), stride=stride, padding=pad, groups=groups)
    pre = pre * s.view(1, -1, 1, 1, 1) + b.view(1, -1, 1, 1, 1)
    absref = apre * s.abs().view(1, -1, 1, 1, 1) + b.abs().view(1, -1, 1, 1, 1)
    ref = _hswish64(pre).permute(0, 2, 3, 4, 1)
    # |d hswish / dx| <= 1.5: the accumulation error of the pre-activation reaches the result at most 1.5 times
    return got, ref, 1.5 * absref.permute(0, 2, 3, 4, 1), pre, ran, Ci // groups * k[0] * k[1] * k[2]


HSWISH_CASES = {
    # name: (N, T, H, W, Ci, Co, kernel, stride, pad, groups, stem, instance prefix); the TMA-fed instances are
    # conv3d_igemm_kernel<BN,BM>: the prefix pins the tile width BN (BN 128 needs enough rows, else BN 64 is taken)
    "tma_bn128": (2, 20, 14, 14, 64, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1, False, "conv3d_igemm_kernel<128,"),
    "tma_bn64": (2, 4, 7, 7, 64, 64, (3, 1, 1), (1, 1, 1), (1, 0, 0), 1, False, "conv3d_igemm_kernel<64,"),
    "tma_bn32_tail": (1, 2, 5, 9, 64, 24, (1, 3, 3), (1, 1, 1), (0, 1, 1), 1, False, "conv3d_igemm_kernel<32,"),
    "tma_bn16_tail": (3, 5, 1, 10, 64, 12, (5, 1, 1), (2, 1, 1), (2, 0, 0), 1, False, "conv3d_igemm_kernel<16,"),
    "gather": (2, 4, 1, 80, 24, 40, (3, 1, 3), (1, 1, 2), (1, 0, 1), 1, False, "conv3d_igemm_gather_kernel"),
    "stem_rows": (2, 2, 40, 40, 3, 24, (1, 3, 3), (1, 2, 2), (0, 1, 1), 1, True, "conv3d_stem_rows_kernel"),
    "temporal_stream": (2, 6, 9, 9, 24, 24, (5, 1, 1), (1, 1, 1), (2, 0, 0), 24, False, "dwconv_temporal_kernel<5>"),
    "depthwise_lane_tail": (2, 4, 13, 13, 54, 54, (3, 3, 3), (1, 2, 2), (1, 1, 1), 54, False, "dwconv3d_lane_kernel"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(HSWISH_CASES))
def test_hardswish_against_float64(name):
    N, T, Hh, W, Ci, Co, k, st, pd, groups, stem, family = HSWISH_CASES[name]
    got, ref, absref, pre, ran, K = _conv_case(L.PV_F16, N, T, Hh, W, Ci, Co, k, st, pd, groups=groups, stem=stem)
    assert any(n.startswith(family) for n in ran), ran
    assert float((pre < -3).double().mean()) > 0.05 and float((pre > 3).double().mean()) > 0.05   # both knees
    TS.assert_close_to_f64(got, ref, absref, K, what=name)


@pytest.mark.gpu
def test_hardswish_direct_f32():
    got, ref, absref, _, ran, _ = _conv_case(L.PV_F32, 2, 3, 9, 9, 20, 36, (3, 1, 3), (1, 1, 2), (1, 0, 1))
    assert any(n.startswith("conv3d_direct_kernel<float>") for n in ran), ran
    assert torch.allclose(got.double(), ref, rtol=1e-5, atol=1e-5 * float(absref.max()))


@pytest.mark.gpu
def test_hardswish_se_scale_act_and_elementwise():
    g = torch.Generator().manual_seed(3)
    N, T, Hh, W, C, Cr = 2, 3, 5, 7, 56, 8
    plan = Plan("cuda", L.PV_F16)
    x = plan.new_tensor(N, T, Hh, W, C)
    w1, b1 = torch.randn(Cr, C, generator=g) * 0.3, torch.randn(Cr, generator=g) * 0.1
    w2, b2 = torch.randn(C, Cr, generator=g) * 0.5, torch.randn(C, generator=g) * 0.1
    plan.emit_se_scale_act(x, w1, b1, w2, b2, L.ACT_HSWISH, "se")
    z = plan.new_tensor(N, T, Hh, W, C)
    plan.emit_act(z, L.ACT_HSWISH, "act")
    plan.finalize()
    xv = TS.f16_exact(torch.randn(N, T, Hh, W, C, generator=g) * 4)
    zv = TS.f16_exact(torch.linspace(-5, 5, N * T * Hh * W * C).reshape(N, T, Hh, W, C))
    x.buf.tensor.view(N, T, Hh, W, C).copy_(xv)
    z.buf.tensor.view(N, T, Hh, W, C).copy_(zv)
    _, ran = TS.launched_kernels(lambda: (plan.run(torch.cuda.current_stream().cuda_stream), torch.cuda.synchronize()))
    assert ran.get("scale_act_kernel", 0) == 2, ran
    xd = xv.double()
    gate = torch.sigmoid(torch.relu(xd.mean((1, 2, 3)) @ w1.double().t() + b1.double()) @ w2.double().t() + b2.double())
    ref = _hswish64(xd * gate.view(N, 1, 1, 1, C))
    got = x.buf.tensor.view(N, T, Hh, W, C).float().cpu().double()
    assert bool(((got - ref).abs() <= 2 * TS.F16_EPS * ref.abs() + 1e-3).all()), float((got - ref).abs().max())
    gotz = z.buf.tensor.view(N, T, Hh, W, C).float().cpu().double()
    refz = _hswish64(zv.double())
    assert bool(((gotz - refz).abs() <= TS.F16_EPS * refz.abs() + 2.0 ** -24).all())


@pytest.mark.gpu
def test_hardswish_linear():
    from pytorchvideo_b200.engine import plan as PL
    g = torch.Generator().manual_seed(4)
    B, Ntok, Cin, Cout = 3, 37, 64, 72
    plan = Plan("cuda", L.PV_F16)
    x = plan.new_tensor(B, 1, 1, Ntok, Cin, Cp=Cin)
    w = TS.f16_exact(torch.randn(Cout, Cin, generator=g) * (6.0 / Cin) ** 0.5)
    b = torch.randn(Cout, generator=g) * 0.5
    y = PL.emit_linear(plan, x, w, b, L.ACT_HSWISH, None, "linear")
    plan.finalize()
    xv = TS.f16_exact(torch.randn(B, Ntok, Cin, generator=g))
    x.buf.tensor.view(B, Ntok, Cin).copy_(xv)
    _, ran = TS.launched_kernels(lambda: (plan.run(torch.cuda.current_stream().cuda_stream), torch.cuda.synchronize()))
    assert any(n.startswith("conv3d_igemm") for n in ran), ran
    got = y.buf.tensor.view(B, Ntok, y.row_stride)[..., :Cout].float().cpu()
    pre = xv.double() @ w.double().t() + b.double()
    absref = xv.double().abs() @ w.double().abs().t() + b.double().abs()
    TS.assert_close_to_f64(got, _hswish64(pre), 1.5 * absref, Cin, what="linear")


def _run(m, x, precision):
    from pytorchvideo_b200 import config
    old = config.get_precision()
    config.set_precision(precision)
    try:
        with torch.no_grad():
            return m.cuda()(x.cuda()).float().cpu()
    finally:
        config.set_precision(old)


# f16: largest |got - ref| / max(1, max|ref|), measured on an H100 80GB HBM3 (400 W), times about 2.5
F16_BOUNDS = {"xs_b2": 2e-3, "xs_b8_f16grid": 1.4e-3, "s_b1": 3.4e-3, "m_b1": 2.3e-3, "xs_no_head": 4.5e-3,
              "xs_head_relu": 1.8e-3, "xs_head_swish": 1.8e-3, "xs_head_hswish": 1.8e-3, "block_hswish_se": 1.9e-3,
              "block_hswish": 1.5e-3, "block_no_residual": 1.6e-3, "block_bias_no_bn": 2.1e-3, "conv_pw_hswish": 1.3e-3,
              "conv_dw_swish": 1.1e-3, "conv_t1_relu": 1.4e-3, "conv_3x1x1_hswish": 1.1e-3,
              "conv_5x1x1_dw_hswish": 2e-3}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(TS.EFFICIENT_CASES))
def test_cases_against_goldens(gold, name):
    m, x = _case(name)
    ref = gold[name]["output"].double()
    scale = max(1.0, float(ref.abs().max()))
    y32 = _run(m, x, "f32").double()
    err32 = float((y32 - ref).abs().max()) / scale
    y16 = _run(m, x, "f16").double()
    err = float((y16 - ref).abs().max()) / scale
    print("%s f32 err/max %.3g  f16 err/max %.3g" % (name, err32, err))
    assert bool(((y32 - ref).abs() <= 1e-3 * ref.abs() + 1e-4 * scale).all()), err32
    assert err <= F16_BOUNDS[name], err


@pytest.mark.gpu
@pytest.mark.parametrize("size,T,B", [("xs", 4, 2), ("s", 13, 1)])
def test_x3d_cross_check_is_bitwise(size, T, B):
    x3, eff = _mapped(getattr(H, "x3d_" + size), getattr(H, "efficient_x3d_" + size))
    x = TS.synthetic_clip(B, T, 160, 160, seed=8).cuda()
    with torch.no_grad():
        a = x3.cuda()(x)
        b = eff.cuda()(x)
    assert torch.equal(a, b), float((a - b).abs().max())


@pytest.mark.gpu
def test_accelerator_routes_give_the_same_output():
    from pytorchvideo_b200.accelerator import B200Block, convert_to_deployable_form, transmute_model
    m, x = _case("xs_b2")
    m = m.cuda()
    x = x.cuda()
    with torch.no_grad():
        direct = m(x).clone()
        one = convert_to_deployable_form(m, x)
        assert isinstance(one, B200Block) and len(one._by_shape) == 1
        via_convert = one(x)
        t = copy.deepcopy(m)
        transmute_model(t, "b200")
        assert sum(isinstance(b, B200Block) for b in t.modules()) == 26
        via_transmute = t(x)
    assert torch.equal(direct, via_convert)
    scale = float(direct.abs().max())
    assert float((via_transmute - direct).abs().max()) <= 1e-3 * scale
    blk, xb = _case("block_hswish_se")
    blk = blk.cuda()
    blk.convert(tuple(xb.shape))
    assert blk.convert_flag
    with pytest.raises(AssertionError, match="already converted"):
        blk.convert(tuple(xb.shape))
    with torch.no_grad():
        assert torch.equal(blk(xb.cuda()), convert_to_deployable_form(blk, xb.cuda())(xb.cuda()))
