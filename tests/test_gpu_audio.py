"""Audiovisual SlowFast, the acoustic ResNet and SeparableBottleneckBlock on the engine, and the post-activation addend
of the convolution epilogue (pv_conv3d_desc.addend) that carries the audio fusion add.

CPU: builder parity with tests/golden/audio.pt, the launch list and structure of the lowering, error types.
GPU: the addend against float64 per kernel family, every golden case in f32 parity mode and in f16, lanes on / off."""
import os

import pytest
import torch
import torch.nn as nn

from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200 import models as M
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.engine.lower import lower_only
from pytorchvideo_b200.engine.packing import fold_bn
from pytorchvideo_b200.engine.plan import Plan, TRef

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "audio.pt")
SEED = 2024


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


def _case(name):
    return TS.build_audio_case(name, M, seed=SEED)


# ------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", sorted(TS.AUDIO_CASES))
def test_builders_match_the_reference(gold, name):
    m, x = _case(name)
    g = gold[name]
    assert repr(m) == g["repr"]
    assert list(m.state_dict().keys()) == g["keys"]
    assert TS.state_checksum(m) == pytest.approx(g["state_checksum"], rel=1e-12)
    xs = x if isinstance(x, list) else [x]
    assert [TS.tensor_checksum(t) for t in xs] == g["input_checksum"]


@pytest.mark.parametrize("name", sorted(TS.AUDIO_CASES))
def test_lowering_of_this_package_equals_the_reference_tree(gold, name):
    m, x = _case(name)
    plan, _ = lower_only(m, x)
    assert [(md["name"], md["kind"]) for md in plan.meta] == [tuple(v) for v in gold[name]["launches"]]


def test_separable_block_is_one_conv_b_launch_and_sum_doubles_conv_c_k():
    for name, k_mult in (("separable_sum", 2), ("separable_cat", 2)):
        m, x = _case(name)
        plan, shp = lower_only(m, x)
        names = [md["name"] for md in plan.meta]
        assert sum(n.endswith(".conv_b") for n in names) == 1, names
        cc = [md for md in plan.meta if md["name"].endswith(".conv_c")][0]
        m_out = shp[0] * shp[2] * shp[3] * shp[4]
        assert cc["flops"] == 2.0 * m_out * 64 * 16 * k_mult      # K = 2 C_inner: [W_c | W_c] for sum, the concat for cat
    m, x = _case("acoustic_r50")
    plan, _ = lower_only(m, x)
    names = [md["name"] for md in plan.meta]
    n_sep = sum(len(s.res_blocks) for s in list(m.blocks)[1:3])
    assert sum(n.endswith(".conv_b") for n in names) == sum(len(s.res_blocks) for s in list(m.blocks)[1:5])
    assert n_sep == 7


def test_acoustic_stem_is_one_convolution():
    for name in ("acoustic_r50", "acoustic_r50_k3"):
        m, x = _case(name)
        plan, _ = lower_only(m, x)
        stem = [md["name"] for md in plan.meta if md["name"].startswith("blocks.0.")]
        assert stem == ["blocks.0.conv"]


def test_addend_on_the_two_concat_writers_and_waits_on_the_audio_lane():
    m, x = _case("avsf_r50")
    plan, _ = lower_only(m, x)
    plan._schedule()
    with_add = [i for i, md in enumerate(plan.meta) if "addend" in md]
    names = [plan.meta[i]["name"] for i in with_add]
    assert names == ["blocks.0.multipathway_blocks.0.conv", "blocks.0.multipathway_fusion.block_fast_to_slow.0",
                     "blocks.1.multipathway_blocks.0.res_blocks.2.branch2.conv_c",
                     "blocks.1.multipathway_fusion.block_fast_to_slow.0",
                     "blocks.2.multipathway_blocks.0.res_blocks.3.branch2.conv_c",
                     "blocks.2.multipathway_fusion.block_fast_to_slow.0",
                     "blocks.3.multipathway_blocks.0.res_blocks.5.branch2.conv_c",
                     "blocks.3.multipathway_fusion.block_fast_to_slow.0"]
    offs = [plan.meta[i]["addend"][1] for i in with_add]
    assert offs == [0, 64, 0, 256, 0, 512, 0, 1024]
    for i in with_add:
        buf = plan.meta[i]["addend"][0]
        writer = max(j for j in range(i) if plan.op_io[j] is not None and any(getattr(t, "buf", t) is buf
                                                                                for t in plan.op_io[j][1]))
        assert plan.op_lane[writer] == 2 and writer in plan.sched["waits"][i]
    # no op reads and rewrites a concat buffer: every writer of a buffer that takes an addend writes it once
    for i in range(len(plan.ops)):
        io = plan.op_io[i]
        if io is not None:
            assert not {id(getattr(t, "buf", t)) for t in io[0]} & {id(getattr(t, "buf", t)) for t in io[1]}, plan.meta[i]


# algorithm of every audio-fusion convolution of AVSlowFast-R50 at B = 2: (5,1,1) on (B, C, T, 1, 1) maps.  The second
# conv of stage 1 (32 -> 320 channels, temporal stride 16) exceeds the TMA-fed kernel's stride product of 8 and runs on
# the CUDA-core kernel; stride 8 and 4 (stages 2, 3) stay on the tensor cores.
FUSION_ROUTES = {
    "blocks.0.multipathway_fusion.block_audio_to_fastslow.0": "tcgen05",
    "blocks.0.multipathway_fusion.block_audio_to_fastslow.3": "tcgen05",
    "blocks.1.multipathway_fusion.block_audio_to_fastslow.0": "tcgen05",
    "blocks.1.multipathway_fusion.block_audio_to_fastslow.3": "direct",
    "blocks.2.multipathway_fusion.block_audio_to_fastslow.0": "tcgen05",
    "blocks.2.multipathway_fusion.block_audio_to_fastslow.3": "tcgen05",
    "blocks.3.multipathway_fusion.block_audio_to_fastslow.0": "tcgen05",
    "blocks.3.multipathway_fusion.block_audio_to_fastslow.3": "tcgen05",
}


def test_audio_fusion_conv_routing():
    import ctypes
    m, x = _case("avsf_r50")
    plan, _ = lower_only(m, x)
    kinds = {md["name"]: md["kind"] for md in plan.meta if ".block_audio_to_fastslow." in md["name"]}
    assert kinds == FUSION_ROUTES
    # and that is what the library reports for each descriptor (stage i's audio map: T = 128 >> max(i - 1, 0))
    lib = L.load()
    for stage in range(4):
        fusion = m.blocks[stage].multipathway_fusion.block_audio_to_fastslow
        T = 128 >> max(stage - 1, 0)
        for i in (0, 3):
            c = fusion[i]
            xi = TRef(None, 2, T, 1, 1, c.in_channels)
            st = tuple(c.stride)
            To = (T + 2 * c.padding[0] - c.kernel_size[0]) // st[0] + 1
            d = plan._conv_desc(xi, (To, 1, 1), c.out_channels, tuple(c.kernel_size), st, tuple(c.padding), (1, 1, 1),
                                1, L.ACT_RELU, None, c.out_channels,
                                xi.Cp if xi.Cp < 64 else (xi.Cp + 63) // 64 * 64)
            tc = bool(lib.pv_conv3d_tcgen05_supported(ctypes.byref(d)))
            name = "blocks.%d.multipathway_fusion.block_audio_to_fastslow.%d" % (stage, i)
            assert FUSION_ROUTES[name] == ("tcgen05" if tc else "direct"), name


def test_oracle_matches_the_goldens(gold):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    try:
        from oracle.audio_ref import audio_forward
    finally:
        sys.path.remove(root)
    for name in ("avsf_r18_norm_none", "avsf_r18_sigmoid", "acoustic_r50_k3", "separable_sum", "separable_cat"):
        m, x = _case(name)
        assert torch.equal(audio_forward(m, x), gold[name]["output"]), name


def test_errors():
    m, x = _case("avsf_r18_sigmoid")
    with pytest.raises(RuntimeError):                       # wrong audio channel count
        lower_only(m, x[:2] + [torch.empty(1, 2, 128, 1, 80)])
    with pytest.raises(RuntimeError):                       # a fuse_a T that neither equals the Slow T nor is 1
        lower_only(m, x[:2] + [torch.empty(1, 1, 96, 1, 80)])
    blk = M.create_acoustic_bottleneck_block(dim_in=16, dim_inner=8, dim_out=16, conv_a_stride=(1, 1, 1),
                                             conv_b_kernel_size=(3, 1, 3), conv_b_padding=(1, 0, 1)).eval()
    blk.act_b[1] = nn.Sigmoid()
    with pytest.raises(NotImplementedError):                # branches with different activations
        lower_only(blk, torch.empty(1, 16, 4, 1, 8))
    blk = M.create_acoustic_bottleneck_block(dim_in=16, dim_inner=8, dim_out=16, conv_a_stride=(1, 1, 1),
                                             conv_b_kernel_size=(3, 1, 3), conv_b_padding=(1, 0, 1)).eval()
    blk.conv_b[1].stride = (1, 1, 2)
    with pytest.raises(NotImplementedError):                # branches without a common stride
        lower_only(blk, torch.empty(1, 16, 4, 1, 8))
    stem = M.create_acoustic_res_basic_stem(in_channels=1, out_channels=8, conv_kernel_size=(3, 1, 3),
                                            conv_padding=(2, 0, 1)).eval()
    stem.conv.convs[1].padding = (5, 0, 1)
    with pytest.raises(NotImplementedError):                # paddings that are not centre-consistent
        lower_only(stem, torch.empty(1, 1, 8, 1, 8))
    av = M.create_audio_visual_slowfast(model_depth=18, head_pool_kernel_sizes=((8, 2, 2), (32, 2, 2), (16, 1, 10)),
                                        stem_pool_kernel_sizes=((3, 3, 3), (1, 3, 3), (1, 3, 3))).eval()
    with pytest.raises(NotImplementedError):                # a stem pool that mixes frames
        lower_only(av, x)


def test_create_slowfast_depth_18_and_create_resnet_rejects_it():
    M.create_slowfast(model_depth=18)
    with pytest.raises(AssertionError):
        M.create_resnet(model_depth=18)


def test_no_new_kernel_instances():
    import re
    here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pytorchvideo_b200", "csrc")
    counts = {}
    for f, tag in (("pv_igemm.cu", "PV_IG_LAUNCH"), ("pv_stem.cu", "PV_ST_LAUNCH"), ("pv_igemm_gather.cu", "PV_GG_LAUNCH")):
        src = open(os.path.join(here, f)).read()
        counts[tag] = len(re.findall(r"\b%s\(\d+" % tag, src))   # launch sites, not the #define
    assert counts == {"PV_IG_LAUNCH": 12, "PV_ST_LAUNCH": 12, "PV_GG_LAUNCH": 4}, counts


# ------------------------------------------------------------------------------------------------- GPU
def _conv_addend_case(dt, N, T, H, W, Ci, Co, k, stride, pad, Ta, a_extra, a_off, act, seed=0, groups=1, stem=False,
                      y_slice=0):
    """One convolution with an addend through the engine's Plan, and its float64 reference.  stem: x is the network
    input (3 channels, converted lazily: the window-mode stem kernels); y_slice > 0: y is written as the last part of a
    channel concat, after y_slice other channels (row stride != Co, channel offset into the buffer)."""
    g = torch.Generator().manual_seed(seed)
    plan = Plan("cuda", dt)
    xv = TS.f16_exact(torch.randn(N, T, H, W, Ci, generator=g))
    if stem:
        src = xv.permute(0, 4, 1, 2, 3).contiguous().cuda()
        x = plan.emit_input_ncdhw(src, Ci, 4)
    else:
        x = plan.new_tensor(N, T, H, W, Ci)
    a = plan.new_tensor(N, Ta, 1, 1, a_off + Co + a_extra)
    w = TS.f16_exact(torch.randn(Co, Ci // groups, *k, generator=g) * (2.0 / (Ci // groups * k[0] * k[1] * k[2])) ** 0.5)
    bn = nn.BatchNorm3d(Co).eval()
    TS.randomize_model(bn, seed=seed)
    y = plan.emit_conv(x, w, None, bn, stride, pad, (1, 1, 1), groups, act, None, "conv", addend=(a, a_off))
    if y_slice:
        other = plan.new_tensor(y.N, y.T, y.H, y.W, y_slice)
        plan.concat_channels([other, y])
    plan.finalize()
    av = TS.f16_exact(torch.randn(N, Ta, 1, 1, a.Cp, generator=g)).to(a.buf.tensor.dtype)
    if not stem:
        x.buf.tensor.view(N, T, H, W, x.Cp)[..., :Ci].copy_(xv)
    a.buf.tensor.view(N, Ta, 1, 1, a.Cp).copy_(av)
    _, ran = TS.launched_kernels(lambda: (plan.run(torch.cuda.current_stream().cuda_stream), torch.cuda.synchronize()))
    got = y.buf.tensor.view(N, y.T, y.H, y.W, y.row_stride)[..., y.ch_off:y.ch_off + Co].float().cpu()
    s, b = (t[:Co].double() for t in fold_bn(None, bn, Co, Co))
    xd = xv.permute(0, 4, 1, 2, 3).double()
    conv = torch.nn.functional.conv3d(xd, w.double(), stride=stride, padding=pad, groups=groups)
    aconv = torch.nn.functional.conv3d(xd.abs(), w.double().abs(), stride=stride, padding=pad, groups=groups)
    pre = conv * s.view(1, -1, 1, 1, 1) + b.view(1, -1, 1, 1, 1)
    post = {L.ACT_RELU: torch.relu, L.ACT_NONE: lambda t: t}[act](pre)
    add = av[..., a_off:a_off + Co].double().permute(0, 4, 1, 2, 3)
    ref = (post + add).permute(0, 2, 3, 4, 1)
    absref = (aconv * s.abs().view(1, -1, 1, 1, 1) + b.abs().view(1, -1, 1, 1, 1) + add.abs()).permute(0, 2, 3, 4, 1)
    return got, ref, absref, post.abs().permute(0, 2, 3, 4, 1), ran, Ci // groups * k[0] * k[1] * k[2]


ADDEND_CASES = {
    # name: (N, T, H, W, Ci, Co, kernel, stride, pad, T_addend, extra channels, channel offset, act, family)
    "tma_bn128_straddle": (2, 20, 14, 14, 64, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 20, 0, 0, L.ACT_RELU, "conv3d_igemm_kernel<128"),
    "tma_bn64_offset_tbcast": (2, 4, 7, 7, 64, 64, (3, 1, 1), (1, 1, 1), (1, 0, 0), 1, 8, 16, L.ACT_RELU, "conv3d_igemm_kernel<64"),
    "tma_bn32_tail": (1, 2, 5, 9, 64, 24, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 0, 8, L.ACT_NONE, "conv3d_igemm_kernel<32"),
    "tma_bn16": (3, 5, 1, 10, 64, 16, (5, 1, 1), (2, 1, 1), (2, 0, 0), 3, 0, 0, L.ACT_RELU, "conv3d_igemm_kernel<16"),
    "gather_h1_w80": (2, 4, 1, 80, 24, 40, (3, 1, 3), (1, 1, 2), (1, 0, 1), 4, 0, 8, L.ACT_RELU, "conv3d_igemm_gather_kernel"),
}
# options of _conv_addend_case per case (the rest take the defaults)
ADDEND_OPTS = {
    # the Slow stem of AVSlowFast: 3-channel network input, (1,7,7) stride (1,2,2), 112x112 output (98 rows / tile)
    "stem_rows_slow_stem": dict(stem=True),
    # grouped mode of the TMA-fed kernel: 256 channels in 32 groups of 8 (4 group spans)
    "grouped_32": dict(groups=32),
    # y is the last part of a channel concat: row stride 48 + 64, channel offset 48
    "tma_concat_slice": dict(y_slice=48),
}
ADDEND_CASES.update({
    "stem_rows_slow_stem": (2, 2, 56, 56, 3, 64, (1, 7, 7), (1, 2, 2), (0, 3, 3), 2, 0, 16, L.ACT_RELU,
                            "conv3d_stem_rows_kernel"),
    "grouped_32": (2, 2, 14, 14, 256, 256, (1, 3, 3), (1, 1, 1), (0, 1, 1), 1, 0, 0, L.ACT_RELU,
                   "conv3d_igemm_grouped_kernel"),
    "tma_concat_slice": (2, 3, 9, 9, 64, 64, (3, 1, 1), (1, 1, 1), (1, 0, 0), 3, 0, 48, L.ACT_RELU,
                         "conv3d_igemm_kernel<64"),
})


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ADDEND_CASES))
def test_addend_against_float64(name):
    N, T, H, W, Ci, Co, k, st, pd, Ta, extra, off, act, family = ADDEND_CASES[name]
    got, ref, absref, post, ran, K = _conv_addend_case(L.PV_F16, N, T, H, W, Ci, Co, k, st, pd, Ta, extra, off, act,
                                                       **ADDEND_OPTS.get(name, {}))
    assert any(n.startswith(family) for n in ran), ran
    # the addend is added to the f16 result in the staged tile: one more rounding of |act(...)|
    TS.assert_close_to_f64(got, ref, absref, K, what=name, extra64=TS.F16_EPS * post)


@pytest.mark.gpu
def test_addend_direct_f32():
    got, ref, absref, _, ran, K = _conv_addend_case(L.PV_F32, 2, 3, 14, 14, 40, 48, (3, 1, 3), (1, 1, 2), (1, 0, 1),
                                                    1, 0, 8, L.ACT_RELU)
    assert any(n.startswith("conv3d_direct_kernel<float>") for n in ran), ran
    assert torch.allclose(got.double(), ref, rtol=1e-5, atol=1e-5 * float(absref.max()))


def _run(m, x, precision):
    from pytorchvideo_b200 import config
    old = config.get_precision()
    config.set_precision(precision)
    try:
        m = m.cuda()
        xs = [t.cuda() for t in x] if isinstance(x, list) else x.cuda()
        with torch.no_grad():
            return m(xs).float().cpu()
    finally:
        config.set_precision(old)


# f16: largest |got - ref| / max(1, max|ref|), measured on an H100 80GB HBM3 (700 W), times about 2.5
F16_BOUNDS = {"avsf_r50": 2e-3, "avsf_r50_b8_f16grid": 1e-3, "avsf_r18_norm_none": 1.5e-3, "avsf_r18_sigmoid": 1e-3, "acoustic_r50": 1.3e-3,
              "acoustic_r50_k3": 3e-4, "separable_sum": 1.5e-3, "separable_cat": 3e-3}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(TS.AUDIO_CASES))
def test_cases_against_goldens(gold, name):
    m, x = _case(name)
    ref = gold[name]["output"].double()
    scale = max(1.0, float(ref.abs().max()))
    y32 = _run(m, x, "f32").double()
    assert bool((( y32 - ref).abs() <= 1e-3 * ref.abs() + 1e-4 * scale).all()), float((y32 - ref).abs().max())
    y16 = _run(m, x, "f16").double()
    err = float((y16 - ref).abs().max()) / scale
    print("%s f16 err/max %.3g" % (name, err))
    assert err <= F16_BOUNDS[name], err


@pytest.mark.gpu
def test_single_stream_is_bitwise_the_same():
    m, x = _case("avsf_r18_sigmoid")
    from pytorchvideo_b200.engine import compile_model
    xs = [t.cuda() for t in x]
    m = m.cuda()
    cm = compile_model(m, xs, "f16", use_graph=False)
    lanes = cm(xs).clone()
    cm.plan.run(torch.cuda.current_stream().cuda_stream, single_stream=True)
    assert torch.equal(lanes, cm.output_view())


@pytest.mark.gpu
def test_wrong_audio_channels_raise():
    m, x = _case("avsf_r18_sigmoid")
    with pytest.raises(RuntimeError):
        m.cuda()([x[0].cuda(), x[1].cuda(), torch.zeros(1, 2, 128, 1, 80, device="cuda")])
