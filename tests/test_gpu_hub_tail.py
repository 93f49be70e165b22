"""GPU: the image MViT-B-16 and SlowFast-16x8-R101-50-50 hub entries against the reference's logits
(tests/golden/hub_tail.pt), and the plane kernel (csrc/pv_dwplane.cu) against float64 per instance."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

import pytorchvideo_b200.models.hub as PH
from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200 import config
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.engine import compile_model

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
# (min in-band fraction, max |d|/max|ref|): the bounds of the video MViT-B-16x4 and SlowFast-R101 cases
# (tests/test_gpu_models.py F16_BOUNDS)
F16_BOUNDS = {"mvit_base_16": (0.67, 1.2e-3), "slowfast_16x8_r101_50_50": (0.84, 1.0e-3)}
# what pv_dwconv3d_fwd runs: the lane and tile kernels, the generic stencil (conv3d_direct_launch) and its 4-wide form
OLD_POOL_KERNELS = ("dwconv3d_lane_kernel", "dwconv3d_tile_kernel", "dwconv3d_kernel", "dwconv3d_w4_kernel",
                    "conv3d_direct_kernel")
PLANE_INSTANCES = {"dwconv_plane_kernel<%s,%s,%s>" % (s, ph, pw) for s in (1, 2) for ph, pw in ((4, 4), (2, 7))} | \
    {"dwconv_plane_kernel<4,1,2>"}


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(HERE, "golden", "hub_tail.pt"), weights_only=False)


def _case(gold, case):
    g = gold[case]
    model, x = TS.build_hub_tail_case(case, PH, weight_seed=g["weight_seed"], input_seed=g["input_seed"])
    assert abs(TS.state_checksum(model) - g["state_checksum"]) <= 1e-6 * abs(g["state_checksum"])
    return g, model, x


def _dev(x):
    return [t.cuda() for t in x] if isinstance(x, list) else x.cuda()


@pytest.mark.parametrize("case", sorted(TS.HUB_TAIL_CASES))
def test_hub_tail_f16(gold, case):
    g, model, x = _case(gold, case)
    ref = g["output"]
    model.cuda()
    try:
        out = model(_dev(x)).float().cpu()
        out2 = model(_dev(x)).float().cpu()
    finally:
        model.cpu()
    assert torch.equal(out, out2)
    assert out.shape == ref.shape
    scale = float(ref.abs().max())
    err = (out - ref).abs()
    inside = float((err <= 1e-3 * ref.abs() + 1e-4 * max(1.0, scale)).float().mean())
    rel = float(err.max()) / scale
    print("PARITY %s f16: max|d|/max|ref| = %.3e, fraction within rtol1e-3/atol1e-4 = %.3f" % (case, rel, inside))
    lo, hi = F16_BOUNDS[case]
    assert rel <= hi and inside >= lo, (rel, inside)


@pytest.mark.parametrize("case", sorted(TS.HUB_TAIL_CASES))
def test_hub_tail_f32_parity_mode(gold, case):
    g, model, x = _case(gold, case)
    ref = g["output"]
    config.set_precision("f32")
    try:
        model.cuda()
        out = model(_dev(x)).float().cpu()
    finally:
        config.set_precision("f16")
        model.cpu()
    scale = max(1.0, float(ref.abs().max()))
    err = (out - ref).abs()
    print("PARITY %s f32: max|d| = %.3e (scale %.3g)" % (case, float(err.max()), scale))
    assert bool((err <= 1e-3 * ref.abs() + 1e-4 * scale).all()), float(err.max())


def test_image_mvit_pools_run_on_the_plane_kernel(gold):
    _, model, x = _case(gold, "mvit_base_16")
    model.cuda()
    try:
        xd = x.cuda()
        cm = compile_model(model, xd, dtype="f16", use_graph=False)
        _, ran = TS.launched_kernels(cm, xd)
    finally:
        model.cpu()
    print("image MViT kernels:", ran)
    assert sum(n for k, n in ran.items() if k.startswith("dwconv_plane_kernel<")) == 19
    assert not [k for k in ran if k.startswith(OLD_POOL_KERNELS)]


def test_video_mvit_keeps_its_pool_kernels():
    """MViT-B-16x4 pools: 3x3x3 convolutions over 8 frames - the lane kernel at stride (1,2,2) and below, the generic
    stencil at (1,4,4) / (1,8,8), as before the plane kernel existed; the plane kernel never runs."""
    model = TS.randomize_model(PH.mvit_base_16x4(), seed=3).eval().cuda()
    try:
        x = TS.synthetic_clip(1, 16, 224, 224, seed=4).cuda()
        cm = compile_model(model, x, dtype="f16", use_graph=False)
        _, ran = TS.launched_kernels(cm, x)
    finally:
        model.cpu()
    print("video MViT kernels:", ran)
    assert not [k for k in ran if k.startswith("dwconv_plane_kernel")]
    pools = sum(n.endswith(".dwconv") for n, _ in cm.plan.ops)
    assert pools == 19
    assert sum(n for k, n in ran.items() if k.startswith(OLD_POOL_KERNELS)) == pools


def test_slowfast_16x8_fast_pathway_kernels(gold):
    """64 Fast frames at batch 8: the streaming Fast stem and the fused Fast bottleneck kernels take T = 64."""
    model = TS.randomize_model(PH.slowfast_16x8_r101_50_50(), seed=5).eval().cuda()
    try:
        x = TS.slowfast_inputs(TS.synthetic_clip(8, 64, 224, 224, seed=6))
        xd = [t.cuda() for t in x]
        cm = compile_model(model, xd, dtype="f16", use_graph=False)
        out, ran = TS.launched_kernels(cm, xd)
    finally:
        model.cpu()
    print("slowfast 16x8 kernels:", ran)
    assert tuple(out.shape) == (8, 400) and bool(torch.isfinite(out).all())
    assert sum(n for k, n in ran.items() if k.startswith("conv3d_stem_stream_kernel")) >= 1
    assert sum(n for k, n in ran.items() if k.startswith("bottleneck_fused_kernel")) == 7


# ---- the plane kernel against float64 at its tile edges -------------------------------------------------------------
# (H = W, stride, channels, token row stride, channel offset, batch): the image MViT's pools (fused K|V slices of the
# QKV GEMM output, pool_q slices) and edge shapes: partial tiles, channel chunks that run past C, odd batches.
PLANE_CASES = [
    (56, 4, 192, 288, 96, 2),      # block 0 K|V, 14x14 out                 <4,1,2>
    (64, 4, 40, 40, 0, 3),         # 16x16 out, 40 channels                 <4,1,2>
    (56, 2, 96, 576, 0, 2),        # block 1 pool_q, 28x28 out              <2,4,4>
    (30, 2, 200, 216, 8, 3),       # 15x15 out: partial 4x4 tiles           <2,4,4>
    (28, 2, 384, 576, 192, 2),     # blocks 1-2 K|V, 14x14 out              <2,2,7>
    (14, 2, 384, 1152, 0, 3),      # block 3 pool_q, 7x7 out                <2,2,7>
    (56, 1, 96, 96, 0, 1),         # 56x56 out                              <1,4,4>
    (14, 1, 768, 1152, 384, 5),    # blocks 3-13 K|V                        <1,2,7>
    (7, 1, 1536, 2304, 768, 3),    # blocks 14-15 K|V                       <1,2,7>
    (56, 4, 192, 288, 96, 3),      # block 0 K|V at batch 3 (the unused stride-4 tensor map was rejected)  <4,1,2>
]


def _run_plane(H, s, C, rs, off, N, seed):
    g = torch.Generator().manual_seed(seed)
    Ho = (H + 2 - 3) // s + 1
    x = (torch.randn(N, 1 + H * H, rs, generator=g)).half().cuda()
    w = (torch.randn(C, 1, 3, 3, generator=g) * 0.3).half()
    scale = torch.rand(C, generator=g) + 0.5
    bias = torch.rand(C, generator=g) - 0.5
    y = torch.full((N, 1 + Ho * Ho, C), 7.0, dtype=torch.float16, device="cuda")
    d = L.Conv3dDesc()
    d.dtype, d.N, d.Ti, d.Hi, d.Wi, d.Ci = L.PV_F16, N, 1, H, H, C
    d.To, d.Ho, d.Wo, d.Co = 1, Ho, Ho, C
    d.kt, d.kh, d.kw = 1, 3, 3
    d.st, d.sh, d.sw = 1, s, s
    d.pt, d.ph, d.pw = 0, 1, 1
    d.dt, d.dh, d.dw = 1, 1, 1
    d.groups = C
    d.x_row_stride, d.y_row_stride = rs, C
    d.x_batch_stride, d.y_batch_stride = (1 + H * H) * rs, (1 + Ho * Ho) * C
    wd = w.reshape(C, 9).t().contiguous().cuda()
    sd, bd = scale.cuda(), bias.cuda()
    lib = L.load()

    def launch():
        L.check(lib.pv_dwplane_fwd(ctypes.byref(d), x.data_ptr() + (rs + off) * 2, wd.data_ptr(), sd.data_ptr(),
                                   bd.data_ptr(), y.data_ptr() + C * 2, torch.cuda.current_stream().cuda_stream),
                "pv_dwplane_fwd")
        torch.cuda.synchronize()
    _, ran = TS.launched_kernels(launch)
    xin = x[:, 1:, off:off + C].double().cpu().reshape(N, H, H, C).permute(0, 3, 1, 2)
    w64 = w.double()
    ref = F.conv2d(xin, w64, stride=s, padding=1, groups=C) * scale.double().view(1, C, 1, 1) + bias.double().view(1, C, 1, 1)
    absref = F.conv2d(xin.abs(), w64.abs(), stride=s, padding=1, groups=C) * scale.double().abs().view(1, C, 1, 1) + \
        bias.double().abs().view(1, C, 1, 1)
    got = y[:, 1:].float().cpu().reshape(N, Ho, Ho, C).permute(0, 3, 1, 2)
    return got, ref, absref, y, ran


def _plane_ids():
    ids = []
    for c in PLANE_CASES:
        i = "h%d_s%d_c%d" % c[:3]
        ids.append(i if i not in ids else i + "_n%d" % c[5])      # a repeated shape at another batch
    return ids


@pytest.mark.parametrize("case", PLANE_CASES, ids=_plane_ids())
def test_plane_kernel_against_float64(case):
    H, s, C, rs, off, N = case
    got, ref, absref, y, ran = _run_plane(H, s, C, rs, off, N, seed=H * 31 + s * 7 + C)
    assert len(ran) == 1 and next(iter(ran)) in PLANE_INSTANCES, ran
    TS.assert_close_to_f64(got, ref, absref, 9, what="dwplane %s %s" % (case, ran))
    assert bool((y[:, 0] == 7.0).all())            # the cls rows are not written


def test_plane_cases_reach_every_instance():
    reached = set()
    for case in PLANE_CASES:
        reached.update(_run_plane(*case, seed=1)[4])
    assert reached == PLANE_INSTANCES
