"""The double-buffered convolution epilogue (pv_epilogue.cuh) against float64, at tile counts that exercise it.

A CTA's k-th tile is staged in buffer k % 2; the epilogue DMA warp loads each tile's residual two tiles ahead and
stores every tile.  The shapes give each CTA at least three tiles on 114 to 132 SMs, with CTAs that end on either
buffer (odd and even tile counts), plus the prologue's edge cases: fewer tiles than SMs (one tile per CTA, the
second buffer never filled) and exactly two tiles per CTA (both prologue loads, no refill).  Each row asserts the
kernel instance that ran, as the kernel matrix does.
"""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200 import testing as TS

CASES = {
    # name: (expected instance, N, Ci, T, H, W, Co, kernel, stride, padding, groups, act, residual, addend)
    # 462 tiles of 128 x 128: 3-4 per CTA on 132 SMs, 4-5 on 114
    "dense_residual": ("conv3d_igemm_kernel<128,128>", 2, 64, 4, 56, 66, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1,
                       L.ACT_RELU, True, False),
    "dense_residual_addend": ("conv3d_igemm_kernel<128,128>", 2, 64, 4, 56, 66, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1,
                              L.ACT_RELU, True, True),
    # C_out 320 = two 128-wide N tiles and a 64-channel tail: 450 tiles
    "n_tiles_64_tail": ("conv3d_igemm_kernel<128,128>", 2, 128, 4, 48, 50, 320, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1,
                        L.ACT_RELU, True, False),
    # 3x3 on 45 x 45 planes: the 128-row boxes are clipped at the H / W edges
    "clipped_m_tiles": ("conv3d_igemm_kernel<128,128>", 4, 64, 6, 45, 45, 128, (1, 3, 3), (1, 1, 1), (0, 1, 1), 1,
                        L.ACT_NONE, True, False),
    # 256 channels in 32 groups of 8: 4 group spans of 64 output channels
    "grouped": ("conv3d_igemm_grouped_kernel<64,128>", 2, 256, 4, 40, 40, 256, (1, 3, 3), (1, 1, 1), (0, 1, 1), 32,
                L.ACT_RELU, True, False),
    # C_in 24: cp.async gather; 430 tiles of 128 x 128
    "gather_residual": ("conv3d_igemm_gather_kernel<128>", 2, 24, 8, 40, 86, 96, (1, 3, 3), (1, 1, 1), (0, 1, 1), 1,
                        L.ACT_RELU, True, False),
    # stem rows: 448 output rows of 56 pixels
    "stem_rows": ("conv3d_stem_rows_kernel<64,2>", 2, 3, 4, 112, 112, 64, (1, 7, 7), (1, 2, 2), (0, 3, 3), 1,
                  L.ACT_RELU, False, False),
    # 13 filter rows and 104 KiB of weights: two ring stages fit beside one staging buffer only
    "stem_rows_one_buffer": ("conv3d_stem_rows_kernel<128,2>", 2, 3, 6, 64, 112, 128, (1, 13, 7), (1, 2, 2),
                             (0, 6, 3), 1, L.ACT_RELU, False, False),
    # 40 tiles: fewer than SMs, one tile per CTA
    "fewer_tiles_than_sms": ("conv3d_igemm_kernel<64,128>", 1, 64, 1, 40, 128, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1,
                             L.ACT_RELU, True, False),
}


def _case(row):
    inst, N, Ci, T, H, W, Co, k, s, p, groups, act, use_res, use_add = row
    stem = Ci == 3
    from pytorchvideo_b200.engine.packing import fold_bn
    from pytorchvideo_b200.engine.plan import Plan
    g = torch.Generator().manual_seed(Ci * 131 + Co + H)
    To, Ho, Wo = [(d + 2 * pp - kk) // ss + 1 for d, kk, ss, pp in zip((T, H, W), k, s, p)]
    plan = Plan("cuda", L.PV_F16)
    xv = TS.f16_exact(torch.randn(N, T, H, W, Ci, generator=g))
    if stem:
        x = plan.emit_input_ncdhw(xv.permute(0, 4, 1, 2, 3).contiguous().cuda(), Ci, 4)
    else:
        x = plan.new_tensor(N, T, H, W, Ci)
    r = plan.new_tensor(N, To, Ho, Wo, Co) if use_res else None
    a = plan.new_tensor(N, To, 1, 1, Co) if use_add else None
    fan = Ci // groups * k[0] * k[1] * k[2]
    w = TS.f16_exact(torch.randn(Co, Ci // groups, *k, generator=g) * (2.0 / fan) ** 0.5)
    bn = nn.BatchNorm3d(Co).eval()
    TS.randomize_model(bn, seed=Co)
    y = plan.emit_conv(x, w, None, bn, s, p, (1, 1, 1), groups, act, r, "conv",
                       addend=None if a is None else (a, 0))
    plan.finalize()
    if not stem:
        x.buf.tensor.view(N, T, H, W, x.Cp)[..., :Ci].copy_(xv)
    rv = av = None
    if use_res:
        rv = TS.f16_exact(torch.randn(N, To, Ho, Wo, Co, generator=g))
        r.buf.tensor.view(N, To, Ho, Wo, r.Cp)[..., :Co].copy_(rv)
    if use_add:
        av = TS.f16_exact(torch.randn(N, To, 1, 1, Co, generator=g))
        a.buf.tensor.view(N, To, 1, 1, a.Cp)[..., :Co].copy_(av)
    _, ran = TS.launched_kernels(lambda: (plan.run(torch.cuda.current_stream().cuda_stream), torch.cuda.synchronize()))
    got = y.buf.tensor.view(N, To, Ho, Wo, y.row_stride)[..., y.ch_off:y.ch_off + Co].float().cpu()

    sc, bi = (t[:Co].double().view(1, -1, 1, 1, 1) for t in fold_bn(None, bn, Co, Co))
    xd = xv.permute(0, 4, 1, 2, 3).double()
    pre = F.conv3d(xd, w.double(), None, s, p, 1, groups) * sc + bi
    absref = F.conv3d(xd.abs(), w.double().abs(), None, s, p, 1, groups) * sc.abs() + bi.abs()
    if use_res:
        rd = rv.permute(0, 4, 1, 2, 3).double()
        pre = pre + rd
        absref = absref + rd.abs()
    post = torch.relu(pre) if act == L.ACT_RELU else pre
    ref, extra = post, None
    if use_add:
        ad = av.permute(0, 4, 1, 2, 3).double()
        ref = post + ad
        absref = absref + ad.abs()
        extra = (TS.F16_EPS * post.abs()).permute(0, 2, 3, 4, 1)   # the addend rounds the staged f16 tile once more
    perm = lambda t: t.permute(0, 2, 3, 4, 1)
    return inst, got, perm(ref), perm(absref), extra, ran, fan


def _tiles_per_cta(row, sm):
    """(fewest, most) tiles per CTA of the TMA-fed 1x1 rows and the gather / stem rows (their tile counts are simple)."""
    inst, N, Ci, T, H, W, Co, k, s, p, groups, act, use_res, use_add = row
    To, Ho, Wo = [(d + 2 * pp - kk) // ss + 1 for d, kk, ss, pp in zip((T, H, W), k, s, p)]
    if inst.startswith("conv3d_stem_rows"):
        tiles = N * To * Ho * -(-Wo // 128)
    else:
        bn = int(inst.split("<")[1].split(",")[0].rstrip(">"))
        tiles = -(-(N * To * Ho * Wo) // 128) * -(-Co // bn)
    grid = min(tiles, sm)
    return tiles // grid, -(-tiles // grid)


@pytest.mark.parametrize("name", ["dense_residual", "n_tiles_64_tail", "gather_residual", "stem_rows"])
@pytest.mark.parametrize("sm", [114, 132])
def test_shapes_give_every_cta_several_tiles_of_both_parities(name, sm):
    lo, hi = _tiles_per_cta(CASES[name], sm)
    assert lo >= 3 and (lo % 2 or hi % 2), (lo, hi)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_epilogue_pipeline_against_float64(name):
    inst, got, ref, absref, extra, ran, K = _case(CASES[name])
    assert inst in ran, "expected %s, launched %s" % (inst, ran)
    TS.assert_close_to_f64(got, ref, absref, K, what=name, extra64=extra)


@pytest.mark.gpu
def test_exactly_two_tiles_per_cta():
    # H = SM count rows of 128 pixels with 64 channels: 2 * SMs tiles of 128 x 64, two per CTA
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    row = ("conv3d_igemm_kernel<64,128>", 1, 64, 2, sm, 128, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1, L.ACT_RELU, True,
           False)
    assert _tiles_per_cta(row, sm) == (2, 2)
    inst, got, ref, absref, extra, ran, K = _case(row)
    assert inst in ran, "expected %s, launched %s" % (inst, ran)
    TS.assert_close_to_f64(got, ref, absref, K, what="two_tiles_per_cta", extra64=extra)
