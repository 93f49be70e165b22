"""GPU: per-kernel parity, CUDA path (through the C ABI) vs the CPU oracle arithmetic (torch fp32)."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda:0")


def _bn(c, seed):
    g = torch.Generator().manual_seed(seed)
    bn = nn.BatchNorm3d(c).eval()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5); bn.bias.copy_(torch.rand(c, generator=g) - 0.5)
        bn.running_mean.copy_(torch.rand(c, generator=g) - 0.5); bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn


def _ref_conv(x, w, b, bn, stride, padding, dilation, groups, act, res):
    y = F.conv3d(x, w, b, stride, padding, dilation, groups)
    if bn is not None:
        y = bn(y)
    if res is not None:
        y = y + res
    if act == "relu":
        y = F.relu(y)
    elif act == "swish":
        y = y * torch.sigmoid(y)
    return y


CONV_CASES = [
    # (N, Ci, T, H, W, Co, k, s, p, groups, act, residual)
    (2, 3, 4, 20, 20, 24, (1, 3, 3), (1, 2, 2), (0, 1, 1), 1, "relu", False),       # X3D stem spatial
    (1, 3, 6, 18, 18, 8, (5, 7, 7), (1, 2, 2), (2, 3, 3), 1, "relu", False),        # SlowFast fast stem
    (2, 24, 4, 10, 10, 54, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1, "relu", False),      # pointwise, odd widths
    (2, 54, 4, 10, 10, 24, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1, None, True),         # project + residual
    (1, 64, 4, 12, 12, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1), 1, "relu", False),      # conv_b
    (1, 64, 4, 12, 12, 64, (1, 3, 3), (1, 2, 2), (0, 1, 1), 1, "relu", False),      # strided conv_b
    (1, 128, 6, 7, 7, 32, (3, 1, 1), (1, 1, 1), (1, 0, 0), 1, "relu", False),       # temporal conv_a
    (1, 8, 16, 6, 6, 16, (7, 1, 1), (4, 1, 1), (3, 0, 0), 1, "relu", False),        # lateral fusion conv
    (2, 80, 2, 8, 8, 256, (1, 1, 1), (1, 2, 2), (0, 0, 0), 1, None, False),         # strided shortcut
    (2, 56, 4, 9, 9, 56, (3, 3, 3), (1, 1, 1), (1, 1, 1), 56, "swish", False),      # depthwise
    (2, 24, 6, 9, 9, 24, (5, 1, 1), (1, 1, 1), (2, 0, 0), 24, "relu", False),       # depthwise temporal
    (1, 16, 4, 9, 9, 16, (3, 3, 3), (2, 2, 2), (1, 1, 1), 16, None, False),         # depthwise strided (CSN)
    (2, 32, 6, 10, 10, 8, (3, 1, 1), (1, 1, 1), (1, 0, 0), 1, "relu", False),       # Fast-pathway conv_a: narrow TMA mode (64 B rows)
    (1, 16, 4, 9, 9, 16, (1, 3, 3), (1, 1, 1), (0, 1, 1), 1, "relu", True),         # Fast-pathway conv_b + residual: narrow TMA (32 B rows)
    (2, 32, 2, 9, 9, 128, (1, 1, 1), (1, 2, 2), (0, 0, 0), 1, None, False),         # strided shortcut from a 32-wide tensor
    (2, 64, 8, 56, 56, 512, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1, "relu", True),      # conv_c + residual, 784 wide tiles: residual ring over several tiles per CTA
    (1, 256, 4, 14, 14, 1024, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1, "relu", True),    # res4 conv_c + residual: one tile per CTA, 4 N tiles
    (1, 216, 3, 39, 39, 216, (3, 3, 3), (1, 2, 2), (1, 1, 1), 216, None, False),    # X3D-L res4 depthwise: odd 39 -> 20, stride 2
    (1, 96, 2, 39, 39, 192, (1, 1, 1), (1, 2, 2), (0, 0, 0), 1, None, False),       # X3D-L strided shortcut on an odd extent
    (1, 24, 2, 78, 156, 54, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1, "relu", False),     # X3D-L wide rows (W = 156)
    (1, 56, 2, 40, 156, 56, (3, 3, 3), (1, 1, 1), (1, 1, 1), 56, "swish", False),   # X3D-L depthwise on W = 156
]


@pytest.mark.parametrize("dtype,algo", [("f32", "direct"), ("f16", "direct"), ("f16", "tcgen05")])
@pytest.mark.parametrize("case", CONV_CASES, ids=[str(i) for i in range(len(CONV_CASES))])
def test_conv3d_bn_act(case, dtype, algo):
    from pytorchvideo_b200 import ops
    N, Ci, T, H, W, Co, k, s, p, groups, act, use_res = case
    if algo == "tcgen05" and groups != 1:
        pytest.skip("tensor-core path is dense only")
    g = torch.Generator().manual_seed(sum(v for v in case[:6]))
    x = torch.randn(N, Ci, T, H, W, generator=g)
    w = torch.randn(Co, Ci // groups, *k, generator=g) * (2.0 / (Ci // groups * np.prod(k))) ** 0.5
    bn = _bn(Co, 5)
    if dtype == "f16":   # compare against the oracle on the same f16-rounded operands
        x, w = x.half().float(), w.half().float()
    with torch.no_grad():
        y0 = F.conv3d(x, w, None, s, p, (1, 1, 1), groups)
        res = torch.randn(y0.shape, generator=g) if use_res else None
        if res is not None and dtype == "f16":
            res = res.half().float()
        ref = _ref_conv(x, w, None, bn, s, p, (1, 1, 1), groups, act, res)
    got, stats = ops.conv3d_bn_act(x.to(_dev()), w, None, bn, s, p, (1, 1, 1), groups, act,
                                   None if res is None else res.to(_dev()), dtype, algo)
    if algo == "tcgen05":
        assert stats["tcgen05"] == 1
    got = got.cpu()
    assert got.shape == ref.shape
    if dtype == "f32":
        assert torch.allclose(got, ref, rtol=1e-3, atol=1e-4), float((got - ref).abs().max())
    else:
        # f16 storage: one rounding of the stored output (2^-11 relative) on top of fp32 accumulation
        err = (got - ref).abs()
        tol = 1e-3 * ref.abs() + 1e-3 * float(ref.abs().max()) * 0.5 + 1e-4
        assert bool((err <= tol).all()), float(err.max())


# depthwise stencil through pv_dwconv3d_fwd (TMA-fed shared-memory kernel for f16) incl. fused SE sums.
# Shapes: X3D res2 / strided / stem temporal / 1x3x3, channel counts exercising the chunking (56, 216->24x9, 96->48x2)
DW_CASES = [
    (2, 56, 4, 20, 20, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    (2, 56, 5, 21, 19, (3, 3, 3), (1, 2, 2), (1, 1, 1)),
    (1, 216, 3, 9, 9, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    (2, 24, 8, 12, 12, (5, 1, 1), (1, 1, 1), (2, 0, 0)),
    (1, 96, 4, 14, 14, (3, 3, 3), (1, 2, 2), (1, 1, 1)),
    (1, 64, 6, 15, 15, (3, 3, 3), (2, 2, 2), (1, 1, 1)),
    (1, 128, 2, 7, 7, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    (1, 10, 3, 6, 6, (3, 3, 3), (1, 1, 1), (1, 1, 1)),       # padded channels (10 -> 16)
    # lane-per-channel-pair kernel (pv_dwlane.cu), X3D-M planes: 2x7 patches on 14x14 / 7x7 (masked row), uneven chunks
    (1, 216, 4, 14, 14, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    (1, 432, 3, 7, 7, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    (1, 216, 3, 28, 28, (3, 3, 3), (1, 2, 2), (1, 1, 1)),    # stride 2 -> 14x14
    (2, 112, 3, 28, 28, (3, 3, 3), (1, 1, 1), (1, 1, 1)),    # 4x4 patches, two chunks of 56
    (1, 54, 5, 56, 56, (3, 3, 3), (1, 1, 1), (1, 1, 1)),     # X3D-M res2 plane (54 -> 56 padded channels)
    # kt x 1 x 1 with SE sums runs the TMA tile kernel (the streaming temporal kernel takes no SE sums; its own rows,
    # same shapes without SE sums, are in tests/test_gpu_kernel_matrix.py): ring longer than the clip, T = 1, 3-tap
    (1, 40, 5, 9, 9, (3, 1, 1), (1, 1, 1), (1, 0, 0)),
    (1, 16, 1, 6, 6, (5, 1, 1), (1, 1, 1), (2, 0, 0)),
    (2, 24, 16, 28, 28, (5, 1, 1), (1, 1, 1), (2, 0, 0)),    # X3D stem geometry (16 frames)
]


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("case", DW_CASES, ids=[str(i) for i in range(len(DW_CASES))])
def test_dwconv3d_se_sums(case, dtype):
    from pytorchvideo_b200 import ops
    N, Cc, T, H, W, k, s, p = case
    g = torch.Generator().manual_seed(Cc + T + H)
    x = torch.randn(N, Cc, T, H, W, generator=g)
    w = torch.randn(Cc, 1, *k, generator=g) * (2.0 / np.prod(k)) ** 0.5
    bn = _bn(Cc, 7)
    if dtype == "f16":
        x, w = x.half().float(), w.half().float()
    with torch.no_grad():
        ref = _ref_conv(x, w, None, bn, s, p, (1, 1, 1), Cc, None, None)
    got, stats = ops.conv3d_bn_act(x.to(_dev()), w, None, bn, s, p, (1, 1, 1), Cc, None, None, dtype, None,
                                   se_sums=True)
    got = got.cpu()
    assert got.shape == ref.shape
    err = (got - ref).abs()
    if dtype == "f32":
        assert torch.allclose(got, ref, rtol=1e-3, atol=1e-4), float(err.max())
    else:
        tol = 1e-3 * ref.abs() + 1e-3 * float(ref.abs().max()) * 0.5 + 1e-4
        assert bool((err <= tol).all()), float(err.max())
    sums = stats["se_sums"].cpu()
    ref_sums = ref.sum(dim=(2, 3, 4))
    # sums are taken in fp32 BEFORE the f16 rounding of the stored output
    assert torch.allclose(sums, ref_sums, rtol=2e-3, atol=2e-3 * float(ref.abs().max()) * ref[0, 0].numel() ** 0.5), \
        float((sums - ref_sums).abs().max())


@pytest.mark.parametrize("Nq,Nk,resid", [(50, 50, False), (393, 393, False), (130, 37, True)])
def test_attention(Nq, Nk, resid):
    from pytorchvideo_b200 import ops
    g = torch.Generator().manual_seed(5)
    B, H, D = 2, 2, 96
    q, k, v = (torch.randn(B, H, n, D, generator=g) for n in (Nq, Nk, Nk))
    scale = D ** -0.5
    attn = ((q * scale) @ k.transpose(-2, -1)).softmax(-1)
    ref = attn @ v + (q if resid else 0)
    got = ops.attention(q.to(_dev()), k.to(_dev()), v.to(_dev()), scale, resid, "f32").cpu()
    assert torch.allclose(got, ref, rtol=1e-3, atol=1e-4), float((got - ref).abs().max())


@pytest.mark.parametrize("Nq,Nk,resid", [(50, 50, False), (393, 393, False), (130, 37, True), (1569, 393, False), (65, 129, True)])
def test_attention_f16_tensor_core(Nq, Nk, resid):
    from pytorchvideo_b200 import ops
    g = torch.Generator().manual_seed(6)
    B, H, D = 2, 3, 96
    q, k, v = (torch.randn(B, H, n, D, generator=g).half().float() for n in (Nq, Nk, Nk))
    scale = D ** -0.5
    attn = ((q * scale) @ k.transpose(-2, -1)).softmax(-1)
    ref = attn @ v + (q if resid else 0)
    got = ops.attention(q.to(_dev()), k.to(_dev()), v.to(_dev()), scale, resid, "f16").cpu()
    err = (got - ref).abs()
    assert float(err.max()) <= 4e-3 * max(1.0, float(ref.abs().max())), float(err.max())


@pytest.mark.parametrize("shape", [
    (8, 256, 8, 14, 14, 256, (1, 3, 3), (0, 1, 1)),      # SlowFast res4 conv_b at bench size (TMA-fed, N = 256)
    (8, 32, 32, 56, 56, 8, (3, 1, 1), (1, 0, 0)),        # Fast pathway res2 conv_a at bench size (narrow TMA mode)
    (8, 8, 32, 56, 56, 8, (1, 3, 3), (0, 1, 1)),         # Fast pathway res2 conv_b at bench size (gather-fed)
])
def test_full_size_conv_is_exactly_homogeneous(shape):
    """Full-size layers are too big for the CPU oracle inside a test; a convolution without bias is
    homogeneous, and scaling by a power of two is exact in f16/fp32 (outside the subnormal range), so
    conv(2x) == 2 conv(x) BIT FOR BIT
    (any dropped / duplicated tap, mis-addressed tile edge or stale shared memory breaks it); plus a
    spot check of 64 output positions against the fp32 reference."""
    from pytorchvideo_b200 import ops
    N, Ci, T, H, W, Co, k, p = shape
    g = torch.Generator().manual_seed(Ci + Co)
    x = (torch.randn(N, Ci, T, H, W, generator=g) * 0.5).half().float()
    w = (torch.randn(Co, Ci, *k, generator=g) * (1.0 / (Ci * np.prod(k))) ** 0.5).half().float()
    y1, _ = ops.conv3d_bn_act(x.to(_dev()), w, None, None, (1, 1, 1), p, (1, 1, 1), 1, None, None, "f16", "tcgen05")
    y2, _ = ops.conv3d_bn_act((2 * x).to(_dev()), w, None, None, (1, 1, 1), p, (1, 1, 1), 1, None, None, "f16", "tcgen05")
    big = y1.abs() > 2.0 ** -12          # below that an f16 result may be subnormal, where doubling is not exact
    assert torch.equal(y2[big], 2 * y1[big])
    assert torch.allclose(y2, 2 * y1, rtol=0, atol=2.0 ** -22)
    y1 = y1.cpu()
    idx = torch.randint(0, N * T * H * W, (64,), generator=g)
    for j in idx.tolist():
        n, r = divmod(j, T * H * W)
        t, r = divmod(r, H * W)
        h, ww = divmod(r, W)
        xp = F.pad(x[n], (p[2], p[2], p[1], p[1], p[0], p[0]))
        patch = xp[:, t:t + k[0], h:h + k[1], ww:ww + k[2]]
        ref = (w * patch.unsqueeze(0)).sum(dim=(1, 2, 3, 4))
        assert torch.allclose(y1[n, :, t, h, ww], ref, rtol=2e-3, atol=2e-3 * float(ref.abs().max()) + 1e-4)


# ---- fused narrow-pathway bottleneck block (csrc/pv_fastblock.cu) ------------------------------------------------
FUSED_BLOCK_CASES = [
    # (N, T, H, W, dim_in, dim_inner, dim_out, kt_a, spatial stride)      SlowFast Fast-pathway geometries, small extents
    (2, 5, 13, 11, 8, 8, 32, 3, 1),        # res2 block 0: projection shortcut from the 8-channel stem output
    (2, 6, 17, 15, 32, 8, 32, 3, 1),       # res2 blocks 1-2: identity shortcut, edge tiles in both directions
    (1, 4, 18, 14, 32, 16, 64, 3, 2),      # res3 block 0: stride 2, projection shortcut
    (1, 7, 9, 20, 64, 16, 64, 3, 1),       # res3 blocks 1-3
    (2, 9, 14, 14, 64, 16, 64, 3, 1),      # small planes: several T chunks per clip
    (1, 4, 12, 12, 32, 8, 32, 1, 1),       # pointwise conv_a (kt = 1)
    (1, 33, 7, 7, 32, 8, 32, 3, 1),        # long clip: ring wrap-around over many frames
]


@pytest.mark.parametrize("case", FUSED_BLOCK_CASES, ids=[str(i) for i in range(len(FUSED_BLOCK_CASES))])
def test_fused_bottleneck_block_matches_oracle_and_unfused(case, monkeypatch):
    """ONE launch for conv_a -> conv_b -> conv_c (+ shortcut) + ReLU vs the oracle's unfused ResBlock.forward
    (models/resnet.py:1179-1189, 1345-1365) on f16-grid operands; also equal (to f16 rounding of the two
    intermediates) to the engine's own unfused lowering."""
    from oracle.interp import oracle_forward
    from pytorchvideo_b200 import testing as TS
    from pytorchvideo_b200.engine import compile_model
    from pytorchvideo_b200.engine.lower import Lowering
    from pytorchvideo_b200.models.resnet import create_bottleneck_block, create_res_block
    N, T, H, W, cin, cmid, cout, kt, s = case
    blk = create_res_block(dim_in=cin, dim_inner=cmid, dim_out=cout, bottleneck=create_bottleneck_block,
                           conv_a_kernel_size=(kt, 1, 1), conv_a_stride=(1, 1, 1), conv_a_padding=(kt // 2, 0, 0),
                           conv_b_stride=(1, s, s))
    blk = TS.randomize_model(blk, seed=sum(case), f16_weights=True).eval()
    x = TS.f16_exact(torch.randn(N, cin, T, H, W, generator=torch.Generator().manual_seed(7)))
    ref = oracle_forward(blk, x)
    cm = compile_model(blk, x.cuda(), dtype="f16", use_graph=False)
    assert cm.plan.stats.get("fused_block", 0) == 1 and cm.plan.num_launches() == 3      # layout in, fused block, layout out
    out = cm(x.cuda()).float().cpu()
    assert out.shape == ref.shape
    scale = float(ref.abs().max())
    err = (out - ref).abs()
    assert bool((err <= 2e-3 * ref.abs() + 1e-3 * scale).all()), float(err.max()) / scale
    monkeypatch.setattr(Lowering, "_fusable_bottleneck", lambda self, m, x: False)
    cm2 = compile_model(blk, x.cuda(), dtype="f16", use_graph=False)
    assert cm2.plan.stats.get("fused_block", 0) == 0
    out2 = cm2(x.cuda()).float().cpu()
    assert bool(((out - out2).abs() <= 2e-3 * ref.abs() + 1e-3 * scale).all())
