"""Deterministic synthetic weights / inputs shared by tests, bench.py and the golden generator.

Fresh builder init zeroes the last BatchNorm gamma of every residual branch
(models/weight_init.py), which makes every bottleneck a no-op in eval mode - a parity test on such
a model passes even with broken kernels (SURVEY section 7, hard part 1).  ``randomize_model`` gives
every BatchNorm random affine + running statistics (as the reference's tests/test_fuse_bn.py:58-63
does) and re-draws conv / linear weights from a fixed seed, on the CPU generator, so the same
state is reproduced bit-for-bit here and on the GPU box.
"""
import math
from fractions import Fraction

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


def f16_exact(t):
    """Round to the nearest f16-representable value (kept in fp32)."""
    return t.half().float()


@torch.no_grad()
def randomize_model(model, seed=1234, f16_weights=False):
    """f16_weights: draw the conv / linear / positional weights on the f16 grid (fp32 tensors whose
    values are exactly representable in f16).  The reference CPU forward and the f16 tensor-core path
    then multiply IDENTICAL weights - what is left between them is activation rounding and summation
    order, not an input difference (the weight rounding of arbitrary fp32 weights alone moves 8-25 %
    of the logits out of the rtol 1e-3 / atol 1e-4 band, tests/test_oracle_pinning.py)."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)

    def u(t, lo, hi):
        t.copy_(torch.rand(t.shape, generator=g, dtype=torch.float32) * (hi - lo) + lo)

    for m in model.modules():
        if isinstance(m, (nn.Conv3d, nn.Conv2d)):
            fan_in = m.weight.shape[1] * m.weight[0, 0].numel()
            m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5)
            if m.bias is not None:
                u(m.bias, -0.1, 0.1)
        elif isinstance(m, nn.modules.batchnorm._BatchNorm):
            if getattr(m, "block_final_bn", False):
                u(m.weight, 0.2, 0.6)       # keep the residual stream well conditioned
            else:
                u(m.weight, 0.5, 1.5)
            u(m.bias, -0.5, 0.5)
            u(m.running_var, 0.5, 1.5)
            u(m.running_mean, -0.5, 0.5)
        elif isinstance(m, nn.Linear):
            m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (1.0 / m.weight.shape[1]) ** 0.5)
            if m.bias is not None:
                u(m.bias, -0.1, 0.1)
        elif isinstance(m, nn.LayerNorm):
            u(m.weight, 0.5, 1.5)
            u(m.bias, -0.2, 0.2)
    for name, p in model.named_parameters():
        if name.endswith(("cls_token", "pos_embed_spatial", "pos_embed_temporal", "pos_embed_class", "pos_embed")):
            p.copy_(torch.randn(p.shape, generator=g) * 0.2)
    if f16_weights:
        for m in model.modules():
            if isinstance(m, (nn.Conv3d, nn.Conv2d, nn.Linear)):
                m.weight.copy_(f16_exact(m.weight))
    return model


def synthetic_clip(batch, t, h, w, seed=42, channels=3, f16_values=False):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    x = torch.rand((batch, channels, t, h, w), generator=g, dtype=torch.float32)
    return f16_exact(x) if f16_values else x


def slowfast_inputs(clip, alpha=4):
    """[slow, fast] as the reference builds them (uniform_temporal_subsample_repeated with
    frame_ratios=(alpha, 1), tests/test_models_slowfast.py:142-144): slow = frames at
    linspace(0, T-1, T//alpha).long()."""
    T = clip.shape[2]
    idx = torch.clamp(torch.linspace(0, T - 1, T // alpha), 0, T - 1).long()
    return [torch.index_select(clip, 2, idx), clip]


def synthetic_u8_clip(t, h, w, seed=0, channels=3):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    return torch.randint(0, 256, (channels, t, h, w), generator=g, dtype=torch.uint8)


def tensor_checksum(t):
    t = t.detach().double().cpu().reshape(-1)
    return [float(t.sum()), float(t.abs().sum()), float((t * t).sum())]


def state_checksum(model):
    s = 0.0
    for _, v in sorted(model.state_dict().items()):
        if v.is_floating_point():
            s += float(v.double().abs().sum())
    return s


MODEL_CASES = {
    # name: (hub builder name, kwargs, batch, T, H, W, is_slowfast)
    "x3d_xs": ("x3d_xs", {}, 2, 4, 160, 160, False),
    "x3d_m": ("x3d_m", {}, 1, 16, 224, 224, False),
    "slowfast_r50": ("slowfast_r50", {}, 1, 32, 224, 224, True),
    "slow_r50": ("slow_r50", {}, 1, 8, 224, 224, False),
    "csn_r101": ("csn_r101", {}, 1, 32, 224, 224, False),
    "r2plus1d_r50": ("r2plus1d_r50", {}, 1, 16, 224, 224, False),
    "i3d_r50": ("i3d_r50", {}, 1, 8, 224, 224, False),
    "mvit_base_16x4": ("mvit_base_16x4", {}, 1, 16, 224, 224, False),
    # same architecture on a 8x112x112 clip (785 tokens): cheap enough for the f32 CUDA-core parity mode
    "mvit_base_8x112": ("mvit_base_16x4", {"spatial_size": 112, "temporal_size": 8}, 2, 8, 112, 112, False),
    # further hub entries of the same families: goldens pin the oracle / module trees (CPU); not in the GPU lists yet
    "slowfast_r101": ("slowfast_r101", {}, 1, 32, 224, 224, True),
    "c2d_r50": ("c2d_r50", {}, 1, 8, 224, 224, False),
    "x3d_s": ("x3d_s", {}, 1, 13, 160, 160, False),
    "x3d_l": ("x3d_l", {}, 1, 16, 312, 312, False),
    "mvit_base_32x3": ("mvit_base_32x3", {}, 1, 32, 224, 224, False),
    # BASELINE.json configs at their REAL batch sizes, weights and clips drawn on the f16 grid (CASE_OPTS)
    "c1_x3d_xs": ("x3d_xs", {}, 1, 4, 160, 160, False),
    "c2_slowfast_r50_b8": ("slowfast_r50", {}, 8, 32, 224, 224, True),
    "c3_mvit_base_16x4_b8": ("mvit_base_16x4", {}, 8, 16, 224, 224, False),
    "c4_x3d_m_b32": ("x3d_m", {}, 32, 16, 224, 224, False),
    "slow_r50_f16w": ("slow_r50", {}, 2, 8, 224, 224, False),
    "mvit_base_8x112_f16w": ("mvit_base_16x4", {"spatial_size": 112, "temporal_size": 8}, 2, 8, 112, 112, False),
}
# per-case options of the golden generator / tests: f16_grid = weights AND input clip exactly representable in f16
CASE_OPTS = {
    # X3D-L (312^2, 55 blocks): with random BatchNorm statistics the residual stream grows to |x| ~ 1e3 by stage 5 and the
    # squeeze-excitation gates there saturate (pre-activations ~ +-140), so a gate near its zero crossing turns a 1e-4
    # relative change of a channel mean (the f16 rounding of the WEIGHTS) into a percent-level change of that channel
    # (tools/debug_block.py x3d_l 4 6: 3.5e-3 with the SE, 8.7e-4 without, same with the CUDA-core depthwise kernel).
    # On the f16 grid both sides multiply identical weights and the comparison is well conditioned again.
    "x3d_l": {"f16_grid": True},
    "c1_x3d_xs": {"f16_grid": True},
    "c2_slowfast_r50_b8": {"f16_grid": True},
    "c3_mvit_base_16x4_b8": {"f16_grid": True},
    "c4_x3d_m_b32": {"f16_grid": True},
    "slow_r50_f16w": {"f16_grid": True},
    "mvit_base_8x112_f16w": {"f16_grid": True},
}


def build_case(case, hub_module, weight_seed=1234, input_seed=42):
    """(model, inputs, is_slowfast) of a MODEL_CASES entry, built from ``hub_module`` (this package's hub)."""
    hub, kw, B, T, H, W, is_sf = MODEL_CASES[case]
    grid = CASE_OPTS.get(case, {}).get("f16_grid", False)
    model = randomize_model(getattr(hub_module, hub)(**kw), seed=weight_seed, f16_weights=grid).eval()
    clip = synthetic_clip(B, T, H, W, seed=input_seed, f16_values=grid)
    return model, (slowfast_inputs(clip) if is_sf else clip), is_sf


# The image MViT and SlowFast-16x8-R101-50-50 hub entries -> tests/golden/hub_tail.pt (oracle/gen_golden_hub.py).
# name: (batch, input shape per sample); the SlowFast input is a 64-frame clip split into 16 Slow + 64 Fast frames.
HUB_TAIL_CASES = {
    "mvit_base_16": (2, (3, 224, 224)),
    "slowfast_16x8_r101_50_50": (1, (3, 64, 224, 224)),
}


def build_hub_tail_case(case, hub_module, weight_seed=1234, input_seed=42):
    """(model, input) of a HUB_TAIL_CASES entry, built from ``hub_module``: an image batch (B, 3, H, W) for the image
    MViT, the [slow, fast] pathway list for the SlowFast."""
    B, shape = HUB_TAIL_CASES[case]
    model = randomize_model(getattr(hub_module, case)(), seed=weight_seed).eval()
    if len(shape) == 3:
        return model, synthetic_clip(B, 1, shape[1], shape[2], seed=input_seed)[:, :, 0].contiguous()
    return model, slowfast_inputs(synthetic_clip(B, shape[1], shape[2], shape[3], seed=input_seed))


# Grouped conv_b (ResNeXt-style group counts, CSN with several channels per group): the builders' own arguments on the
# hub entries.  Kept apart from MODEL_CASES, whose host lowering test counts every groups > 1 conv as depthwise.
# name: (hub builder name, kwargs, batch, T, H, W, is_slowfast, f16_grid) -> tests/golden/model_grouped_<name>.pt
GROUPED_MODEL_CASES = {
    "slow_r50_g32": ("slow_r50", {"stage_conv_b_num_groups": (32,) * 4}, 1, 8, 224, 224, False, False),
    "csn_r101_w8": ("csn_r101", {"stage_conv_b_width_per_group": 8}, 1, 32, 224, 224, False, False),
    "slowfast_r50_g": ("slowfast_r50", {"stage_conv_b_num_groups": ((32,) * 4, (2,) * 4)}, 1, 32, 224, 224, True, False),
    "slow_r50_g32_f16w": ("slow_r50", {"stage_conv_b_num_groups": (32,) * 4}, 2, 8, 224, 224, False, True),
}


def build_grouped_case(case, hub_module, weight_seed=1234, input_seed=42):
    """(model, inputs, is_slowfast) of a GROUPED_MODEL_CASES entry, built from ``hub_module``."""
    hub, kw, B, T, H, W, is_sf, grid = GROUPED_MODEL_CASES[case]
    model = randomize_model(getattr(hub_module, hub)(**kw), seed=weight_seed, f16_weights=grid).eval()
    clip = synthetic_clip(B, T, H, W, seed=input_seed, f16_values=grid)
    return model, (slowfast_inputs(clip) if is_sf else clip), is_sf



# The layer goldens are stored in two files (tests/golden/layers.pt, layers_conv.pt) to keep each under 1 MB.
LAYER_GOLDEN_FILES = ("layers.pt", "layers_conv.pt")
LAYER_GOLDEN_CONV = ("conv_reduce_cat", "conv_reduce_sum", "patch_embed")   # the cases stored in layers_conv.pt


def load_layer_goldens(golden_dir):
    import os
    out = {}
    for f in LAYER_GOLDEN_FILES:
        out.update(torch.load(os.path.join(golden_dir, f), weights_only=False))
    return out


# ---- layer-level cases (tests/golden/layers*.pt): name -> (builder, input shape, thw or None) --------------------
def _layer_builders():
    import torch.nn as nn
    from functools import partial
    from .layers.attention import Mlp, MultiScaleAttention, MultiScaleBlock
    from .layers.convolutions import ConvReduce3D, create_conv_2plus1d
    from .layers.positional_encoding import SpatioTemporalClsPositionalEncoding
    from .models.head import create_vit_basic_head
    from .models.stem import create_conv_patch_embed
    ln = partial(nn.LayerNorm, eps=1e-6)
    return {
        "conv_reduce_sum": (lambda: ConvReduce3D(in_channels=16, out_channels=32, kernel_size=((1, 1, 1), (3, 3, 3), (1, 3, 3)),
                                                 stride=((1, 1, 1), (1, 1, 1), None), padding=((0, 0, 0), (1, 1, 1), (0, 1, 1)),
                                                 bias=(False, True, None), reduction_method="sum"), (2, 16, 4, 12, 12), None),
        "conv_reduce_cat": (lambda: ConvReduce3D(in_channels=16, out_channels=24, kernel_size=((1, 1, 1), (3, 1, 1)),
                                                 padding=((0, 0, 0), (1, 0, 0)), reduction_method="cat"), (2, 16, 4, 12, 12), None),
        "conv2plus1d_xy_first": (lambda: create_conv_2plus1d(in_channels=16, out_channels=32, inner_channels=24, conv_xy_first=True,
                                                             stride=(1, 2, 2)), (2, 16, 4, 12, 12), None),
        "conv2plus1d": (lambda: create_conv_2plus1d(in_channels=16, out_channels=32, stride=(2, 1, 1)), (2, 16, 4, 12, 12), None),
        "mlp": (lambda: Mlp(in_features=96, hidden_features=384, out_features=192), (2, 50, 96), None),
        # MViT-B block 1 geometry at a small grid: Q pooled (1,2,2), K/V pooled (1,4,4), 2 heads of 96
        "attention_pool_qkv": (lambda: MultiScaleAttention(192, num_heads=2, qkv_bias=True, kernel_q=(3, 3, 3), kernel_kv=(3, 3, 3),
                                                           stride_q=(1, 2, 2), stride_kv=(1, 4, 4), norm_layer=ln,
                                                           residual_pool=False), (2, 1 + 4 * 8 * 8, 192), (4, 8, 8)),
        "attention_residual_pool_nocls": (lambda: MultiScaleAttention(64, num_heads=2, kernel_kv=(3, 3, 3), stride_kv=(1, 2, 2),
                                                                      has_cls_embed=False, norm_layer=ln, residual_pool=True),
                                          (2, 2 * 8 * 8, 64), (2, 8, 8)),
        "block_widen_pool": (lambda: MultiScaleBlock(96, 192, 1, qkv_bias=True, norm_layer=ln, attn_norm_layer=ln,
                                                     kernel_q=(3, 3, 3), kernel_kv=(3, 3, 3), stride_q=(1, 2, 2),
                                                     stride_kv=(1, 2, 2)), (2, 1 + 4 * 8 * 8, 96), (4, 8, 8)),
        "block_dim_mul_in_att": (lambda: MultiScaleBlock(64, 128, 2, qkv_bias=True, norm_layer=ln, attn_norm_layer=ln,
                                                         dim_mul_in_att=True, kernel_kv=(3, 3, 3), stride_kv=(1, 2, 2)),
                                 (2, 1 + 2 * 8 * 8, 64), (2, 8, 8)),
        "posenc": (lambda: SpatioTemporalClsPositionalEncoding(96, (4, 7, 7), sep_pos_embed=True, has_cls=True), (2, 4 * 7 * 7, 96), None),
        "patch_embed": (lambda: create_conv_patch_embed(in_channels=3, out_channels=96, conv_kernel_size=(3, 7, 7),
                                                        conv_stride=(2, 4, 4), conv_padding=(1, 3, 3)), (2, 3, 8, 56, 56), None),
        "vit_head": (lambda: create_vit_basic_head(in_features=192, out_features=40, seq_pool_type="cls"), (3, 17, 192), None),
    }


LAYER_CASES = tuple(sorted(["conv_reduce_sum", "conv_reduce_cat", "conv2plus1d_xy_first", "conv2plus1d", "mlp",
                            "attention_pool_qkv", "attention_residual_pool_nocls", "block_widen_pool",
                            "block_dim_mul_in_att", "posenc", "patch_embed", "vit_head"]))


def build_layer_case(name, seed=77):
    """(module, input, thw) with weights AND input on the f16 grid (same operands for reference and engine)."""
    make, shape, thw = _layer_builders()[name]
    torch.manual_seed(seed)
    m = randomize_model(make(), seed=seed, f16_weights=True).eval()
    g = torch.Generator(device="cpu")
    g.manual_seed(seed + 1)
    x = f16_exact(torch.randn(shape, generator=g) if len(shape) == 3 else torch.rand(shape, generator=g))
    return m, x, thw


# ---- detection cases (tests/golden/detection.pt): trunk + RoIAlign head, weights / clips on the f16 grid ----------
DETECTION_CASES = {
    # name: (hub builder, kwargs, batch, T, H, W, is_slowfast, number of boxes)
    # head_activation=None: compare LOGITS (with random weights the default Sigmoid saturates to 0 / 1 and hides errors)
    "slow_r50_detection": ("slow_r50_detection", {"head_activation": None}, 2, 4, 128, 128, False, 6),
    "slowfast_r50_detection": ("slowfast_r50_detection", {"head_activation": None}, 2, 32, 128, 128, True, 5),
    "slow_r50_detection_sigmoid": ("slow_r50_detection", {}, 1, 4, 96, 96, False, 4),      # the hub default head
}


def synthetic_boxes(n_boxes, batch, H, W, seed=9):
    """[K, 5] fp32 (batch index, x1, y1, x2, y2) in input pixels: random boxes plus the shapes the RoIAlign boundary
    rules care about - one reaching outside the frame, one smaller than a feature cell, the whole frame."""
    g = torch.Generator().manual_seed(seed)
    b = torch.randint(0, batch, (n_boxes,), generator=g).float()
    x1 = torch.rand(n_boxes, generator=g) * W * 0.6
    y1 = torch.rand(n_boxes, generator=g) * H * 0.6
    x2 = x1 + 8 + torch.rand(n_boxes, generator=g) * W * 0.5
    y2 = y1 + 8 + torch.rand(n_boxes, generator=g) * H * 0.5
    boxes = torch.stack([b, x1, y1, x2, y2], 1)
    if n_boxes >= 3:
        boxes[0, 1:] = torch.tensor([-20.0, -12.0, W + 30.0, H * 0.5])      # sticks out left / top / right
        boxes[1, 1:] = torch.tensor([W * 0.5, H * 0.5, W * 0.5 + 3.0, H * 0.5 + 2.0])   # sub-cell box -> size clamp 1
        boxes[2, 1:] = torch.tensor([0.0, 0.0, float(W), float(H)])
    return boxes.contiguous()


def build_detection_case(case, hub_module, weight_seed=1234, input_seed=42):
    """(model, clip inputs, boxes, is_slowfast) of a DETECTION_CASES entry."""
    hub, kw, B, T, H, W, is_sf, K = DETECTION_CASES[case]
    model = randomize_model(getattr(hub_module, hub)(**kw), seed=weight_seed, f16_weights=True).eval()
    clip = synthetic_clip(B, T, H, W, seed=input_seed, f16_values=True)
    return model, (slowfast_inputs(clip) if is_sf else clip), synthetic_boxes(K, B, H, W), is_sf


def roi_align_case(seed=5):
    """Op-level RoIAlign case: feature map on the f16 grid + boxes (see synthetic_boxes), several (output size, scale,
    sampling ratio) settings.  Golden = torchvision.ops.roi_align (tests/golden/detection.pt["roi_align"])."""
    g = torch.Generator().manual_seed(seed)
    x = f16_exact(torch.randn(2, 24, 9, 11, generator=g))
    boxes = synthetic_boxes(7, 2, 144, 176, seed=seed + 1)
    settings = [((7, 7), 1.0 / 16.0, 0), ((7, 7), 1.0 / 16.0, 2), ((3, 5), 0.25, 0), ((1, 1), 1.0 / 16.0, 3)]
    return x, boxes, settings


# ---- kernel-instance ledger and a float64 comparator for the kernel tests -----------------------------------------
def kernel_counts():
    """Snapshot of the library's per-instance launch counts ({"conv3d_igemm_kernel<64,128>": 3, ...})."""
    from . import _lib
    return _lib.kernel_counts()


def kernel_count_diff(before, after):
    """Launches per instance between two kernel_counts() snapshots (instances that did not launch are left out)."""
    return {k: n - before.get(k, 0) for k, n in sorted(after.items()) if n != before.get(k, 0)}


def launched_kernels(fn, *args, **kwargs):
    """Run fn(*args, **kwargs) and return (its result, {instance: launches} of the library kernels it ran)."""
    before = kernel_counts()
    out = fn(*args, **kwargs)
    return out, kernel_count_diff(before, kernel_counts())


F16_EPS = 2.0 ** -11          # unit roundoff of f16 (one round-to-nearest of the stored result)
ACC_EPS = 2.0 ** -20          # fp32 accumulation allowance per unit of |x|.|w| magnitude, see assert_close_to_f64


F32_EPS = 2.0 ** -24          # unit roundoff of fp32 (rnd_eps of a kernel that stores fp32)


def assert_close_to_f64(got, ref64, absref64, k_len, acc_eps=ACC_EPS, what="", extra64=None, rnd_eps=F16_EPS):
    """Compare an f16-storage (or, with rnd_eps=F32_EPS, fp32-storage) kernel result with its float64 reference.

    ref64: the operation in float64 on the exact f16-grid operands the kernel received.  absref64: the same operation
    on |x| and |w| with |scale|, plus |bias| and |residual| - the magnitude the result is summed from.  Each element
    may differ from ref64 by one f16 rounding of the stored result (2^-11 |ref|) plus an fp32 accumulation term
    proportional to absref64 that grows with the reduction length K, plus half the smallest f16 subnormal step.
    extra64 (optional, same shape): a further per-element allowance, the error of rounded intermediates propagated to
    the result (fused kernels that keep intermediates in f16, see fused_block_ref64 in the kernel-matrix tests).
    Rounding must also be unbiased: over the normal-range elements the mean error in the direction of |ref| must stay
    well below the mean rounding step (truncation toward zero moves it to about -0.7 of a step).  extra64 does not
    enter that limit: it is a worst case (every rounding of every intermediate at its extreme, all with the same sign),
    while the intermediates are rounded to nearest, so their share of the mean signed error is zero-mean noise that
    shrinks like 1 / sqrt(n).  Charging the worst case would hide a truncated intermediate, whose bias is what the
    check must see.  Returns (largest err / tol,
    largest share of the accumulation term used, largest share of extra64 used): a correctly rounded result may use
    nearly all of the rounding term, so the second number is the margin of the accumulation constant; the third
    charges everything beyond the rounding term to extra64 (0.0 without extra64).
    rnd_eps: the unit roundoff of the stored result; the absolute floor scales with it (2^-24 for f16 storage, half
    its smallest subnormal step; 2^-37 for fp32 storage)."""
    got64 = got.detach().double().cpu()
    ref64, absref64 = ref64.double().cpu(), absref64.double().cpu()
    assert got64.shape == ref64.shape, (what, tuple(got64.shape), tuple(ref64.shape))
    assert bool(torch.isfinite(got64).all()), "%s: non-finite output" % what
    err = got64 - ref64
    acc = acc_eps * (1.0 + k_len / 64.0) * absref64
    floor = 2.0 ** -24 * (rnd_eps / F16_EPS)
    tol = rnd_eps * ref64.abs() + acc + floor
    if extra64 is not None:
        extra64 = extra64.double().cpu()
        assert extra64.shape == ref64.shape and bool((extra64 >= 0).all()), what
        tol = tol + extra64
    ratio = (err.abs() / tol)
    worst = int(ratio.argmax())
    excess = (err.abs() - rnd_eps * ref64.abs() - floor).clamp_min(0)
    acc_ratio = float((excess / acc.clamp_min(1e-300)).max()) if bool((acc > 0).any()) else 0.0
    extra_ratio = 0.0
    if extra64 is not None and bool((extra64 > 0).any()):
        extra_ratio = float((excess / extra64.clamp_min(1e-300)).max())
    assert float(ratio.max()) <= 1.0, "%s: err/tol %.3g at flat index %d (got %r, ref %r, absref %r)" % (
        what, float(ratio.max()), worst, float(got64.reshape(-1)[worst]), float(ref64.reshape(-1)[worst]),
        float(absref64.reshape(-1)[worst]))
    normal = ref64.abs() >= 2.0 ** -14
    n = int(normal.sum())
    if n >= 256:
        bias = float((err[normal] * ref64[normal].sign()).mean())
        step = rnd_eps * float(ref64[normal].abs().mean())
        limit = 0.25 * step + acc_eps * float(absref64[normal].mean())
        assert abs(bias) <= limit, "%s: mean signed error %.3g exceeds %.3g (biased rounding)" % (what, bias, limit)
    return float(ratio.max()), acc_ratio, extra_ratio



# ---- float64 references shared by the kernel matrices and the per-launch workload audit ---------------------------
# Bound of a run of K fp32 operations (additions, fused multiply-adds) on terms whose magnitudes sum to A:
# |err| <= K * 2^-24 * A.  Expressed through the comparator's accumulation term acc_eps * (1 + K / 64) * A with
# acc_eps = 2^-18 = 64 * 2^-24, i.e. (64 + K) * 2^-24 * A: the K roundings plus up to 64 further roundings of
# intermediates of the same magnitude (divisions by the count, the final multiply-add, conversions).
SUM_EPS = 2.0 ** -18
# Attention error bound: the tensor-core kernels round the probabilities to f16 before P.V while the row sum l keeps
# them in fp32, so an output may move by ~2 * 2^-11 of sum_j p_j |v_j| on top of its own rounding, independent of Nk;
# ACC_EPS_ATTN (with k_len = 0) allows twice that (absref = p.|v| + |q|).  A probability below 2^-14 of its row's
# running maximum is an f16 subnormal, rounded to the absolute step 2^-24 instead: attn_p16_floor64 charges half that
# step for every key (a sharp softmax whose winning key has v ~ 0 leaves o made of such probabilities).
ACC_EPS_ATTN = 2.0 ** -9
# fp32 attention (attention_kernel<float, D>, attention_wide_simt_kernel<float, D>: fp32 storage, fp32 maths, P never
# rounded to f16).  Per query the kernel forms o = (sum_j p_j v_j) / l, l = sum_j p_j, online over key tiles of 32:
#   s_j = sum_c fmaf(q_c * scale, k_c, .)         D + 1 roundings of terms of magnitude S_j = |scale| |q|.|k_j|
#   p_j = __expf(s_j - m)                         the subtraction (one rounding of |x_j|, x_j = s_j - m) and __expf,
#                                                 within (2 + 1.173 |x_j|) ulp (as act_err64 charges it)
#   l, acc rescaled by __expf(m_old - m_new) once per tile (the same factor on both: it cancels in acc / l), summed
#   by fmaf over Nk keys (acc) and a 32-lane shuffle tree plus one add per tile (l), then acc * (1 / l) (+ q).
# The relative errors e_j of p_j move o as attn_score_extra64 bounds (to first order: sum_j p_j e_j |v_j| +
# (sum_j p_j e_j) sum_j p_j |v_j|).  The tensor-core kernels form the same fp32 scores, so their bound carries it too.
# The sums, rescales and the final division take at most Nk + 3 ceil(Nk / 32) + 10 roundings of p.|v| + |q|; with
# k_len = Nk the comparator's accumulation term acc_eps (1 + Nk / 64) = (128 + 2 Nk) 2^-24 covers them.
ACC_EPS_ATTN_F32 = 2.0 ** -17
# Lipschitz constants of the activations (largest slope)
LIP = {"none": 1.0, "relu": 1.0, "swish": 1.1, "gelu": 1.13, "sigmoid": 0.25, "hswish": 1.5}


def act64(v, act):
    if act in (None, "none"):
        return v
    if act == "relu":
        return v.clamp_min(0)
    if act == "swish":
        return v * torch.sigmoid(v)
    if act == "gelu":
        return 0.5 * v * (1 + torch.erf(v / math.sqrt(2.0)))
    if act == "sigmoid":
        return torch.sigmoid(v)
    if act == "hswish":
        return v * (v + 3).clamp(0, 6) / 6
    raise ValueError(act)


def act_err64(v, act):
    """Error of apply_act (pv_common.cuh) evaluated in fp32 at the exact argument v.  __expf(x) is within
    2 + floor(1.173 |x|) ulp (<= 2^-23 relative each) of e^x; the sigmoid factor s (1 - s) carries that relative
    error into 1 / (1 + e).  erff is within 2 ulp.  Each further fp32 operation adds one rounding of the result."""
    U = F32_EPS
    a, y = v.abs(), act64(v, act).abs()
    if act in (None, "none", "relu"):
        return torch.zeros_like(v)
    s = torch.sigmoid(v)
    rel_e = (2 + 1.173 * a) * 2.0 ** -23
    if act == "swish":
        return a * s * (1 - s) * rel_e + 2 * U * y
    if act == "sigmoid":
        return s * (1 - s) * rel_e + 2 * U * s
    if act == "gelu":
        erf = torch.erf(v / math.sqrt(2.0))
        return 0.5 * a * (2.0 ** -22 * erf.abs() + 0.5 * U + U * (1 + erf).abs()) + 2 * U * y
    return U * a * (a + 3) / 6 + 2 * U * y                      # hswish: x + 3, x * clamp, / 6


def conv_ref64(x, w, scale, bias, stride, padding, dilation, groups, act, res):
    """(ref64, absref64) of y = act(conv(x, w) * scale + bias (+ res)) in float64 on x's device; absref is taken
    before the activation (the magnitude the pre-activation sum is built from)."""
    dev = x.device
    x64, w64 = x.double(), w.double().to(dev)
    sc, bi = scale.double().to(dev).view(1, -1, 1, 1, 1), bias.double().to(dev).view(1, -1, 1, 1, 1)
    y = F.conv3d(x64, w64, None, stride, padding, dilation, groups) * sc + bi
    a = F.conv3d(x64.abs(), w64.abs(), None, stride, padding, dilation, groups) * sc.abs() + bi.abs()
    if res is not None:
        y = y + res.double()
        a = a + res.double().abs()
    return act64(y, act), a


def attn_probs64(q, k, scale, mask=None):
    """Float64 softmax(scale q k^T) over the keys, q [B, H, Nq, D], k [B, H, Nk, D]; mask (bool [B, Nk]): keys where
    it is False take no weight, and a query without a valid key has all-zero probabilities."""
    s = (q.double() * scale) @ k.double().transpose(-2, -1)
    if mask is None:
        return s.softmax(-1)
    s = s.masked_fill(~mask.to(s.device)[:, None, None, :], float("-inf"))
    return s.softmax(-1).nan_to_num(0.0)


def attn_ref64(q, k, v, scale, resid, normalize=0, mask=None):
    """q: [..., Nq, D], k / v: [..., Nk, D] (the operands the kernel read) -> (ref64, absref64) with
    absref = P . |v| (+ |q|).  normalize = 0: P = softmax(scale q k^T) (masked keys as attn_probs64); 1: the linear mode
    P = scale q k^T / Nk, whose magnitude is |P| = |scale| |q| |k|^T / Nk."""
    q64, k64, v64 = q.double(), k.double(), v.double()
    if normalize:
        nk = k.shape[-2]
        p = ((q64 * scale) @ k64.transpose(-2, -1)) / nk
        absp = (q64.abs() @ k64.abs().transpose(-2, -1)) * abs(scale) / nk
    else:
        p = absp = attn_probs64(q64, k64, scale, mask)
    ref = p @ v64
    absref = absp @ v64.abs()
    if resid:
        ref, absref = ref + q64, absref + q64.abs()
    return ref, absref


def _score_err64(q, k, scale, mask):
    """(p, e): the float64 probabilities and a bound on the relative error of the kernel's fp32 probability of every
    key: D + 2 roundings of |scale| |q|.|k_j| in the score, one of |x_j| = |s_j - m| in the subtraction and the
    __expf error at x_j (masked keys and queries without a valid key: 0)."""
    q64, k64 = q.double(), k.double()
    s = (q64 * scale) @ k64.transpose(-2, -1)
    S = (q64.abs() * abs(scale)) @ k64.abs().transpose(-2, -1)
    p = attn_probs64(q64, k64, scale, mask)
    valid = p > 0
    x = torch.where(valid, s - s.masked_fill(~valid, float("-inf")).max(-1, keepdim=True).values, torch.zeros_like(s))
    x = x.abs()
    e = (q.shape[-1] + 2) * F32_EPS * S + F32_EPS * x + (2 + 1.173 * x) * 2.0 ** -23
    return p, torch.where(valid, e, torch.zeros_like(e))


def attn_score_extra64(q, k, v, scale, mask=None):
    """extra64 of softmax attention: the error of the kernel's fp32 scores and __expf probabilities (_score_err64)
    carried to o, for q [..., Nq, D], k / v [..., Nk, D].  With p_j off by a factor within exp(+-e_j),
    |o' - o| <= (sum_j p_j E_j |v_j| + (sum_j p_j E_j) |o|) / sum_j p_j exp(-e_j), E_j = exp(e_j) - 1, and
    |o| <= sum_j p_j |v_j|.  Where the logits are so large that e_j reaches 1 (fp32 cannot resolve which key wins)
    the bound grows accordingly."""
    p, e = _score_err64(q, k, scale, mask)
    pE = p * torch.expm1(e)
    av = v.double().abs()
    den = (p * torch.exp(-e)).sum(-1, keepdim=True)
    den = torch.where(den > 0, den, torch.ones_like(den))         # queries without a valid key: o = 0 exactly
    return (pE @ av + pE.sum(-1, keepdim=True) * (p @ av)) / den


def attn_weights_err64(q, k, scale, mask=None):
    """(ref, err) of the head-averaged attention weights [B, Nq, Nk] pv_attention_weights writes in fp32 from the
    row log-sum-exp of the attention launch: w_j = sum_h __expf(s_hj - lse_h) / H.  Each term carries the relative
    error of its score and __expf (_score_err64), the score error of the row maximum inside lse, and lse's own error:
    log of a row sum with at most Nk + 3 ceil(Nk / 32) + 10 roundings, logf and the add (4 roundings of |lse|).  The
    sum over heads and the division take H + 1 roundings of w."""
    p, e = _score_err64(q, k, scale, mask)
    H, Nk = q.shape[1], k.shape[-2]
    s = (q.double() * scale) @ k.double().transpose(-2, -1)
    lse = torch.logsumexp(s if mask is None else s.masked_fill(~mask.to(s.device)[:, None, None, :], float("-inf")), -1,
                          keepdim=True).nan_to_num(0.0, neginf=0.0)
    S = (q.double().abs() * abs(scale)) @ k.double().abs().transpose(-2, -1)
    Smax = torch.where(p > 0, S, torch.zeros_like(S)).max(-1, keepdim=True).values
    e_lse = (q.shape[-1] + 2) * F32_EPS * Smax + (Nk + 3 * -(-Nk // 32) + 10) * F32_EPS + 4 * F32_EPS * lse.abs()
    w = p.mean(1)
    return w, (p * (e + e_lse)).mean(1) + (H + 1) * F32_EPS * w


def lstm_ref64(G, W, lengths, H, nd, h16=False):
    """float64 restatement of the LSTM recurrence on the operands the kernel received: G [B][T][nd*4H] (input
    projection plus biases), W^T [nd][H][4H]; the first lengths[b] steps of row b, walked forward (and backward by the
    second direction).  h16: h enters the product rounded to f16 (the tensor-core operand of the cluster kernel).
    Returns (h_n [B, nd*H], err): err bounds the kernel's fp32 error, propagated to first order step by step:
      z = G + h W        H + 2 roundings of |G| + |h| |W|, the carried error of h through |W| (and h's f16 rounding)
      sigmoid = 1 / (1 + expf(-z)), tanhf    each within 2 ulp, and the slope s (1 - s) or 1 - t^2 times z's error
      c = f c + i g, h = o tanhf(c)          the carried errors of f, c, i, g, o and 3 / 2 roundings."""
    G, W = G.double().cpu(), W.double().cpu()
    U = F32_EPS
    B = G.shape[0]
    out = torch.zeros(B, nd * H, dtype=torch.float64)
    err = torch.zeros(B, nd * H, dtype=torch.float64)
    for b in range(B):
        n = int(lengths[b])
        for d in range(nd):
            h, c, eh, ec = (torch.zeros(H, dtype=torch.float64) for _ in range(4))
            Wd = W[d]
            for s_ in range(n):
                t = s_ if d == 0 else n - 1 - s_
                g_t = G[b, t, d * 4 * H:(d + 1) * 4 * H]
                hop = h.half().double() if h16 else h
                z = g_t + hop @ Wd
                ez = (H + 2) * U * (g_t.abs() + h.abs() @ Wd.abs()) + eh @ Wd.abs()
                if h16:
                    ez = ez + F16_EPS * (h.abs() @ Wd.abs())
                sg = z.sigmoid()
                es = sg * (1 - sg) * (ez + 4 * U) + 3 * U * sg
                tg = z.tanh()
                et = (1 - tg * tg) * ez + 4 * U * tg.abs()
                i, f, gg, o = sg[:H], sg[H:2 * H], tg[2 * H:3 * H], sg[3 * H:]
                ei, ef, eg, eo = es[:H], es[H:2 * H], et[2 * H:3 * H], es[3 * H:]
                c_new = f * c + i * gg
                ec = (f.abs() * ec + c.abs() * ef + i.abs() * eg + gg.abs() * ei
                      + 3 * U * ((f * c).abs() + (i * gg).abs()))
                c = c_new
                tc = c.tanh()
                h = o * tc
                eh = tc.abs() * eo + o.abs() * ((1 - tc * tc) * ec + 4 * U * tc.abs()) + 2 * U * h.abs()
            out[b, d * H:(d + 1) * H] = h
            err[b, d * H:(d + 1) * H] = eh
    return out, err


def attn_p16_floor64(v, Nq, mask=None):
    """extra64 of the f16 rounding of subnormal probabilities (see ACC_EPS_ATTN): 2^-25 sum_j |v_j| over the valid keys
    for every query (the probabilities are relative to the row maximum, so the row sum l >= 1), v [B, H, Nk, D]."""
    av = v.double().abs()
    if mask is not None:
        av = av * mask.to(av.device)[:, None, :, None]
    return (2.0 ** -25 * av.sum(-2, keepdim=True)).expand(*v.shape[:2], Nq, v.shape[-1])


def prologue_conv_ref64(x, pre_s, pre_b, w, scale, bias, stride, padding, dilation=(1, 1, 1)):
    """The depthwise pooling conv with the BatchNorm + GELU prologue (pv_conv3d_desc.pre_*): conv(GELU(x * pre_s +
    pre_b), w) * scale + bias in float64 on x's device, the prologue applied to in-bounds inputs before the zero
    padding.  Returns (ref, absref, u, pre): u = GELU(pre) is what the stencil reads, pre its argument."""
    C = x.shape[1]
    view = (1, C, 1, 1, 1)
    pre = x.double() * pre_s.double().to(x.device).view(view) + pre_b.double().to(x.device).view(view)
    u = act64(pre, "gelu")
    ref, absref = conv_ref64(u, w, scale, bias, stride, padding, dilation, C, "none", None)
    return ref, absref, u, pre


def _conv_bn(x, w, scale, bias, stride=1, padding=0):
    return F.conv3d(x, w, None, stride, padding) * scale.view(1, -1, 1, 1, 1) + bias.view(1, -1, 1, 1, 1)


def fused_block_ref64(x, wa, wb, wc, ws, folds, kt, sb, act):
    """The fused bottleneck block in float64 on the f16-grid operands and the exact fp32 folded BatchNorm the kernel
    uses.

    Returns (y, A, B, Y, prop): y the result; A, B, Y the magnitude sums of a, b and y (the same sums over |x|, |w|,
    |scale| and |bias|, plus |shortcut| for Y); prop the error of the kernel's f16 intermediates a and b propagated to
    y.  Each intermediate may be off by one f16 rounding plus its fp32 accumulation term plus what it inherits (relu
    is 1-Lipschitz, and a is exactly 0 outside the image where conv_b pads):
      ea = F16_EPS |a| + ACC(Ka) A + 2^-24
      eb = F16_EPS |b| + ACC(Kb) B + |sb| conv_b(ea, |wb|) + 2^-24
      prop = |sc| conv_c(eb, |wc|)
    with ACC(K) = 2^-20 (1 + K / 64).  The caller compares with assert_close_to_f64(got, y, Y, Kc + Ks, extra64=prop).
    Runs on x's device."""
    dev = x.device
    f64 = [None if t is None else t.double().to(dev) for t in folds]
    sa, ba, sbn, bbn, sc, bc, ssc, bsc = f64
    x64 = x.double()
    wa, wb, wc = (t.double().to(dev) for t in (wa, wb, wc))
    pa, pb, st = (kt // 2, 0, 0), (0, 1, 1), (1, sb, sb)
    cin, cmid = x.shape[1], wa.shape[0]

    def acc(k):
        return ACC_EPS * (1.0 + k / 64.0)
    a = _conv_bn(x64, wa, sa, ba, 1, pa).clamp_min(0)
    A = _conv_bn(x64.abs(), wa.abs(), sa.abs(), ba.abs(), 1, pa)
    b = _conv_bn(a, wb, sbn, bbn, st, pb).clamp_min(0)
    B = _conv_bn(a, wb.abs(), sbn.abs(), bbn.abs(), st, pb)
    ea = F16_EPS * a + acc(kt * cin) * A + 2.0 ** -24
    eb = (F16_EPS * b + acc(9 * cmid) * B + sbn.abs().view(1, -1, 1, 1, 1) * F.conv3d(ea, wb.abs(), None, st, pb)
          + 2.0 ** -24)
    del ea
    if ws is None:
        short = x64[:, :, :, ::sb, ::sb]
        S = short.abs()
    else:
        ws = ws.double().to(dev)
        short = _conv_bn(x64, ws, ssc, bsc, st)
        S = _conv_bn(x64.abs(), ws.abs(), ssc.abs(), bsc.abs(), st)
    y = act64(_conv_bn(b, wc, sc, bc) + short, act)
    Y = _conv_bn(b, wc.abs(), sc.abs(), bc.abs()) + S
    prop = sc.abs().view(1, -1, 1, 1, 1) * F.conv3d(eb, wc.abs())
    return y, A, B, Y, prop


def ln_ref64(v, gamma, beta, gps, depth, eps):
    """(ref, absref, K, extra) of LayerNorm over the last dim of v [rows, groups, C]; group j uses set j // gps of
    gamma / beta [sets, C].  The kernel sums a row at depth ``depth`` (see the LayerNorm rows of the CUDA-core
    matrix); the mean is off by (depth + 1) 2^-24 mean|x|, rsqrtf by 2 ulp; the output takes <= 4 roundings."""
    v = v.double()
    G = v.shape[1]
    idx = torch.arange(G, device=v.device) // gps
    g64, b64 = gamma.double().to(v.device)[idx], beta.double().to(v.device)[idx]
    mu = v.mean(-1, keepdim=True)
    var = ((v - mu) ** 2).mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(var + float(torch.tensor(eps, dtype=torch.float32)))
    xh = (v - mu) * rstd
    ref = xh * g64 + b64
    m_abs = v.abs().mean(-1, keepdim=True)
    absref = g64.abs() * (rstd * m_abs + xh.abs()) + b64.abs()
    dmu = (depth + 1) * F32_EPS * m_abs * rstd
    extra = (g64 * xh).abs() * (2.0 ** -22 + 0.5 * dmu ** 2)
    return ref, absref, depth + 5, extra


def ln_dispatch(C, aligned=True):
    """(launch, lanes per row, chunks per lane) pv_layernorm_sets picks."""
    chunks = -(-C // 8)
    lg = 2
    while (1 << lg) < chunks and lg < 5:
        lg += 1
    nch = -(-chunks // (1 << lg))
    if nch <= 3 and aligned:
        return "layernorm_reg_kernel", 1 << lg, nch
    return "layernorm_kernel", 32, -(-chunks // 32)


# ---- RoIAlign (pv_roi_align_fwd): torchvision's fp32 sampling geometry and the float64 reference ------------------
def round32(q):
    """A Fraction rounded to the nearest float32 (ties to even), without double rounding through float64."""
    r = np.float32(float(q))
    best = r
    for cand in (np.nextafter(r, np.float32(-np.inf)), np.nextafter(r, np.float32(np.inf))):
        d0, d1 = abs(Fraction(float(best)) - q), abs(Fraction(float(cand)) - q)
        if d1 < d0 or (d1 == d0 and int(np.array(cand).view(np.int32)) % 2 == 0):
            best = cand
    return best


def fma32(a, b, c):
    return round32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def roi_geometry(box, H, W, ph_n, pw_n, scale, sr, contract=False, mutation=None):
    """torchvision's fp32 sampling geometry of one RoI (oracle.interp.roi_align_ref's arithmetic): per bin, the list
    of kept samples (y_low, x_low, y_high, x_high, w1, w2, w3, w4), the count, and (grid_h, grid_w).
    contract=True evaluates `end * scale - start` and `start + ph * bin` as single-rounding FMAs, as nvcc contracts
    them unless told not to; mutation injects a known bug."""
    s = np.float32(scale)
    x1, y1, x2, y2 = (np.float32(v) for v in box[1:5])
    sw, sh = x1 * s, y1 * s
    if contract:
        rw, rh = fma32(x2, s, -sw), fma32(y2, s, -sh)
    else:
        rw, rh = x2 * s - sw, y2 * s - sh
    rw, rh = max(rw, np.float32(1)), max(rh, np.float32(1))
    bh, bw = rh / np.float32(ph_n), rw / np.float32(pw_n)
    rnd = np.floor if mutation == "floor" else np.ceil
    gh = sr if sr > 0 else int(rnd(rh / np.float32(ph_n)))
    gw = sr if sr > 0 else int(rnd(rw / np.float32(pw_n)))
    count = max(gh * gw, 1)
    half = np.float32(0) if mutation == "iy" else np.float32(0.5)
    bins = []
    for ph in range(ph_n):
        st_y = fma32(np.float32(ph), bh, sh) if contract else sh + np.float32(ph) * bh
        for pw in range(pw_n):
            st_x = fma32(np.float32(pw), bw, sw) if contract else sw + np.float32(pw) * bw
            samples = []
            for iy in range(gh):
                yy0 = st_y + (np.float32(iy) + half) * bh / np.float32(gh)
                for ix in range(gw):
                    xx = st_x + (np.float32(ix) + half) * bw / np.float32(gw)
                    yy = yy0
                    y_out = (yy >= H) if mutation == "ge_H" else (yy > H)
                    if yy < -1 or y_out or xx < -1 or xx > W:
                        continue
                    yy, xx = max(yy, np.float32(0)), max(xx, np.float32(0))
                    yl, xl = int(yy), int(xx)
                    if yl >= H - 1:
                        yh = yl = H - 1
                        yy = np.float32(yl)
                    else:
                        yh = yl + 1
                    if xl >= W - 1:
                        xh = xl = W - 1
                        xx = np.float32(xl)
                    else:
                        xh = xl + 1
                    ly, lx = yy - np.float32(yl), xx - np.float32(xl)
                    hy, hx = np.float32(1) - ly, np.float32(1) - lx
                    samples.append((yl, xl, yh, xh, hy * hx, hy * lx, ly * hx, ly * lx))
            bins.append(samples)
    return bins, count, (gh, gw)


def roi_ref64(x, rois, geom, mutation=None, emulate=False, contract=False):
    """x [N, H, W, C], geom (pooled h, pooled w, spatial scale, sampling ratio); returns (ref, absref) [K, ph, pw, C]
    in float64 (weights from the fp32 geometry), or the fp32 emulation in the kernel's order (acc += w1 v1 + w2 v2 +
    w3 v3 + w4 v4 per sample, then / count).  Invalid batch indices give zeros.  contract: the geometry as nvcc
    contracts it (see roi_geometry)."""
    N, H, W, C = x.shape
    ph_n, pw_n, scale, sr = geom
    dt = torch.float32 if emulate else torch.float64
    X = x.to(dt)
    out = torch.zeros(len(rois), ph_n * pw_n, C, dtype=dt)
    absout = torch.zeros(len(rois), ph_n * pw_n, C, dtype=torch.float64)
    for k, box in enumerate(rois):
        n = int(box[0])
        if not 0 <= n < N:
            continue
        bins, count, _ = roi_geometry(box, H, W, ph_n, pw_n, scale, sr, contract=contract, mutation=mutation)
        Xn = X[n]
        for b, samples in enumerate(bins):
            acc = torch.zeros(C, dtype=dt)
            mag = torch.zeros(C, dtype=torch.float64)
            for (yl, xl, yh, xh, w1, w2, w3, w4) in samples:
                v = (Xn[yl, xl], Xn[yl, xh], Xn[yh, xl], Xn[yh, xh])
                acc = acc + (float(w1) * v[0] + float(w2) * v[1] + float(w3) * v[2] + float(w4) * v[3])
                if not emulate:
                    mag = mag + sum(float(w) * t.abs() for w, t in zip((w1, w2, w3, w4), v))
            out[k, b] = acc / float(count)
            absout[k, b] = mag / float(count)
    shape = (len(rois), ph_n, pw_n, C)
    return out.view(shape), absout.view(shape)


def roi_acc_eps(rois, geom, H, W):
    """About 4 roundings per sample (the four products summed, the accumulation) plus one for the division."""
    grids = [roi_geometry(b, H, W, *geom)[2] for b in rois]
    return (4 * max(gh * gw for gh, gw in grids) + 1) * F32_EPS



# ---- per-launch audit of a compiled plan (tests/test_gpu_workload_audit.py, tests/test_gpu_model_audit.py) --------
# Each op of a plan carries a record of what it computes (Plan.op_spec).  audit_plan walks the plan on one stream,
# reads each op's inputs just before it runs, runs it, asserts the launched instances belong to the family the record
# implies, and compares the output with the same operation in float64 under the kernel-matrix bounds; the stored
# dtype of each output sets its rounding term (f16 or fp32), and the reference multiplies the operands the kernel read
# (the weights in the plan's storage dtype, as engine/packing.py packs them).
NO_VALUE_SUFFIXES = (".se_zero",)        # ops that produce no value of their own: the clear of an SE-sum accumulator

_TC = ("conv3d_igemm_kernel<", "conv3d_igemm_gather_kernel<", "conv3d_igemm_grouped_kernel<",
       "conv3d_stem_rows_kernel<", "conv3d_stem_stream_kernel<")
_DW = ("dwconv3d_lane_kernel<", "dwconv_temporal_kernel<", "dwconv3d_tile_kernel<", "dwconv_plane_kernel<",
       "dwconv3d_kernel<", "dwconv3d_w4_kernel<")
_LN = ("layernorm_reg_kernel", "layernorm_kernel")
_ATTN = ("attention_wgmma_kernel<", "attention_mma_kernel<", "attention_kernel<", "attention_wide_kernel<",
         "attention_wide_simt_kernel<")
_CVT = ("ncdhw_to_ndhwc_kernel", "ncdhw_to_ndhwc_padw_kernel", "ncdhw_f32_to_ndhwc4_padw_kernel")
# instance families a record's launch may take, by record kind (conv: by route).  The prefixes cover the f16 and the
# fp32 instances (conv3d_direct_kernel<float>, dwconv3d_kernel<float>, dwconv3d_w4_kernel<float,..>,
# attention_kernel<float,..>, attention_wide_simt_kernel<float,..>); FAMILY_F32 lists the fp32 ones an f32 plan takes.
FAMILY = {
    "tcgen05": _TC, "grouped": _TC, "stem_stream": _TC, "direct": ("conv3d_direct_kernel<",),
    "depthwise": _DW + ("channel_sum_kernel",), "token_conv": _DW, "channel_affine": _DW,
    "to_ndhwc": _CVT, "tokens_in": _CVT, "to_f32": ("ndhwc_to_ncdhw_kernel",), "copy": ("copy_rows_kernel",),
    "tap_sum": ("temporal_tap_sum_kernel",), "fused_block": ("bottleneck_fused_kernel<",),
    "pool": ("pool3d_kernel", "global_pool_kernel"), "head_reduce": ("head_reduce_kernel",),
    "se_gate": ("se_gate_kernel",), "scale_act": ("scale_act_kernel",), "pos_cls": ("add_pos_cls_kernel",),
    "layernorm": _LN + ("add_layernorm_kernel",), "layernorm_sets": _LN, "add_layernorm": ("add_layernorm_kernel",),
    "attention": _ATTN, "copy_cls": ("copy_rows_kernel",), "roi_align": ("roi_align_kernel<",),
    "mask_force_first": ("mask_force_first_kernel",), "masked_pool": ("masked_pool_kernel<",),
    "masked_default": ("masked_default_kernel<",), "reduce_fusion": ("reduce_fusion_kernel<",),
    "copy_tokens": ("copy_rows_kernel",),
    "attention_masked": ("attention_wgmma_masked_kernel<", "attention_mma_masked_kernel<", "attention_masked_kernel<"),
    "attention_weights": ("attention_weights_kernel<",),
    "lstm": ("lstm_recurrence_kernel<", "lstm_cluster_kernel"),
}
_DW32 = ("dwconv3d_kernel<float", "dwconv3d_w4_kernel<float,")       # <float>, <float,pre>, <float,kt,sw>(,pre)
FAMILY_F32 = {"direct": ("conv3d_direct_kernel<float>",), "depthwise": _DW32 + ("channel_sum_kernel",),
              "token_conv": _DW32, "channel_affine": _DW32,
              "attention": ("attention_kernel<float,", "attention_wide_simt_kernel<float,"),
              "attention_masked": ("attention_masked_kernel<float,",),
              "attention_weights": ("attention_weights_kernel<float>",),
              "masked_pool": ("masked_pool_kernel<float,",), "masked_default": ("masked_default_kernel<float>",),
              "reduce_fusion": ("reduce_fusion_kernel<float,",), "lstm": ("lstm_recurrence_kernel<float>",)}

_ACT_NAMES = ("none", "relu", "swish", "gelu", "sigmoid", "hswish")       # by the library's ACT_* value


def supported(spec):
    """True when the audit has a reference for this record."""
    return spec is not None and (spec["route"] if spec["kind"] == "conv" else spec["kind"]) in FAMILY


def family_of(spec, f32=False):
    key = spec["route"] if spec["kind"] == "conv" else spec["kind"]
    return FAMILY_F32.get(key, FAMILY[key]) if f32 else FAMILY[key]


def record_io(spec):
    """(plan tensors the op reads, plan tensors it writes) according to its record."""
    k = spec["kind"]
    if k == "conv":
        ins = [spec["x"]] + [t for t in (spec["residual"],) if t is not None]
        if spec["addend"] is not None:
            ins.append(spec["addend"][0])
        sums = [spec["se_sums"]] if spec["se_sums"] is not None else []      # accumulated onto: read and written
        return ins + sums, [spec["y"]] + sums
    if k in ("to_ndhwc", "tokens_in"):
        return [], [spec["y"]]
    if k in ("head_reduce", "to_f32"):
        return [spec["x"]], [spec["out"]]
    if k == "se_gate":
        return [spec["sums"]], [spec["gate"]]
    if k == "channel_sum":
        return [spec["x"]], [spec["sums"]]
    if k == "scale_act":
        return [spec["x"]] + ([spec["gate"]] if spec["gate"] is not None else []), [spec["y"]]
    if k == "add_layernorm":
        return [spec["a"], spec["br"]], [t for t in (spec["s"], spec["y"]) if t is not None]
    if k == "layernorm_sets":
        return ([spec["x"]] if spec["cls"] else []) + [spec["y"]], [spec["y"]]
    if k == "attention":
        return [spec["q"], spec["k"], spec["v"]], [spec["o"]]
    if k == "mask_force_first":
        return list(spec["mask"].io()), list(spec["out"].io())
    if k in ("masked_pool", "masked_default"):
        return [spec["x"]] + list(_mask_io(spec["mask"])), [spec["y"]]
    if k == "reduce_fusion":
        return list(spec["parts"]), [spec["y"]]
    if k == "attention_masked":
        return [spec["q"], spec["k"], spec["v"]] + list(spec["mask"].io()), \
            [spec["o"]] + ([spec["lse"]] if spec["lse"] is not None else [])
    if k == "attention_weights":
        return [spec["q"], spec["k"], spec["lse"]] + list(spec["mask"].io()), [spec["w"]]
    if k == "lstm":
        return [spec["g"]] + list(_mask_io(spec["mask"])), [spec["y"]]
    return [spec["x"]], [spec["y"]]


def _mask_io(mask):
    return mask.io() if mask is not None else ()


def mask_bool(mask, clips):
    """The (n, T) bool mask a MaskRef holds for the selected clips (None: every step valid)."""
    if mask is None:
        return None
    return record_rows(None, mask)[clips] != 0


def io_buffers(items):
    """ids of the plan buffers behind a list of TRefs / Bufs."""
    from .engine.plan import Buf
    return {id(t if isinstance(t, Buf) else t.buf) for t in items if t is not None and
            (isinstance(t, Buf) or t.buf is not None)}


def io_problems(plan):
    """[(op name, "reads" | "writes")] where a record reads or writes a buffer its declared I/O (which orders the
    lanes) does not list."""
    bad = []
    for (n, _), s, io in zip(plan.ops, plan.op_spec, plan.op_io):
        if io is None or s is None:
            continue
        ins, outs = record_io(s)
        if not io_buffers(ins) <= io_buffers(io[0]):
            bad.append((n, "reads"))
        if not io_buffers(outs) <= io_buffers(io[1]):
            bad.append((n, "writes"))
    return bad


# ---- declared footprints, the lanes' happens-before order and the footprint walk ------------------------------------
# (tests/test_plan_schedule.py, tests/test_gpu_launch_footprint.py)
class Footprint:
    """A set of elements of plan buffers.  Per buffer, blocks (base, n, n_stride, rows, row_stride, width), each the
    elements base + i * n_stride + r * row_stride + c for i < n, r < rows, c < width (in elements of the buffer)."""

    def __init__(self):
        self.blocks = {}            # id(buf) -> (buf, [block])

    def add(self, buf, block):
        self.blocks.setdefault(id(buf), (buf, []))[1].append(tuple(int(v) for v in block))

    def bufs(self):
        return [b for b, _ in self.blocks.values()]

    def __contains__(self, buf):
        return id(buf) in self.blocks

    def extent(self, buf):
        """One past the last element of ``buf`` the footprint covers (0 when it has none)."""
        return max([base + (n - 1) * ns + (r - 1) * rs + w for base, n, ns, r, rs, w in self.blocks[id(buf)][1]
                    if n and r and w] or [0])

    def mark(self, buf, out, offset=0, scale=1):
        """Set True the elements of ``buf`` the footprint covers in the flat bool tensor ``out``, which holds the
        buffer from position ``offset`` in units of 1 / ``scale`` of its elements (scale = element size: a byte map)."""
        for base, n, ns, r, rs, w in self.blocks.get(id(buf), (None, ()))[1]:
            if n and r and w:
                out.as_strided((n, r, w * scale), (ns * scale, rs * scale, 1), offset + base * scale).fill_(True)

    def mask(self, buf):
        """[numel] bool CPU tensor of the elements of ``buf`` the footprint covers."""
        m = torch.zeros(max(buf.numel, self.extent(buf)), dtype=torch.bool)
        self.mark(buf, m)
        return m


def footprint(item, span=None):
    """The elements of its buffer a TRef, Buf or MaskRef covers.  A TRef covers its N * npos rows at row_stride,
    channels [ch_off, ch_off + Cp) (the pad channels are part of the tensor); W-padded stem rows (padw) their whole
    physical rows.  span: a slice of each sample's npos rows (token_span), else all of them.  A Buf or a plan-owned
    mask covers its whole buffer."""
    from .engine.plan import Buf, MaskRef, TRef
    fp = Footprint()
    if isinstance(item, MaskRef):
        item = item.buf
    if isinstance(item, Buf):
        fp.add(item, (0, 1, 0, 1, 0, item.numel))
    elif isinstance(item, TRef) and item.padw is not None:
        fp.add(item.buf, (0, 1, 0, 1, 0, item.N * item.T * item.H * item.padw[1] * item.Cp))
    elif isinstance(item, TRef):
        r0, r1, _ = (span or slice(None)).indices(item.npos)
        fp.add(item.buf, (item.ch_off + r0 * item.row_stride, item.N, item.npos * item.row_stride, max(r1 - r0, 0),
                          item.row_stride, item.Cp))
    return fp


def op_footprints(plan, i):
    """(read footprint, write footprint) of op i from its declared I/O (Plan.op_io), each TRef narrowed to the token
    rows its record reads / writes (token_span); None when the op declares no I/O."""
    io = plan.op_io[i]
    if io is None:
        return None
    spec = plan.op_spec[i]
    out = []
    for items, role in ((io[0], "read"), (io[1], "write")):
        fp = Footprint()
        for t in items:
            span = token_span(spec, t, role) if spec is not None and hasattr(t, "ch_off") else None
            for buf, blocks in footprint(t, span).blocks.values():
                for blk in blocks:
                    fp.add(buf, blk)
        out.append(fp)
    return tuple(out)


def happens_before(plan, waits=None):
    """Vector clocks of the plan's multi-lane run (Plan.run): hb[i][M] is the last op of lane M ordered before op i or
    op i itself.  Edges: stream order within a lane, the cross-lane waits (plan.sched["waits"], or ``waits``); every
    lane starts after the fork, which precedes every op.  Op j reaches op i iff hb[i].get(lane of j, -1) >= j."""
    waits = plan.sched["waits"] if waits is None else waits
    hb, last = [], {}
    for i, L in enumerate(plan.op_lane):
        c = dict(hb[last[L]]) if L in last else {}
        for j in waits[i]:
            assert j < i, "op %d waits for a later op %d" % (i, j)
            for M, k in hb[j].items():
                if c.get(M, -1) < k:
                    c[M] = k
        c[L] = i
        hb.append(c)
        last[L] = i
    return hb


def schedule_conflicts(plan, waits=None):
    """[(i, j, hazard, message)]: pairs of ops i < j on different lanes that no path of the happens-before graph
    orders although they conflict: their declared footprints share an element and at least one of them writes it
    (RAW, WAR or WAW), or one of them declares no I/O (it may touch anything)."""
    hb = happens_before(plan, waits)
    lane = plan.op_lane
    names = [n for n, _ in plan.ops]
    fps = [op_footprints(plan, i) for i in range(len(plan.ops))]
    buf_no = {id(b): k for k, b in enumerate(plan.bufs)}
    ordered = lambda j, i: hb[i].get(lane[j], -1) >= j        # noqa: E731

    def msg(i, j, what):
        return "op %d %s (lane %d) and op %d %s (lane %d): %s, and no wait orders them" % (
            i, names[i], lane[i], j, names[j], lane[j], what)
    bad = []
    unknown = [i for i, f in enumerate(fps) if f is None]
    for u in unknown:
        for k in range(len(fps)):
            if k != u and lane[k] != lane[u]:
                i, j = min(u, k), max(u, k)
                if not ordered(i, j):
                    bad.append((i, j, "unknown", msg(i, j, "op %d declares no I/O" % u)))
    access = {}                                   # id(buf) -> [(op, is write, footprint)]
    for i, f in enumerate(fps):
        if f is None:
            continue
        for w, fp in ((False, f[0]), (True, f[1])):
            for b in fp.bufs():
                access.setdefault(id(b), []).append((i, w, fp, b))
    masks = {}

    def mask(i, w, fp, b):
        key = (i, w, id(b))
        if key not in masks:
            masks[key] = fp.mask(b)
        return masks[key]
    seen = set()
    for acc in access.values():
        for x in range(len(acc)):
            for y in range(x + 1, len(acc)):
                (i, wi, fi, b), (j, wj, fj, _) = sorted((acc[x], acc[y]), key=lambda a: a[0])
                if i == j or lane[i] == lane[j] or not (wi or wj) or ordered(i, j):
                    continue
                mi, mj = mask(i, wi, fi, b), mask(j, wj, fj, b)
                n = min(len(mi), len(mj))
                hit = torch.nonzero(mi[:n] & mj[:n])
                if len(hit) and (i, j, wi, wj) not in seen:
                    seen.add((i, j, wi, wj))
                    hazard = "WAW" if wi and wj else ("RAW" if wi else "WAR")
                    bad.append((i, j, hazard, msg(i, j, "%s on buffer %d (%d shared elements, first %d)" % (
                        hazard, buf_no.get(id(b), -1), len(hit), int(hit[0])))))
    return sorted(bad)


def legal_orders(plan):
    """Two topological orders of the plan's happens-before graph (stream order + waits) for a single-stream run: the
    highest lane's ops as early as their waits allow, and as late as they allow."""
    n = len(plan.ops)
    top = max(plan.op_lane)
    preds = [set(plan.sched["waits"][i]) for i in range(n)]
    prev = {}
    for i, L in enumerate(plan.op_lane):
        if L in prev:
            preds[i].add(prev[L])
        prev[L] = i
    orders = []
    for early in (True, False):
        done, order = set(), []
        heads = {}
        for i, L in enumerate(plan.op_lane):
            heads.setdefault(L, []).append(i)
        pos = {L: 0 for L in heads}
        while len(order) < n:
            ready = [ops[pos[L]] for L, ops in heads.items() if pos[L] < len(ops) and preds[ops[pos[L]]] <= done]
            assert ready, "the schedule has a cycle"
            pick = min(ready, key=lambda i: ((plan.op_lane[i] != top) if early else (plan.op_lane[i] == top), i))
            order.append(pick)
            done.add(pick)
            pos[plan.op_lane[pick]] += 1
        orders.append(order)
    return orders


def address_buffers(plan):
    """Plan buffers some op reads as addresses, counts or geometry: masks (MaskRef buffers) and every non-float
    buffer.  The footprint walk never fills them with a canary (an arbitrary value could steer an address); it checks
    them for undeclared writes only."""
    from . import _lib as L
    from .engine.plan import MaskRef
    out = {id(b) for b in plan.bufs if b.dt not in (L.PV_F16, L.PV_F32)}
    for spec in plan.op_spec:
        for v in (spec or {}).values():
            if isinstance(v, MaskRef) and v.buf is not None:
                out.add(id(v.buf))
    return out


# byte patterns the walk fills undeclared elements with: all ones (NaN in f16 and fp32), and 0x7B (f16 60768, fp32
# 1.3e36: large finite values), so that a value equal to one canary cannot hide a read
FOOTPRINT_CANARIES = (0xFF, 0x7B)
_ARENA_ALIGN = 1024            # byte alignment of each buffer in the arena, and the canary guard after each


def _arenas(plan, n):
    """Lay every plan buffer out in ``n`` flat byte arenas of one layout, each buffer 1 KiB aligned and followed by at
    least 1 KiB of guard bytes that belong to no buffer, the first arena holding the buffers' current values.  Returns
    (arenas, [(byte offset, byte size)] per buffer, per arena the byte view of every buffer, the buffers' dtypes)."""
    layout, pos = [], _ARENA_ALIGN
    for b in plan.bufs:
        nbytes = b.tensor.numel() * b.tensor.element_size()
        layout.append((pos, nbytes))
        pos = -(-(pos + nbytes + _ARENA_ALIGN) // _ARENA_ALIGN) * _ARENA_ALIGN
    arenas = [torch.zeros(pos + 64 * _ARENA_ALIGN, dtype=torch.uint8, device=plan.device) for _ in range(n)]
    views = [[a[off:off + nbytes] for off, nbytes in layout] for a in arenas]
    dts = [b.tensor.dtype for b in plan.bufs]
    for b, v in zip(plan.bufs, views[0]):
        v.view(b.tensor.dtype).copy_(b.tensor.reshape(-1))
    return arenas, layout, views, dts


def _point(plan, views, dts):
    """Point every plan buffer at its byte view in one arena (the ops resolve their pointers when they run)."""
    for b, v, dt in zip(plan.bufs, views, dts):
        b.tensor = v.view(dt)


def _locate(layout, plan, byte):
    """'buffer k element e' (or 'guard after buffer k') for a byte offset of an arena."""
    import bisect
    k = bisect.bisect_right([o for o, _ in layout], byte) - 1
    if k < 0:
        return "guard before buffer 0"
    off, nbytes = layout[k]
    if byte >= off + nbytes:
        return "guard after buffer %d" % k
    return "buffer %d element %d" % (k, (byte - off) // plan.bufs[k].tensor.element_size())


def footprint_walk(plan, static_in, check=None, canaries=FOOTPRINT_CANARIES):
    """Run the plan op by op on one stream, in program order, and check that every launch touches only what it
    declares (Plan.op_io, as op_footprints reads it).  With S_i the plan buffers just before op i and R = S_{i+1} its
    result, for each canary: op i runs on a copy of the buffers in which every element (and every guard byte between
    buffers) it does not declare as read holds the canary and every element it declares as read holds its value in
    S_i; every element it declares as written must then equal R bit for bit (else it read something undeclared, or
    left part of its declared output as it was), and every other byte must hold what it held (else it wrote outside
    its declaration).  Buffers address_buffers names always hold their values in S_i, never a canary; they are only
    checked for writes.  After the walk the constants and the staged inputs must be bit-unchanged.
    The buffers live in two arenas of one layout: the true state, which every op advances, and the canary copy, which
    holds the canary everywhere between ops, so each op costs its own buffers plus one word-wise comparison of the
    canary arena with the canary.  check: the op indices to check (default all; the others only run).
    Returns (ops checked, failures [(op index, name, message)], skipped [(op index, name, reason)])."""
    (true, canary, start), layout, (tv, cv, _), dts = _arenas(plan, 3)
    start.copy_(true)
    kno = {id(b): k for k, b in enumerate(plan.bufs)}
    addr = sorted(kno[a] for a in address_buffers(plan))
    sp = torch.cuda.current_stream().cuda_stream
    consts0 = [c.clone() for c in plan.consts]
    static0 = [s.clone() for s in static_in]
    words = canary.view(torch.int64)
    flag = torch.empty(words.shape, dtype=torch.bool, device=words.device)
    fps, failures, skipped, msgs = {}, [], [], {}
    for i, (name, _) in enumerate(plan.ops):
        if check is not None and i not in check:
            continue
        f = op_footprints(plan, i)
        if f is None:
            skipped.append((i, name, "no declared I/O"))
            continue
        over = [kno[id(b)] for fp in f for b in fp.bufs() if fp.extent(b) > b.tensor.numel()]
        if over:
            failures.append((i, name, "declared footprint runs past the end of buffer %s" % over))
            continue
        fps[i] = f
    for K in canaries:
        true.copy_(start)
        canary.fill_(K)
        kword = int.from_bytes(bytes([K]) * 8, "little", signed=True)
        for i, (name, fn) in enumerate(plan.ops):
            if i not in fps:
                _point(plan, tv, dts)
                fn(sp)
                continue
            rd, wr = fps[i]
            touched = sorted({kno[id(b)] for b in rd.bufs() + wr.bufs()} | set(addr))
            saved = []
            for k in touched:
                b, esz = plan.bufs[k], plan.bufs[k].tensor.element_size()
                rb = torch.zeros(layout[k][1], dtype=torch.bool, device=flag.device)
                wb = torch.zeros_like(rb)
                if k in addr:
                    rb.fill_(True)
                rd.mark(b, rb, 0, esz)
                wr.mark(b, wb, 0, esz)
                s_k = tv[k].clone()
                torch.where(rb, s_k, cv[k], out=cv[k])
                saved.append((k, rb, wb, s_k))
            _point(plan, cv, dts)
            fn(sp)
            _point(plan, tv, dts)
            fn(sp)
            n_r = n_w = 0
            first_r = first_w = None
            for k, rb, wb, s_k in saved:
                want = torch.where(wb, tv[k], s_k.masked_fill(~rb, K))
                bad = cv[k] != want
                if bool(bad.any()):
                    inw = bad & wb
                    out = bad & ~wb
                    if bool(inw.any()):
                        n_r += int(inw.sum())
                        first_r = first_r or _locate(layout, plan, layout[k][0] + int(torch.nonzero(inw)[0]))
                    if bool(out.any()):
                        n_w += int(out.sum())
                        first_w = first_w or _locate(layout, plan, layout[k][0] + int(torch.nonzero(out)[0]))
                cv[k].fill_(K)
            torch.ne(words, kword, out=flag)
            if bool(flag.any()):
                bad = torch.nonzero(canary != K).flatten()
                n_w += len(bad)
                first_w = first_w or _locate(layout, plan, int(bad[0]))
                canary.fill_(K)
            parts = []
            if n_r:
                parts.append("%d bytes of its declared output differ from the true run (reads undeclared input or "
                             "does not write all of it; first at %s)" % (n_r, first_r))
            if n_w:
                parts.append("%d bytes outside its declared output changed (first at %s)" % (n_w, first_w))
            if parts:
                msgs.setdefault(i, []).append("canary 0x%02X: %s" % (K, "; ".join(parts)))
    _point(plan, tv, dts)
    torch.cuda.synchronize()
    failures += [(i, plan.ops[i][0], " | ".join(m)) for i, m in sorted(msgs.items())]
    for k, (c, c0) in enumerate(zip(plan.consts, consts0)):
        if not torch.equal(_bits(c), _bits(c0)):
            failures.append((-1, "const %d" % k, "a plan constant changed during the walk"))
    for k, (s, s0) in enumerate(zip(static_in, static0)):
        if not torch.equal(_bits(s), _bits(s0)):
            failures.append((-1, "input %d" % k, "a staged input changed during the walk"))
    return len(fps), failures, skipped


def run_in_order(plan, order):
    """Zero every plan buffer and run the ops on one stream in ``order``; returns a copy of every buffer."""
    sp = torch.cuda.current_stream().cuda_stream
    for b in plan.bufs:
        b.tensor.zero_()
    for i in order:
        plan.ops[i][1](sp)
    torch.cuda.synchronize()
    return [b.tensor.clone() for b in plan.bufs]


# ---- reading plan tensors
def full_rows(t):
    """[N, T, H, W, row_stride] view of the whole rows a TRef lives in (W-padded stem inputs: their visible columns)."""
    b = t.buf.tensor
    if t.padw is not None:
        wp, wphys = t.padw
        return b[:t.N * t.T * t.H * wphys * t.Cp].view(t.N, t.T, t.H, wphys, t.Cp)[:, :, :, wp:wp + t.W]
    return b[:t.N * t.npos * t.row_stride].view(t.N, t.T, t.H, t.W, t.row_stride)


def ndhwc(t, clips):
    """The C valid channels of TRef t as [n, T, H, W, C] for the selected clips (a copy)."""
    return full_rows(t)[clips][..., t.ch_off:t.ch_off + t.C].clone()


def ncdhw64(t, clips):
    return ndhwc(t, clips).permute(0, 4, 1, 2, 3).double()


def rows64(t, clips):
    """[n, npos, C] float64 (token tensors and pooled rows)."""
    return ndhwc(t, clips).reshape(len(clips), t.npos, t.C).double()


def span64(spec, t, clips, role):
    """[n, rows, C] float64 of the token rows of TRef t the record's op reads or writes (record_rows)."""
    return record_rows(spec, t, role)[clips].reshape(len(clips), -1, t.C).double()


def buf_view(b, shape):
    n = math.prod(shape)
    return b.tensor[:n].view(*shape)


def token_span(spec, t, role):
    """The token rows of TRef t that the record's op reads (role "read") or writes ("write") when that is not all of
    them (a slice), else None: the class-token rows another op writes, or the one row an op takes from its input."""
    k, cls = spec["kind"], spec.get("cls") or 0
    x, y = spec.get("x"), spec.get("y")
    if role == "write" and t is y:
        if k in ("pool", "token_conv") and cls:
            return slice(cls, None)
        if k == "copy_cls":
            return slice(0, 1)
        if k == "copy_tokens":
            return slice(spec["row0"], spec["row0"] + x.npos)
    if role == "read" and x is not y:
        if k in ("pool", "token_conv") and cls and t is x:
            return slice(cls, None)
        if k == "layernorm_sets" and cls and (t is x or t is y):
            return slice(0, cls) if t is x else slice(cls, None)      # the class rows from x, the others in place
        if (k == "copy_cls" or (k == "layernorm" and spec["first_row_only"])) and t is x:
            return slice(0, 1)
    return None


def record_rows(spec, t, role=None):
    """The values an operand of a record holds, as a view [N, ...] whose first axis is the clip (the RoI for the
    tensors a RoIAlign head computes per box), without the pad channels and without the other producers' channels of
    a shared buffer.  t: a TRef, a MaskRef, a Buf the record reads or writes (its layout follows from the record's
    kind), the record's RoIs (their coordinates), or a plain tensor (a staged plan input, taken as it is).  role
    "read" / "write": only the token rows the op reads / writes (token_span), as [N, rows, C]."""
    from .engine.plan import MaskRef, TRef
    if torch.is_tensor(t):
        return t
    if isinstance(t, TRef):
        v = full_rows(t)[..., t.ch_off:t.ch_off + t.C]
        span = token_span(spec, t, role) if role is not None else None
        return v if span is None else v.reshape(t.N, t.npos, t.C)[:, span]
    if spec is not None and t is spec.get("rois"):
        return t.tensor[:, 1:]
    if isinstance(t, MaskRef) or all(hasattr(t, a) for a in ("B", "T", "tensor", "buf")):
        return (t.tensor if t.tensor is not None else t.buf.tensor[:t.B * t.T]).view(t.B, t.T)
    for v in spec.values():
        if isinstance(v, MaskRef) and v.buf is t:
            return record_rows(spec, v)
    k = spec["kind"]
    if k == "to_f32":
        x = spec["x"]
        return buf_view(t, (x.N, x.C, x.T, x.H, x.W) if spec["layout"] == "ncdhw" else (x.N, x.npos, x.C))
    if k == "head_reduce":
        return buf_view(t, (spec["x"].N, spec["x"].C))
    if t is spec.get("gate"):
        x = spec["x"]
        return buf_view(t, (x.N, x.Cp))[:, :x.C]
    if t is spec.get("sums") or t is spec.get("se_sums"):
        # an SE accumulator: int64 fixed-point (2^-24) sums per (sample, channel)
        x = spec["y"] if k == "conv" else spec["x"]
        return t.tensor[:2 * x.N * x.Cp].view(torch.int64).view(x.N, x.Cp)[:, :x.C]
    if t is spec.get("lse"):
        return buf_view(t, (spec["q"].N, spec["heads"] * spec["q"].npos))
    if k == "attention_weights" and t is spec["w"]:
        return buf_view(t, (spec["q"].N, spec["q"].npos, spec["k"].npos))
    raise AssertionError("%s: no per-clip layout for operand %r" % (k, t))


def _grid(rows, cls, thw):
    """[n, cls + THW, C] token rows -> the patch grid [n, C, T, H, W]."""
    n, _, C = rows.shape
    return rows[:, cls:].reshape(n, *thw, C).permute(0, 4, 1, 2, 3)


def _rows_of(grid):
    n, C = grid.shape[:2]
    return grid.permute(0, 2, 3, 4, 1).reshape(n, -1, C)


def _tdt(t):
    """torch dtype a TRef / Buf is stored in."""
    from .engine.plan import _TORCH_DT
    return _TORCH_DT[t.dt]


def _is32(t):
    return _tdt(t) == torch.float32


def _rnd(t):
    """Unit roundoff of the stored result."""
    return F32_EPS if _is32(t) else F16_EPS


def _wq(w, t):
    """The weights as the kernel writing TRef t read them: packed in t's storage dtype (engine/packing.py)."""
    return w.detach().to(_tdt(t)).double()


# ---- per kind: inputs (read before the op runs), output (after) and the comparison
def gather_inputs(spec, clips):
    k = spec["kind"]
    if k in ("to_ndhwc", "tokens_in"):
        return {"src": spec["src"][clips].clone()}
    if k == "conv":
        d = {"x": ncdhw64(spec["x"], clips)}
        d["res"] = ncdhw64(spec["residual"], clips) if spec["residual"] is not None else None
        if spec["addend"] is not None:
            a, off = spec["addend"]
            co = spec["weight"].shape[0]
            full = full_rows(a)[clips][..., a.ch_off + off:a.ch_off + off + co]
            d["addend"] = full.permute(0, 4, 1, 2, 3).double()
        return d
    if k == "tap_sum":
        return {"x": ndhwc(spec["x"], clips).double()}
    if k == "fused_block":
        return {"x": ncdhw64(spec["x"], clips)}
    if k in ("pool", "token_conv", "copy_cls", "pos_cls", "head_reduce", "layernorm", "to_f32", "copy",
             "channel_affine"):
        return {"x": span64(spec, spec["x"], clips, "read"), "x_raw": ndhwc(spec["x"], clips)}
    if k == "se_gate":
        x = spec["x"]
        return {"sums": record_rows(spec, spec["sums"])[clips].double() * 2.0 ** -24}
    if k == "scale_act":
        x = spec["x"]
        g = record_rows(spec, spec["gate"])[clips].double() if spec["gate"] is not None else None
        return {"x": rows64(x, clips), "gate": g}
    if k == "add_layernorm":
        return {"a": rows64(spec["a"], clips).float(), "br": rows64(spec["br"], clips).float()}
    if k == "layernorm_sets":
        return {"x": span64(spec, spec["x"], clips, "read"), "y": span64(spec, spec["y"], clips, "read")}
    if k == "attention":
        return {n: rows64(spec[n], clips) for n in ("q", "k", "v")}
    if k == "mask_force_first":
        return {"src": record_rows(spec, spec["mask"])[clips].clone()}
    if k in ("masked_pool", "masked_default", "copy_tokens"):
        return {"x": rows64(spec["x"], clips), "x_raw": ndhwc(spec["x"], clips),
                "mask": mask_bool(spec.get("mask"), clips)}
    if k == "reduce_fusion":
        return {"parts": [rows64(t, clips) for t in spec["parts"]],
                "parts_raw": [ndhwc(t, clips).reshape(len(clips), t.npos, t.C) for t in spec["parts"]]}
    if k in ("attention_masked", "attention_weights"):
        d = {n: rows64(spec[n], clips) for n in ("q", "k", "v") if n in spec}
        d["mask"] = mask_bool(spec["mask"], clips)
        return d
    if k == "lstm":
        return {"g": rows64(spec["g"], clips), "mask": mask_bool(spec["mask"], clips)}
    if k == "roi_align":
        # the boxes may sample any clip: the whole feature map, and every box
        x = spec["x"]
        return {"x": ndhwc(x, list(range(x.N)))[:, 0].double().cpu(), "rois": spec["rois"].tensor.float().cpu()}
    raise AssertionError("no reference for %s" % k)


def _heads(r, H):
    n, N, C = r.shape
    return r.view(n, N, H, C // H).permute(0, 2, 1, 3)


def compare(spec, inp, clips, launched, cpu_ref=False):
    """Run the comparison of one op; returns [(what, err / tol)] (0.0 for bit-exact checks).  cpu_ref: compute the
    float64 reference on the CPU instead (self-check of the GPU path) and return it instead of comparing."""
    from . import _lib as L
    from .engine import packing as PK
    k = spec["kind"]
    if cpu_ref is not False:
        inp = {n: (v.to(cpu_ref) if torch.is_tensor(v) else v) for n, v in inp.items()}
    n = len(clips)
    out = []
    live = cpu_ref is False

    def bound(got, ref, absref, K, acc_eps=ACC_EPS, extra=None, rnd=F16_EPS, what=k):
        if not live:
            out.append((what, ref))
            return
        r = assert_close_to_f64(got, ref, absref, K, acc_eps=acc_eps, what=what, extra64=extra, rnd_eps=rnd)
        out.append((what, r[0]))

    def exact(got, want, what=k):
        if not live:
            out.append((what, want.double()))
            return
        g, w = got.contiguous(), want.to(got.dtype).contiguous()
        bits = {torch.float16: torch.int16, torch.float32: torch.int32}[g.dtype]
        diff = g.view(bits) != w.view(bits)
        assert not bool(diff.any()), "%s: %d elements differ from the bit-exact reference" % (what, int(diff.sum()))
        out.append((what, 0.0))

    if k in ("to_ndhwc", "tokens_in"):
        y = spec["y"]
        src = inp["src"]
        if k == "to_ndhwc":
            want, got = src.permute(0, 2, 3, 4, 1), ndhwc(y, clips) if live else None
        else:
            want, got = src.reshape(n, -1, y.C), ndhwc(y, clips).reshape(n, -1, y.C) if live else None
        exact(got, want.to(_tdt(y)))
    elif k == "to_f32":
        x, o = spec["x"], spec["out"]
        if spec["layout"] == "ncdhw":
            want = inp["x_raw"].permute(0, 4, 1, 2, 3)
        else:
            want = inp["x_raw"].reshape(n, x.npos, x.C)
        exact(record_rows(spec, o)[clips] if live else None, want.float())
    elif k == "copy":
        exact(ndhwc(spec["y"], clips) if live else None, inp["x_raw"])
    elif k == "conv":
        y = spec["y"]
        w = _wq(spec["weight"], y)
        x = inp["x"]
        ref, absref = conv_ref64(x, w, spec["scale"], spec["bias"], spec["stride"], spec["padding"],
                                 spec["dilation"], spec["groups"], _ACT_NAMES[spec["act"]], inp["res"])
        extra = None
        if spec["addend"] is not None:
            # the tensor-core epilogue adds the addend to the stored-precision result: one more rounding of |act(.)|
            extra = _rnd(y) * ref.abs()
            ref, absref = ref + inp["addend"], absref + inp["addend"].abs()
        K = w.shape[1] * math.prod(w.shape[2:])
        got = ncdhw64(y, clips) if live else None
        bound(got, ref, absref, K, extra=extra, rnd=_rnd(y))
        if spec["se_sums"] is not None:
            ntaps = math.prod(w.shape[2:])
            ref_s, npos = ref.sum(dim=(2, 3, 4)), ref[0, 0].numel()
            if not live:
                out.append(("se_sums", ref_s))
            else:
                # the SE-sum bound of test_depthwise_instance (fp32 sums of the pre-rounding outputs, fixed point)
                sums = (record_rows(spec, spec["se_sums"])[clips].double() * 2.0 ** -24).cpu()
                ref_s, absref_s = ref_s.cpu(), absref.sum(dim=(2, 3, 4)).cpu()
                tol = 2.0 ** -20 * (1 + ntaps / 64.0) * absref_s + npos * 2.0 ** -23 + 2.0 ** -22 * ref_s.abs()
                if any(i.startswith(("dwconv3d_kernel<", "dwconv3d_w4_kernel<")) for i in launched):
                    # the generic path sums the stored outputs (pv_channel_sum after the stencil): their rounding, and
                    # the fp32 partial sums of its threads over up to channel_sum_adds positions each
                    per_elem = _rnd(y) + (channel_sum_adds(npos, y.Cp) + 1) * F32_EPS
                    tol = tol + per_elem * ref.abs().sum(dim=(2, 3, 4)).cpu()
                r = float(((sums - ref_s).abs() / tol).max())
                assert r <= 1.0, "se_sums: err/tol %.3g" % r
                out.append(("se_sums", r))
    elif k == "tap_sum":
        x, y = inp["x"], spec["y"]
        co, kt, st, pt, dil = y.C, spec["kt"], spec["st"], spec["pt"], spec["dil"]
        cop = PK.pad8(co)
        Ti, To = x.shape[1], y.T
        acc = torch.zeros(n, To, y.H, y.W, co, dtype=torch.float64, device=x.device)
        aab = torch.zeros_like(acc)
        for t in range(To):
            for d in range(kt):
                ti = t * st + d * dil - pt
                if 0 <= ti < Ti:
                    tap = x[:, ti, :, :, d * cop:d * cop + co]
                    acc[:, t] += tap
                    aab[:, t] += tap.abs()
        sc, bi = spec["scale"].double().to(x.device), spec["bias"].double().to(x.device)
        pre = acc * sc + bi
        act = _ACT_NAMES[spec["act"]]
        absref = LIP[act] * (aab * sc.abs() + bi.abs())
        got = ndhwc(y, clips) if live else None
        bound(got, act64(pre, act), absref, kt + 2, acc_eps=SUM_EPS, extra=act_err64(pre, act), rnd=_rnd(y))
    elif k == "fused_block":
        y = spec["y"]
        wa, wb, wc = (_wq(spec[m], y) for m in ("wa", "wb", "wc"))
        ws = _wq(spec["ws"], y) if spec["ws"] is not None else None
        yr, _, _, Y, prop = fused_block_ref64(inp["x"], wa, wb, wc, ws, spec["folds"], spec["kt"], spec["sb"],
                                              _ACT_NAMES[spec["act"]])
        K = wa.shape[0] + (wa.shape[1] if ws is not None else 0)
        got = ncdhw64(y, clips) if live else None
        bound(got, yr, Y, K, extra=prop, rnd=_rnd(y))
    elif k == "pool":
        x, y, cls = spec["x"], spec["y"], spec["cls"]
        thw = spec.get("thw", (x.T, x.H, x.W))
        g = _grid(inp["x"], 0, thw)
        kk, s, p = spec["kernel"], spec["stride"], spec["padding"]
        pad = (p[2], p[2], p[1], p[1], p[0], p[0])
        got = span64(spec, y, clips, "write") if live else None
        if spec["mode"] == L.POOL_MAX:
            ref = F.max_pool3d(F.pad(g, pad, value=-math.inf), kk, s)
            exact(got.to(_tdt(y)) if live else None, _rows_of(ref).to(_tdt(y)))
        else:
            ref = F.avg_pool3d(F.pad(g, pad), kk, s)
            absref = F.avg_pool3d(F.pad(g.abs(), pad), kk, s)
            glob = "global_pool_kernel" in launched
            K = (math.ceil(math.prod(thw) / 32) + 32) if glob else math.prod(kk)
            bound(got, _rows_of(ref), _rows_of(absref), K, acc_eps=SUM_EPS, rnd=_rnd(y))
    elif k == "token_conv":
        x, y, cls = spec["x"], spec["y"], spec["cls"]
        g = _grid(inp["x"], 0, spec["thw"])
        w = _wq(spec["weight"], y)
        C = w.shape[0]
        ones = torch.ones(C, dtype=torch.float64)
        got = span64(spec, y, clips, "write") if live else None
        if not spec["prologue"]:
            ref, absref = conv_ref64(g, w, ones, torch.zeros_like(ones), spec["stride"], spec["padding"],
                                     spec["dilation"], C, "none", None)
            bound(got, _rows_of(ref), _rows_of(absref), math.prod(w.shape[2:]), rnd=_rnd(y))
        else:
            ref, absref, u, pre = prologue_conv_ref64(g, spec["pre_scale"], spec["pre_bias"], w, ones,
                                                      torch.zeros_like(ones), spec["stride"], spec["padding"],
                                                      spec["dilation"])
            # the prologue's own error carried by the stencil: GELU in fp32 (act_err64) at an argument rounded once,
            # and the f16 rounding of u where the TMA kernels stage it in shared memory
            eu = act_err64(pre, "gelu") + LIP["gelu"] * F32_EPS * pre.abs() + _rnd(y) * u.abs()
            extra = F.conv3d(eu, w.abs().to(eu.device), None, spec["stride"], spec["padding"], spec["dilation"], C)
            bound(got, _rows_of(ref), _rows_of(absref), math.prod(w.shape[2:]), extra=_rows_of(extra), rnd=_rnd(y))
    elif k == "channel_affine":
        y = spec["y"]
        v = inp["x"]
        sc, sh = (spec[m].double().to(v.device) for m in ("scale", "shift"))
        got = rows64(y, clips) if live else None
        bound(got, v * sc + sh, v.abs() * sc.abs() + sh.abs(), 1, rnd=_rnd(y))
    elif k == "copy_cls":
        exact(record_rows(spec, spec["y"], "write")[clips] if live else None, inp["x"])
    elif k == "pos_cls":
        y = spec["y"]
        xr = inp["x_raw"].reshape(n, -1, spec["x"].C).float()
        pos = spec["pos"].to(xr.device)
        hc = 1 if spec["has_cls"] else 0
        want = torch.empty(n, hc + xr.shape[1], xr.shape[2], dtype=torch.float32, device=xr.device)
        if hc:
            want[:, 0] = pos[0]
        want[:, hc:] = xr + pos[hc:]
        got = ndhwc(y, clips).reshape(n, y.npos, y.C) if live else None
        exact(got, want.to(_tdt(y)))
    elif k == "head_reduce":
        x64 = inp["x"]
        C = x64.shape[2]
        got = record_rows(spec, spec["out"])[clips] if live else None
        if not spec["softmax"]:
            bound(got, x64.mean(1), x64.abs().mean(1), x64.shape[1] + 1, acc_eps=SUM_EPS, rnd=F32_EPS)
        else:
            p = torch.softmax(x64, 2)
            d = x64 - x64.max(2, keepdim=True).values
            rel = 2.0 ** -22 + F32_EPS * d.abs()
            extra = (p * (rel + rel.max(2, keepdim=True).values)).mean(1)
            D = -(-C // 256) + 13
            bound(got, p.mean(1), p.mean(1), x64.shape[1] + D + 3, acc_eps=SUM_EPS, extra=extra, rnd=F32_EPS)
    elif k == "se_gate":
        x = spec["x"]
        dev = inp["sums"].device
        mean = inp["sums"] / x.npos
        w1, b1, w2, b2 = (spec[m].double().to(dev) for m in ("w1", "b1", "w2", "b2"))
        hid = (b1 + mean @ w1.t()).clamp_min(0)
        a = b2 + hid @ w2.t()
        gate = torch.sigmoid(a)
        Hm = b1.abs() + mean.abs() @ w1.abs().t()
        A = b2.abs() + Hm @ w2.abs().t()
        extra = gate * (1 - gate) * (2 + 1.173 * a.abs()) * 2.0 ** -23 + F32_EPS * gate
        got = record_rows(spec, spec["gate"])[clips] if live else None
        bound(got, gate, 0.25 * A, x.C + w1.shape[0] + 3, acc_eps=SUM_EPS, extra=extra, rnd=F32_EPS)
    elif k == "scale_act":
        y = spec["y"]
        v = inp["x"]
        if inp["gate"] is not None:
            v = v * inp["gate"].unsqueeze(1)
        act = _ACT_NAMES[spec["act"]]
        got = rows64(y, clips) if live else None
        bound(got, act64(v, act), LIP[act] * v.abs(), 0, acc_eps=F32_EPS, extra=act_err64(v, act), rnd=_rnd(y))
    elif k == "layernorm":
        v = inp["x"]
        C = v.shape[2]
        name = next(iter(launched))
        _, lpr, nch = ln_dispatch(C) if name in ("layernorm_reg_kernel", "add_layernorm_kernel") else \
            ("layernorm_kernel", 32, -(-(-(-C // 8)) // 32))
        ref, absref, K, extra = ln_ref64(v.reshape(-1, 1, C), spec["gamma"].view(1, -1), spec["beta"].view(1, -1), 1,
                                         nch * 8 + int(math.log2(lpr)), spec["eps"])
        got = rows64(spec["y"], clips).reshape(-1, 1, C) if live else None
        bound(got, ref, absref, K, acc_eps=SUM_EPS, extra=extra, rnd=_rnd(spec["y"]))
    elif k == "add_layernorm":
        s = inp["a"] + inp["br"]                               # fp32, as the kernel adds
        if spec["s"] is not None:
            exact(ndhwc(spec["s"], clips).reshape(s.shape) if live else None, s, what="add_layernorm.sum")
        if spec["y"] is not None:
            C = s.shape[2]
            _, lpr, nch = ln_dispatch(C)
            ref, absref, K, extra = ln_ref64(s.reshape(-1, 1, C), spec["gamma"].view(1, -1),
                                             spec["beta"].view(1, -1), 1, nch * 8 + int(math.log2(lpr)), spec["eps"])
            got = rows64(spec["y"], clips).reshape(-1, 1, C) if live else None
            bound(got, ref, absref, K, acc_eps=SUM_EPS, extra=extra, rnd=_rnd(spec["y"]))
    elif k == "layernorm_sets":
        y, cls, hd = spec["y"], spec["cls"], spec["head_dim"]
        v = torch.cat([inp["x"], inp["y"]], 1) if cls and spec["x"] is not y else inp["y"]
        C = v.shape[2]
        G = C // hd
        nsets = spec["gamma"].numel() // hd
        name = next(iter(launched))
        _, lpr, nch = ln_dispatch(hd) if name == "layernorm_reg_kernel" else \
            ("layernorm_kernel", 32, -(-(-(-hd // 8)) // 32))
        ref, absref, K, extra = ln_ref64(v.reshape(-1, G, hd), spec["gamma"].view(nsets, hd),
                                         spec["beta"].view(nsets, hd), G // nsets, nch * 8 + int(math.log2(lpr)),
                                         spec["eps"])
        got = rows64(y, clips).reshape(-1, G, hd) if live else None
        bound(got, ref, absref, K, acc_eps=SUM_EPS, extra=extra, rnd=_rnd(y))
    elif k == "attention":
        H, o, norm = spec["heads"], spec["o"], spec["normalize"]
        q, kk, v = (_heads(inp[m], H) for m in ("q", "k", "v"))
        ref, absref = attn_ref64(q, kk, v, spec["scale"], spec["residual"], norm)
        back = lambda t: t.permute(0, 2, 1, 3).reshape(n, t.shape[2], -1)        # noqa: E731
        got = rows64(o, clips) if live else None
        if norm:
            # the linear mode: D-term dot products and an Nk-term sum, each rounding charged (f16: P rounded as well)
            if _is32(o):
                bound(got, back(ref), back(absref), kk.shape[2] + q.shape[3], acc_eps=ACC_EPS_ATTN_F32, rnd=F32_EPS)
            else:
                bound(got, back(ref), back(absref), 0, acc_eps=ACC_EPS_ATTN)
        elif not _is32(o):
            extra = back(attn_score_extra64(q, kk, v, spec["scale"]) + attn_p16_floor64(v, q.shape[2]))
            bound(got, back(ref), back(absref), 0, acc_eps=ACC_EPS_ATTN, extra=extra)
        else:
            extra = back(attn_score_extra64(q, kk, v, spec["scale"]))
            bound(got, back(ref), back(absref), kk.shape[2], acc_eps=ACC_EPS_ATTN_F32, extra=extra, rnd=F32_EPS)
    elif k == "mask_force_first":
        want = inp["src"].clone()
        want[:, 0] = 1
        if not live:
            out.append((k, want.double()))
        else:
            got = record_rows(spec, spec["out"])[clips]
            assert torch.equal(got, want.to(got.device)), "mask_force_first: the mask copy differs"
            out.append((k, 0.0))
    elif k == "masked_pool":
        x, y = inp["x"], spec["y"]
        m = inp["mask"] if inp["mask"] is not None else torch.ones(x.shape[:2], dtype=torch.bool, device=x.device)
        m = m.to(x.device)
        cnt = m.sum(1, keepdim=True)
        got = ndhwc(y, clips).reshape(n, y.C) if live else None
        if spec["mode"] == L.MPOOL_MAX:
            # the largest valid step; a row without one pools to 0
            ref = x.masked_fill(~m[..., None], -math.inf).max(1).values
            exact(got, torch.where(cnt > 0, ref, torch.zeros_like(ref)))
        else:
            # fp32 sum over the valid steps in order, then (avg) one division by the valid count (1 when none)
            mf = m[..., None].double()
            ref, absref = (x * mf).sum(1), (x.abs() * mf).sum(1)
            if spec["mode"] == L.MPOOL_AVG:
                ref, absref = ref / cnt.clamp_min(1), absref / cnt.clamp_min(1)
            bound(got.double() if live else None, ref, absref, x.shape[1] + 2, acc_eps=SUM_EPS, rnd=_rnd(y))
    elif k == "masked_default":
        # x * a + default * (1 - a) in fp32, a = 1 where the row has a valid step: x or the default, exactly
        y = spec["y"]
        xr = inp["x_raw"].reshape(n, y.C).float()
        a = (inp["mask"].any(1, keepdim=True) if inp["mask"] is not None else
             torch.ones(n, 1, dtype=torch.bool)).float().to(xr.device)
        want = xr * a + spec["default"].to(xr.device).view(1, -1) * (1 - a)
        exact(ndhwc(y, clips).reshape(n, y.C) if live else None, want.to(_tdt(y)))
    elif k == "copy_tokens":
        x, y = spec["x"], spec["y"]
        exact(record_rows(spec, y, "write")[clips] if live else None, inp["x_raw"].reshape(n, x.npos, x.C))
    elif k == "reduce_fusion":
        y, parts = spec["y"], inp["parts"]
        got = ndhwc(y, clips).reshape(n, y.npos, y.C) if live else None
        if spec["op"] == L.REDUCE_MAX:
            ref = parts[0]
            for t in parts[1:]:
                ref = torch.maximum(ref, t)
            exact(got, ref.to(_tdt(y)))
        else:
            ref, absref = parts[0], parts[0].abs()
            for t in parts[1:]:
                ref, absref = (ref + t, absref + t.abs()) if spec["op"] == L.REDUCE_SUM else (ref * t, absref * t.abs())
            bound(got.double() if live else None, ref, absref, len(parts), acc_eps=SUM_EPS, rnd=_rnd(y))
    elif k == "attention_masked":
        H, o = spec["heads"], spec["o"]
        q, kk, v = (_heads(inp[m], H) for m in ("q", "k", "v"))
        ref, absref = attn_ref64(q, kk, v, spec["scale"], False, mask=inp["mask"])
        back = lambda t: t.permute(0, 2, 1, 3).reshape(n, t.shape[2], -1)        # noqa: E731
        got = rows64(o, clips) if live else None
        if not _is32(o):
            extra = back(attn_score_extra64(q, kk, v, spec["scale"], inp["mask"]) +
                         attn_p16_floor64(v, q.shape[2], inp["mask"]))
            bound(got, back(ref), back(absref), 0, acc_eps=ACC_EPS_ATTN, extra=extra)
        else:
            extra = back(attn_score_extra64(q, kk, v, spec["scale"], inp["mask"]))
            bound(got, back(ref), back(absref), kk.shape[2], acc_eps=ACC_EPS_ATTN_F32, extra=extra, rnd=F32_EPS)
    elif k == "attention_weights":
        H, wb = spec["heads"], spec["w"]
        q, kk = (_heads(inp[m], H) for m in ("q", "k"))
        Nq, Nk = q.shape[2], kk.shape[2]
        ref, err = attn_weights_err64(q, kk, spec["scale"], inp["mask"])
        got = record_rows(spec, wb)[clips] if live else None
        bound(got, ref, err, 0, acc_eps=1.0, rnd=F32_EPS)
    elif k == "lstm":
        y, Hd, nd = spec["y"], spec["hidden"], spec["dirs"]
        g = inp["g"]
        T = g.shape[1]
        m = inp["mask"]
        lengths = (m.sum(1) if m is not None else torch.full((n,), T)).clamp(1, T)
        cluster = "lstm_cluster_kernel" in launched
        W = spec["w_hh_t"].half() if cluster else spec["w_hh_t"]
        ref, err = lstm_ref64(g, W, lengths, Hd, nd, h16=cluster)
        got = ndhwc(y, clips).reshape(n, -1) if live else None
        # the propagated fp32 error is the whole accumulation term (acc_eps = 1, k_len = 0)
        bound(got, ref, err, 0, acc_eps=1.0, rnd=_rnd(y))
    elif k == "roi_align":
        x, y = spec["x"], spec["y"]
        rois = [tuple(float(v) for v in r) for r in inp["rois"]]
        ref, absref = roi_ref64(inp["x"].cpu(), rois, spec["geom"])
        got = ndhwc(y, list(range(y.N)))[:, 0] if live else None
        bound(got, ref, absref, 0, acc_eps=roi_acc_eps(rois, spec["geom"], x.H, x.W), rnd=_rnd(y))
    else:
        raise AssertionError("no reference for %s" % k)
    return out


def _outputs(spec):
    from .engine.plan import TRef
    return [t for t in record_io(spec)[1] if isinstance(t, TRef)]


def check_layout(spec, before):
    """Pad channels of every TRef output are zero; channels of its rows outside [ch_off, ch_off + Cp) are as they were
    before the op (other producers' slices of a concat buffer)."""
    for i, t in enumerate(_outputs(spec)):
        rows = full_rows(t)
        pad = rows[..., t.ch_off + t.C:t.ch_off + t.Cp]
        assert not bool(pad.any()), "pad channels [%d, %d) not zero" % (t.C, t.Cp)
        if before[i] is not None:
            was = before[i]
            keep = torch.ones(t.row_stride, dtype=torch.bool, device=rows.device)
            keep[t.ch_off:t.ch_off + t.Cp] = False
            same = torch.equal(rows[..., keep], was[..., keep])
            assert same, "channels outside this op's slice of the shared buffer changed"


def channel_sum_adds(npos, C):
    """The most positions one thread of pv_channel_sum adds in fp32 before its fixed-point atomic (chunks of at most
    2048 positions, at most 1024 chunks; 256 threads share a chunk, 8 channels each)."""
    chunks = min(-(-npos // 2048), 1024)
    chunk = -(-npos // chunks)
    per_iter = 256 // (-(-C // 8))
    return chunk if per_iter == 0 else -(-chunk // per_iter)


def audit_clips(B):
    """The clips the audit compares: the first, the middle and the last (the first tiles, the middle and the last,
    ragged tiles of every launch's walk)."""
    return sorted({0, B // 2, B - 1})


def audit_plan(plan, clips, corrupt=None, cpu_check=None):
    """Walk the plan on one stream, comparing every op with its float64 reference.  Returns (failures, stats):
    failures [(op index, name, message)], stats {family: (launches, largest err / tol, instances)}.
    corrupt(i, spec): called after op i ran, before its comparison.  cpu_check: a dict filled with
    {kind: largest relative difference between the float64 references computed on the GPU and on the CPU} for the
    first op of each kind."""
    from . import _lib as L
    f32 = plan.dt == L.PV_F32
    stream = torch.cuda.current_stream()
    sp = stream.cuda_stream
    failures, stats = [], {}
    for i, ((name, fn), spec) in enumerate(zip(plan.ops, plan.op_spec)):
        if spec is None:
            assert name.endswith(NO_VALUE_SUFFIXES), name
            fn(sp)
            continue
        try:
            inp = gather_inputs(spec, clips)
            before = [full_rows(t).clone() if (t.row_stride > t.Cp and t.padw is None) else None
                      for t in _outputs(spec)]
        except Exception as e:                          # noqa: BLE001 - reported with the op's name
            failures.append((i, name, "reading inputs: %r" % e))
            fn(sp)
            continue
        c0 = kernel_counts()
        fn(sp)
        torch.cuda.synchronize()
        launched = kernel_count_diff(c0, kernel_counts())
        fam = family_of(spec, f32)
        key = spec["route"] if spec["kind"] == "conv" else spec["kind"]
        if corrupt is not None:
            corrupt(i, spec)
        try:
            assert launched and all(n.startswith(fam) for n in launched), \
                "launched %s, outside the %s family" % (launched, key)
            res = compare(spec, inp, clips, launched)
            check_layout(spec, before)
        except AssertionError as e:
            failures.append((i, name, str(e)[:400]))
            continue
        if cpu_check is not None and spec["kind"] not in cpu_check:
            gpu = compare(spec, inp, clips, launched, cpu_ref=torch.device("cuda"))
            cpu = compare(spec, inp, clips, launched, cpu_ref=torch.device("cpu"))
            rel = 0.0
            for (_, g), (_, c) in zip(gpu, cpu):
                g, c = g.double().cpu(), c.double().cpu()
                rel = max(rel, float((g - c).abs().max()) / max(float(c.abs().max()), 1e-300))
            cpu_check[spec["kind"]] = rel
        n_, worst, inst = stats.get(key, (0, 0.0, set()))
        stats[key] = (n_ + 1, max([worst] + [r for _, r in res]), inst | set(launched))
    return failures, stats


def _bits(t):
    """Bit patterns: SE-sum buffers hold int64 fixed-point sums in f32 storage, some of which read as NaN."""
    return t.view({torch.float16: torch.int16, torch.float32: torch.int32}.get(t.dtype, t.dtype))


def check_graph_replay(cm, ins, alt):
    """Capture the compiled model's plan as it runs in service (lanes on side streams, one CUDA graph) and replay it
    on ``ins``, on ``alt`` and on ``ins`` again: after the first and the last replay every plan buffer must equal the
    single-stream run that left the buffers as they are now, bit for bit (a lane reading a buffer before its
    producer finished would see the other input's values).  Returns (lanes, buffers)."""
    plan = cm.plan
    single = [b.tensor.clone() for b in plan.bufs]
    for b in plan.bufs:
        b.tensor.zero_()
    cm._capture()
    for k, inputs in enumerate((ins, alt, ins)):
        for s, t in zip(cm.static_in, inputs):
            s.copy_(t)
        cm.graph.replay()
        torch.cuda.synchronize()
        if k == 1:
            continue
        bad = [i for i, (b, s) in enumerate(zip(plan.bufs, single)) if not torch.equal(_bits(b.tensor), _bits(s))]
        assert not bad, "replay %d: %d of %d buffers differ from the single-stream run (first: buffer %d)" % (
            k, len(bad), len(single), bad[0])
    return len(plan.sched["lanes"]), len(single)


# ---- the audit catalogue at any batch, and bitwise invariance across clip positions and batch sizes ----------------
# (tests/test_gpu_model_audit.py, tests/test_gpu_batch_audit.py)
def audit_catalogue(workloads):
    """[(family, case, is a workload shape)] in a fixed order: every case the suite compiles.  workloads: bench.py's
    WORKLOADS (the architecture / shape pairs the workload audit runs in f16)."""
    shapes = {(v[0], v[2], v[3], v[4]) for v in workloads.values()}
    cases = []
    for name, (hub, kw, B, T, H, W, _) in sorted(MODEL_CASES.items()):
        if name[:3] in ("c1_", "c2_", "c3_", "c4_") or name.endswith("_f16w"):
            continue
        cases.append(("model", name, not kw and (hub, T, H, W) in shapes))
    cases += [("hub_tail", c, False) for c in sorted(HUB_TAIL_CASES)]
    cases += [("grouped", c, False) for c in sorted(GROUPED_MODEL_CASES) if not c.endswith("_f16w")]
    cases += [("detection", c, False) for c in sorted(DETECTION_CASES)]
    cases += [("audio", c, False) for c in sorted(AUDIO_CASES)]
    cases += [("efficient", c, False) for c in sorted(EFFICIENT_CASES)]
    cases += [("mvit_variant", c, False) for c in sorted(MVIT_VARIANT_CASES)]
    cases += [("nonlocal", c, False) for c in sorted(NONLOCAL_CASES)]
    cases += [("nonlocal", "i3d_nln", False)]
    cases += [("masked", c, False) for c in MASKED_CASES]
    return cases


def audit_cases(workloads):
    """[(precision, family, case)] the model audit runs: f16 less the workload shapes, f32 all of them."""
    cat = audit_catalogue(workloads)
    return [("f16", f, c) for f, c, w in cat if not w] + [("f32", f, c) for f, c, _ in cat]


def batch_sweep(workloads):
    """[(precision, family, case, batch, checks)] of the batch audit; checks "abc" = float64 on every clip, position
    invariance and batch-size invariance, "bc" = the two bitwise checks (the workload audit runs float64 there)."""
    rows = []
    for arch in sorted(workloads):
        for B in ((1, 3) if arch == "x3d_xs" else (2, 3)):
            rows.append(("f16", "model", arch, B, "abc"))
        rows.append(("f16", "model", arch, workloads[arch][1], "bc"))
    rows += [("f16", f, c, 3, "abc") for p, f, c in audit_cases(workloads) if p == "f16"]
    rows += [("f32", "model", c, 3, "abc") for c in ("x3d_xs", "mvit_base_8x112")]
    rows += [("f32", "masked", c, 3, "abc") for c in MASKED_CASES]
    rows += [("f32", "detection", c, 3, "abc") for c in sorted(DETECTION_CASES)]
    rows += [(p, "ssl", c, B, "abc") for p in ("f16", "f32") for c in SSL_TRUNK_CASES for B in (1, 2, 3)]
    return rows


def multi_lane_case(family, case):
    """True for the catalogue cases whose plans run on more than one lane: SlowFast (two pathways), Audiovisual
    SlowFast (three) and the masked multipath models (one per stream)."""
    if family == "model":
        return bool(MODEL_CASES[case][6])
    if family in ("hub_tail", "grouped", "detection"):
        return case.startswith("slowfast")
    return (family == "audio" and case.startswith("avsf")) or (family == "masked" and case.startswith("multipath"))


FOOTPRINT_PARTS = ("f16", "f32")


def footprint_cases(workloads, sweep=False):
    """[(precision, family, case, batch or None = the case's own)] of the footprint checks: every audit_catalogue case
    in f16 and in f32, and the multi-lane cases at batch 3 in both (tiles and the Fast-stem route change there).
    sweep: the multi-lane cases also at every batch of batch_sweep."""
    cat = audit_catalogue(workloads)
    rows = [(p, f, c, None) for p in ("f16", "f32") for f, c, _ in cat]
    multi = [(f, c) for f, c, _ in cat if multi_lane_case(f, c)]
    extra = {(p, f, c, 3) for p in ("f16", "f32") for f, c in multi}
    if sweep:
        extra |= {(p, f, c, B) for p, f, c, B, _ in batch_sweep(workloads) if (f, c) in multi}
    return rows + sorted(extra)


def footprint_part(row):
    """The file of the GPU footprint walk a footprint_cases row runs in: one per precision."""
    return row[0]


def build_audit_case(family, case):
    """(model, engine inputs (a tensor or a list), extra, indices of inputs that stay fixed on the replay) of a case of
    the audit catalogue."""
    import pytorchvideo_b200.models as M
    import pytorchvideo_b200.models.hub as PH
    extra, fixed = (), set()
    if family == "model":
        m, x, _ = build_case(case, PH)
    elif family == "hub_tail":
        m, x = build_hub_tail_case(case, PH)
    elif family == "grouped":
        m, x, _ = build_grouped_case(case, PH)
    elif family == "detection":
        m, x, boxes, _ = build_detection_case(case, PH)
        x = (x if isinstance(x, list) else [x]) + [boxes]
        fixed = {len(x) - 1}
    elif family == "audio":
        m, x = build_audio_case(case, M)
    elif family == "efficient":
        m, x = build_efficient_case(case, efficient_namespace())
    elif family == "mvit_variant":
        from pytorchvideo_b200.layers.attention import MultiScaleBlock
        from pytorchvideo_b200.models.vision_transformers import create_multiscale_vision_transformers
        m, x, ex = build_mvit_variant_case(case, create_multiscale_vision_transformers, MultiScaleBlock)
        extra = tuple(tuple(e) for e in ex)
    elif family == "nonlocal":
        from pytorchvideo_b200.layers.nonlocal_net import create_nonlocal
        if case == "i3d_nln":
            m, x = build_i3d_nln(PH, create_nonlocal)
        else:
            m, x = build_nonlocal_case(case, create_nonlocal)
    elif family == "ssl":
        m, x = build_ssl_trunk(case)
    else:
        m = build_masked_case(case, masked_namespace())
        x, mask = masked_case_inputs(case)
        x, extra = masked_engine_args(case, x, mask)
        fixed = {i for i, t in enumerate(x if isinstance(x, list) else [x]) if t.dtype == torch.bool}
    return m, x, extra, fixed


SSL_TRUNK_CASES = ("embedding_chain", "moco_key")


def build_ssl_trunk(case):
    """(module, clip) of a self-supervised trunk as the models lower it: "embedding_chain" is the video SimCLR case's
    Slow-R50 trunk and its 2048-2048-128 BatchNorm1d projector as one EmbeddingChain (one plan with fused rows);
    "moco_key" is the chain MoCo v2's slow_r50 case compiles for its momentum (key) encoder."""
    import types
    from .layers import make_multilayer_perceptron
    from .models import moco_v2
    from .models.embedding import EmbeddingChain
    from .models.resnet import create_resnet
    from .models.simclr import SimCLR
    if case == "embedding_chain":
        ns = types.SimpleNamespace(SimCLR=SimCLR, create_resnet=create_resnet,
                                   make_multilayer_perceptron=make_multilayer_perceptron)
        m, (x1, _) = build_ssl_case("simclr_video", ns)
        return EmbeddingChain(m.backbone, m.mlp).eval(), x1[:1].contiguous()
    ns = types.SimpleNamespace(MOCO=moco_v2.MOCO, create_moco_resnet_50=moco_v2.create_moco_resnet_50,
                               create_mlp_util=moco_v2.create_mlp_util, create_resnet=create_resnet)
    m, views, _, _ = build_moco_case("moco_slow_r50", ns)
    return m._state()["mmt"].eval(), views[0][:1].contiguous()


def _roll_clip(t, k):
    """Clip k of a pool made from the clips of ``t``: clip k % B0 itself for k < B0, else that clip rolled along its
    last axis by k // B0 places (the same values, on the same grid, at other positions)."""
    c = t[k % t.shape[0]]
    return c if k < t.shape[0] else c.roll(k // t.shape[0], -1)


def _pool_boxes(H, W, pool):
    """[K, 5] boxes over ``pool`` clips, grouped by clip in clip order: clip 0 takes the three boundary boxes of
    synthetic_boxes (outside the frame, smaller than a feature cell, the whole frame), clip 1 none, every further clip
    two of the case's random boxes."""
    rows = [torch.cat([torch.zeros(1), b[1:]]) for b in synthetic_boxes(3, 1, H, W)]
    rnd = synthetic_boxes(max(5, 2 * pool), 1, H, W, seed=19)[3:]
    for c in range(2, pool):
        for b in rnd[2 * (c - 2):2 * (c - 1)]:
            rows.append(torch.cat([torch.tensor([float(c)]), b[1:]]))
    return torch.stack(rows).contiguous()


class BatchCase:
    """A catalogue case at any batch B <= pool: its model, and inputs whose clip j is the same tensor at every B (a
    pool of ``pool`` clips is drawn once; a batch is its first B clips).  Per-clip side inputs follow their clip:
    masks are rows of the pool, detection boxes carry their clip's batch index (clip 1 has none)."""

    def __init__(self, family, case, pool):
        self.family, self.case, self.pool = family, case, pool
        self.model, x, self.extra, fixed = build_audit_case(family, case)
        self.multi = isinstance(x, (list, tuple))
        xs = list(x) if self.multi else [x]
        self.box_slot = len(xs) - 1 if family == "detection" else None
        self.inputs = []
        for i, t in enumerate(xs):
            if i == self.box_slot:
                H, W = xs[0].shape[-2:]
                self.inputs.append(_pool_boxes(H, W, pool))
            else:
                self.inputs.append(torch.stack([_roll_clip(t, k) for k in range(pool)]))

    def boxes_of(self, B):
        """Per clip of a batch of B: the rows of its boxes (None without boxes)."""
        if self.box_slot is None:
            return None
        idx = self.inputs[self.box_slot][:, 0].long()
        keep = [int(i) for i in torch.nonzero(idx < B).flatten()]
        return [[r for r, i in enumerate(keep) if int(idx[i]) == c] for c in range(B)]

    def batch(self, B, rotate=False):
        """The engine inputs of the first B clips; rotate: clip c at position (c + 1) % B, boxes re-indexed."""
        out = []
        for i, t in enumerate(self.inputs):
            if i == self.box_slot:
                t = t[t[:, 0] < B].clone()
                if rotate:
                    t[:, 0] = (t[:, 0] + 1) % B
            else:
                t = t[:B].roll(1, 0) if rotate else t[:B]
            out.append(t.contiguous())
        return out

    def single(self, c):
        """The engine inputs of clip c alone (a clip without boxes gets two whole-frame boxes, whose rows nothing
        compares, so that its plan has the same ops)."""
        out = []
        for i, t in enumerate(self.inputs):
            if i == self.box_slot:
                t = t[t[:, 0] == c].clone()
                t[:, 0] = 0
                if not len(t):
                    H, W = self.inputs[0].shape[-2:]
                    t = torch.tensor([[0.0, 0.0, 0.0, float(W), float(H)]] * 2)
            else:
                t = t[c:c + 1]
            out.append(t.contiguous())
        return out

    def example(self, ins):
        return ins if self.multi else ins[0]


def clip_rows_fn(B, boxes=None, perm=None, n_rois=None):
    """clip_rows for clip_digests: a per-clip operand (B rows) holds clip c in row perm[c] (default c); a per-RoI one
    (n_rois rows, default all of boxes) holds clip c in the rows boxes[c]."""
    perm = list(range(B)) if perm is None else perm
    n_rois = sum(len(b) for b in boxes) if n_rois is None and boxes is not None else n_rois

    def rows(n, per_roi):
        if per_roi:
            assert boxes is not None and n == n_rois, (n, n_rois)
            return boxes
        assert n == B, (n, B)
        return [[perm[c]] for c in range(B)]
    return rows


def clip_operands(spec):
    """(operands a record reads, operands it writes) with the staged inputs that are not plan buffers (the source
    clip, a staged mask, the RoIs of a RoIAlign), each to be sliced by record_rows."""
    from .engine.plan import MaskRef
    ins, outs = record_io(spec)
    ins = list(ins)
    k = spec["kind"]
    if k in ("to_ndhwc", "tokens_in"):
        ins.append(spec["src"])
    m = spec.get("mask")
    if isinstance(m, MaskRef) and m.tensor is not None:
        ins.append(m)
    if k == "roi_align":
        ins.append(spec["rois"])
    return ins, list(outs)


def _buf_id(t):
    from .engine.plan import Buf
    if isinstance(t, Buf):
        return id(t)
    b = getattr(t, "buf", None)
    return id(b) if b is not None and not torch.is_tensor(t) else None


_DIGEST_W = {}


def _digest_weights(n, device):
    """Odd 64-bit weights w_i, a fixed function of the index i (a multiplicative hash)."""
    w = _DIGEST_W.get(device)
    if w is None or w.numel() < n:
        i = torch.arange(max(n, 1 << 20), dtype=torch.int64, device=device)
        w = i * -7046029254386353131
        w = w ^ (w >> 31)
        w = (w * -4658895280553007687) | 1
        _DIGEST_W[device] = w
    return w[:n]


def row_digests(v):
    """One 64-bit digest per row of v [N, ...]: sum_i bits_i * w_i mod 2^64 over the bit patterns of the row, with odd
    weights w_i, so a change of any one element always changes the digest (a change of several cancels with
    probability ~2^-64).  Computed on the tensor's device; the digest includes the row's shape."""
    n = v.shape[0]
    if n == 0:
        return []
    v = v.contiguous().reshape(n, -1)
    if v.dtype == torch.bool:
        v = v.to(torch.uint8)
    v = v.view({torch.float16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}.get(v.dtype, v.dtype))
    w = _digest_weights(v.shape[1], v.device)
    d = torch.stack([(r.long() * w).sum() for r in v])
    return [(v.shape[1], h) for h in d.tolist()]


def _clip_digests_of(spec, items, role, clip_rows, per_roi):
    per_clip = None
    for t in items:
        rows = record_rows(spec, t, role)
        dig = row_digests(rows)
        sel = clip_rows(rows.shape[0], per_roi(t))
        if per_clip is None:
            per_clip = [[] for _ in sel]
        for c, r in enumerate(sel):
            per_clip[c].append(tuple(dig[j] for j in r))
    return [tuple(d) for d in per_clip] if per_clip is not None else None


def clip_digests(plan, clip_rows, corrupt=None):
    """Run the plan op by op on one stream and digest, for every op with a record and every clip, the rows of each
    operand it reads (just before it runs) and of each it writes (just after), the rows the op reads / writes
    (record_rows with a role).  clip_rows(n, per_roi): for an operand with n rows, the rows of each clip.  An operand
    is per RoI when it is a RoIAlign's RoIs or a buffer an op wrote from a per-RoI operand (the plan's data flow, not
    its row count).  corrupt(i, spec): called after op i ran, before its digests.
    Returns {(op name, occurrence): (launched instances, [input digests per clip], [output digests per clip], ids of
    the buffers the op reads, ids of those it writes)}."""
    sp = torch.cuda.current_stream().cuda_stream
    out, seen, roi_bufs = {}, {}, set()
    for i, ((name, fn), spec) in enumerate(zip(plan.ops, plan.op_spec)):
        key = (name, seen.get(name, 0))
        seen[name] = key[1] + 1
        if spec is None:
            fn(sp)
            continue
        ins, outs = clip_operands(spec)

        def per_roi(t):
            return t is spec.get("rois") or _buf_id(t) in roi_bufs
        d_in = _clip_digests_of(spec, ins, "read", clip_rows, per_roi)
        roi_op = any(per_roi(t) for t in ins)
        reads = frozenset(b for b in map(_buf_id, ins) if b is not None)
        writes = frozenset(b for b in map(_buf_id, outs) if b is not None)
        roi_bufs = (roi_bufs | writes) if roi_op else (roi_bufs - writes)
        c0 = kernel_counts()
        fn(sp)
        torch.cuda.synchronize()
        launched = frozenset(kernel_count_diff(c0, kernel_counts()))
        if corrupt is not None:
            corrupt(i, spec)
        out[key] = (launched, d_in, _clip_digests_of(spec, outs, "write", clip_rows, per_roi), reads, writes)
    return out


def invariance_failures(want, got, exempt_prefixes=()):
    """Bitwise invariance between two runs' clip_digests, clip by clip (the lists are matched by position): where an
    op launched the same instances in both runs and read bit-equal rows for a clip, it must write bit-equal rows for
    that clip.  An op that launched other instances, or an instance named by exempt_prefixes (kernels whose bits
    depend on the batch by design), makes no claim (exempt).  Returns (failures [(op key, clips)],
    held [op keys whose claim was checked on every clip], exempt [(op key, instances in want, instances in got)],
    unexplained [op keys neither held, exempt nor failed that read no buffer written downstream of an exempt op in
    want's plan]).  With no failure and no exemption every op must be held: any other op read a row the two runs
    wrote differently without an op that wrote it being named."""
    assert list(want) == list(got), sorted(set(want) ^ set(got))[:10]
    failures, held, exempt, unexplained = [], [], [], []
    tainted = set()
    for key, w in want.items():
        inst_w, in_w, out_w, reads, writes = w
        inst_g, in_g, out_g = got[key][:3]
        if inst_w != inst_g or (exempt_prefixes and any(n.startswith(tuple(exempt_prefixes)) for n in inst_w)):
            exempt.append((key, sorted(inst_w), sorted(inst_g)))
            tainted |= writes
            continue
        n = len(out_w)
        same_in = [in_w is None or in_w[c] == in_g[c] for c in range(n)]
        bad = [c for c in range(n) if same_in[c] and out_w[c] != out_g[c]]
        if bad:
            failures.append((key, bad))
        elif all(same_in):
            held.append(key)
        elif reads & tainted:
            tainted |= writes
        else:
            unexplained.append(key)
    return failures, held, exempt, unexplained


def merge_single(digests):
    """The clip_digests of the batch-1 runs of clips 0..B-1 as one run of B clips (for invariance_failures), with the
    instances all the runs launched (they differ only where the clips' plans do: the RoI count of a detection head)."""
    out = {}
    for k in digests[0]:
        inst = frozenset().union(*(d[k][0] for d in digests))
        ins = None if digests[0][k][1] is None else [d[k][1][0] for d in digests]
        out[k] = (inst, ins, [d[k][2][0] for d in digests])
    return out


# ---- the batch audit's runs (tests/test_gpu_batch_audit*.py): one (precision, case, batch) row -----------------------
BATCH_AUDIT_PARTS = ("workloads", "models", "families", "layers", "ssl")


def batch_sweep_part(row, workloads):
    """The file of the batch audit a sweep row runs in, each about ten minutes on an H100: "workloads" the bench
    architectures but csn_r101, "models" csn_r101 and the other f16 MODEL_CASES, "families" the grouped, hub-tail,
    detection and Non-local cases in f16, "ssl" the SSL trunks, "layers" the rest (audio, efficient, MViT variants,
    masked in f16; every f32 row but the trunks)."""
    p, f, c = row[:3]
    if f == "ssl":
        return "ssl"
    if p == "f16" and f == "model":
        return "workloads" if c in workloads and c != "csn_r101" else "models"
    if p == "f16" and f in ("grouped", "hub_tail", "detection", "nonlocal"):
        return "families"
    return "layers"


def batch_pools(sweep):
    """(family, case) -> the largest batch the sweep runs it at (the size of its clip pool)."""
    pools = {}
    for r in sweep:
        pools[r[1:3]] = max(pools.get(r[1:3], 1), r[3])
    return pools


_BATCH_CASE = {}
_BATCH_SINGLE = {}           # (precision, family, case, clip) -> clip_digests of the clip's batch-1 plan


def batch_case(family, case, pool):
    """The BatchCase of a case (one kept at a time)."""
    key = (family, case, pool)
    if key not in _BATCH_CASE:
        _BATCH_CASE.clear()
        _BATCH_CASE[key] = BatchCase(family, case, pool)
    return _BATCH_CASE[key]


def batch_compile(bc, ins, prec):
    from .engine import compile_model
    return compile_model(bc.model, bc.example([t.cuda() for t in ins]), dtype=prec, use_graph=False, extra=bc.extra)


def batch_digests(cm, ins, rows, corrupt=None):
    for s, t in zip(cm.static_in, ins):
        s.copy_(t)
    torch.cuda.synchronize()
    with torch.no_grad():
        return clip_digests(cm.plan, rows, corrupt)


def batch_single_digests(prec, bc, B):
    """clip_digests of the batch-1 plan of clips 0..B-1 (compiled once per case; per clip with boxes, whose RoI count
    is the plan's)."""
    cm = None
    for c in range(B):
        key = (prec, bc.family, bc.case, c)
        if key in _BATCH_SINGLE:
            continue
        ins = bc.single(c)
        if cm is None or bc.box_slot is not None:
            cm = batch_compile(bc, ins, prec)
        boxes = None
        if bc.box_slot is not None:
            boxes = [list(range(len(bc.boxes_of(c + 1)[c])))]
        _BATCH_SINGLE[key] = batch_digests(cm, ins, clip_rows_fn(1, boxes, n_rois=None if boxes is None else
                                                                 len(ins[bc.box_slot])))
    del cm
    torch.cuda.empty_cache()
    return [_BATCH_SINGLE[(prec, bc.family, bc.case, c)] for c in range(B)]


def _fmt_keys(items):
    return "; ".join("%s#%d%s" % (k[0], k[1], "" if c is None else " on clips %s" % c) for k, c in items[:20])


def run_batch_audit(prec, family, case, B, checks, pool, batch_dependent=()):
    """One row of the batch audit: (a) audit_plan on every clip (when "a" in checks), (b) position invariance under a
    rotation of the clips, in which every op must be held, (c) batch-size invariance against each clip's batch-1 plan,
    in which every op is held, exempt (other instances, or one of ``batch_dependent``'s instance prefixes) or reads
    what an exempt op's data flow wrote.  Returns the report lines (RESULT, EXEMPT, INSTANCES)."""
    import time
    t0 = time.time()
    bc = batch_case(family, case, pool)
    ins = bc.batch(B)
    cm = batch_compile(bc, ins, prec)
    plan = cm.plan
    boxes = bc.boxes_of(B)
    line = "RESULT %s %s b%d:" % (prec, case, B)
    if "a" in checks:
        for s, t in zip(cm.static_in, ins):
            s.copy_(t)
        torch.cuda.synchronize()
        with torch.no_grad():
            failures, stats = audit_plan(plan, list(range(B)))
        assert not failures, "\n".join("op %d %s: %s" % f for f in failures[:20])
        n_checked = sum(v[0] for v in stats.values())
        assert n_checked + sum(1 for s in plan.op_spec if s is None) == len(plan.ops)
        line += " (a) %d launches on %d clips, largest err/tol %s;" % (
            n_checked, B, ", ".join("%s %.3f" % (k, v[1]) for k, v in sorted(stats.items())))
    want = batch_digests(cm, ins, clip_rows_fn(B, boxes))
    rot = batch_digests(cm, bc.batch(B, rotate=True), clip_rows_fn(B, boxes, perm=[(c + 1) % B for c in range(B)]))
    del cm, plan
    torch.cuda.empty_cache()
    fb, held_b, ex_b, un_b = invariance_failures(want, rot)
    assert not fb, "position invariance: " + _fmt_keys(fb)
    not_held = [(k, None) for k in want if k not in set(held_b)]
    assert not ex_b and not not_held, "position invariance: not held: " + _fmt_keys(not_held)
    fc, held_c, exempt, un_c = invariance_failures(want, merge_single(batch_single_digests(prec, bc, B)),
                                                   exempt_prefixes=batch_dependent)
    assert not fc, "batch-size invariance against batch 1: " + _fmt_keys(fc)
    assert not un_c, "batch-size invariance: read differing rows downstream of no exempt op: " + _fmt_keys(
        [(k, None) for k in un_c])
    line += " (b) %d of %d ops held; (c) %d held, %d exempt, %d downstream of an exempt op; %.1f s" % (
        len(held_b), len(want), len(held_c), len(exempt), len(want) - len(held_c) - len(exempt), time.time() - t0)
    return [line,
            "EXEMPT %s %s b%d: %s" % (prec, case, B, "; ".join("%s: %s -> %s" % (k[0], ",".join(w), ",".join(g))
                                                              for k, w, g in exempt)),
            "INSTANCES %s %s b%d: %s" % (prec, case, B, "; ".join("%s=%s" % (k[0], ",".join(sorted(v[0])))
                                                                 for k, v in want.items()))]

# ---- Non-local block cases (tests/golden/nonlocal.pt): name -> (create_nonlocal kwargs, input shape) ---------------
NONLOCAL_CASES = {
    # I3D-NLN res3 / res4 widths (softmax, (1,2,2) pool): the wide tensor-core kernel at D = 256 / 512
    "softmax_pool_512_256": (dict(dim_in=512, dim_inner=256, pool_size=(1, 2, 2)), (1, 512, 1, 6, 8)),
    "softmax_pool_1024_512": (dict(dim_in=1024, dim_inner=512, pool_size=(1, 2, 2)), (1, 1024, 1, 4, 6)),
    # the remaining cases keep dim_in narrow (it only sets the GEMM widths and the size of the stored output) and
    # dim_inner at the head width under test
    # "dot_product" without a pool: one theta|phi|g GEMM, the linear mode at D = 256
    "dot_product_nopool_64_256": (dict(dim_in=64, dim_inner=256, pool_size=None, instantiation="dot_product"),
                                  (1, 64, 2, 6, 6)),
    "softmax_pool_norm_none": (dict(dim_in=64, dim_inner=256, pool_size=(1, 2, 2), norm=None), (1, 64, 2, 8, 8)),
    # ragged grid the pool floors: 3x7x9 -> 3x3x4 keys
    "softmax_pool_ragged": (dict(dim_in=64, dim_inner=256, pool_size=(1, 2, 2)), (1, 64, 3, 7, 9)),
    # narrow heads: softmax on the MViT kernels, the linear mode on the wide family
    "softmax_pool_32_64": (dict(dim_in=32, dim_inner=64, pool_size=(1, 2, 2)), (1, 32, 2, 8, 8)),
    "softmax_pool_32_128": (dict(dim_in=32, dim_inner=128, pool_size=(1, 2, 2)), (1, 32, 2, 8, 8)),
    "dot_product_pool_32_64": (dict(dim_in=32, dim_inner=64, pool_size=(1, 2, 2), instantiation="dot_product"),
                               (1, 32, 2, 8, 8)),
}


def build_nonlocal_case(name, create_nonlocal, seed=91):
    """(module, input) of a NONLOCAL_CASES entry built with ``create_nonlocal`` (this package's or the reference's);
    weights and input on the f16 grid, random BatchNorm statistics."""
    kw, shape = NONLOCAL_CASES[name]
    torch.manual_seed(seed)
    m = randomize_model(create_nonlocal(**kw), seed=seed, f16_weights=True).eval()
    g = torch.Generator(device="cpu")
    g.manual_seed(seed + 1)
    return m, f16_exact(torch.randn(shape, generator=g))


# I3D-R50 with the I3D-NLN layout of Non-local blocks: blocks[3] = res3, blocks[4] = res4 (blocks[2] is the stage-1
# pool); block index -> residual blocks followed by a NonLocal of half their width
I3D_NLN_LAYOUT = {3: (1, 3), 4: (1, 3, 5)}


def build_i3d_nln(hub_module, create_nonlocal):
    """(model, clip) of the I3D-NLN case: hub i3d_r50 with Non-local blocks after the I3D_NLN_LAYOUT residual blocks,
    weights and a 2 x 8 x 224^2 clip on the f16 grid."""
    model = hub_module.i3d_r50()
    for stage, idx in I3D_NLN_LAYOUT.items():
        blocks = model.blocks[stage].res_blocks
        for i in idx:
            c = blocks[i].branch2.conv_c.out_channels
            blocks[i] = nn.Sequential(blocks[i], create_nonlocal(dim_in=c, dim_inner=c // 2, pool_size=(1, 2, 2)))
    model = randomize_model(model, seed=1234, f16_weights=True).eval()
    return model, synthetic_clip(2, 8, 224, 224, seed=42, f16_values=True)


# ---- audio model / layer cases (tests/golden/audio.pt): name -> (builder, kwargs, inputs) ----------------------------
# inputs: ("avsf", B, T_fast, crop, (T_audio, F)) - slow / fast clips via slowfast_inputs (alpha 4) and a (B, 1, T, 1, F)
# spectrogram; ("audio", B, T, F); ("layer", shape) - one tensor.
AUDIO_CASES = {
    "avsf_r50": ("create_audio_visual_slowfast", {}, ("avsf", 2, 32, 224, (128, 80))),
    # the benchmarked shape, weights and inputs on the f16 grid (AUDIO_F16_GRID)
    "avsf_r50_b8_f16grid": ("create_audio_visual_slowfast", {}, ("avsf", 8, 32, 224, (128, 80))),
    "avsf_r18_norm_none": ("create_audio_visual_slowfast",
                           dict(model_depth=18, norm=None, head_pool_kernel_sizes=((8, 2, 2), (32, 2, 2), (16, 1, 10))),
                           ("avsf", 1, 32, 64, (128, 80))),
    "avsf_r18_sigmoid": ("create_audio_visual_slowfast",
                         dict(model_depth=18, activation=nn.Sigmoid,
                              head_pool_kernel_sizes=((8, 2, 2), (32, 2, 2), (16, 1, 10))),
                         ("avsf", 1, 32, 64, (128, 80))),
    "acoustic_r50": ("create_acoustic_resnet", {}, ("audio", 2, 128, 80)),
    # the reference test's arguments: kernel 3 stem, stride-2 stage 1, softmax head
    "acoustic_r50_k3": ("create_acoustic_resnet",
                        dict(stem_conv_kernel_size=(3, 1, 3), stage_temporal_stride=(2, 2, 2, 2),
                             head_pool_kernel_size=(2, 1, 2), head_activation=nn.Softmax),
                        ("audio", 2, 32, 32)),
    # SeparableBottleneckBlock alone: W-only stride (1,1,2) on an H = 1 input
    "separable_sum": ("create_acoustic_bottleneck_block",
                      dict(dim_in=32, dim_inner=16, dim_out=64, conv_a_stride=(1, 1, 1), conv_b_kernel_size=(3, 1, 3),
                           conv_b_stride=(1, 1, 2), conv_b_padding=(1, 0, 1)), ("layer", (2, 32, 6, 1, 20))),
    "separable_cat": ("create_acoustic_bottleneck_block",
                      dict(dim_in=32, dim_inner=16, dim_out=64, conv_a_stride=(1, 1, 1), conv_b_kernel_size=(3, 1, 3),
                           conv_b_stride=(1, 1, 2), conv_b_padding=(1, 0, 1)), ("layer", (2, 32, 6, 1, 20))),
}


AUDIO_F16_GRID = ("avsf_r50_b8_f16grid",)


def build_audio_case(name, builders, seed=2024):
    """(module, inputs) of an AUDIO_CASES entry built from ``builders`` (a module exposing the builder functions:
    this package's ``models`` or the reference's).  Weights from randomize_model (fresh init zeroes norm_c)."""
    fn, kw, spec = AUDIO_CASES[name]
    torch.manual_seed(seed)
    m = getattr(builders, fn)(**kw)
    if name == "separable_cat":
        m.reduce_method = "cat"
        m.conv_c = nn.Conv3d(2 * kw["dim_inner"], kw["dim_out"], kernel_size=(1, 1, 1), bias=False)
    grid = name in AUDIO_F16_GRID
    m = randomize_model(m, seed=seed, f16_weights=grid).eval()
    if spec[0] == "avsf":
        _, B, T, crop, (ta, f) = spec
        x = slowfast_inputs(synthetic_clip(B, T, crop, crop, seed=seed + 1, f16_values=grid)) + \
            [synthetic_clip(B, ta, 1, f, seed=seed + 2, channels=1, f16_values=grid)]
    elif spec[0] == "audio":
        _, B, ta, f = spec
        x = synthetic_clip(B, ta, 1, f, seed=seed + 2, channels=1, f16_values=grid)
    else:
        g = torch.Generator(device="cpu")
        g.manual_seed(seed + 3)
        x = torch.randn(spec[1], generator=g)
    return m, x


# ---- masked multistream cases (tests/golden/masked.pt): models/masked_multistream.py, layers/fusion.py --------------
# Every case runs at B = 5 (not a multiple of 8) on MASKED_MASK: ragged prefixes, a full row, a non-prefix pattern and
# a row with no valid step; "*_t1" cases run T = 1.  Feature widths are multiples of 8 (f16 token rows).
MASKED_MASK = [[1, 1, 1, 0, 0, 0, 0], [1, 1, 1, 1, 1, 1, 1], [0, 1, 0, 1, 1, 0, 0], [0, 0, 0, 0, 0, 0, 0],
               [1, 1, 1, 1, 1, 0, 0]]
MASKED_FUSIONS = ("concat", "temporal_concat", "max", "sum", "prod")
MASKED_CASES = tuple(["pool_max", "pool_avg", "pool_sum", "pool_avg_nomask", "pool_max_t1", "default", "posenc", "mha",
                      "mha_nomask", "mha_d32_t1", "mha_d128", "chain", "encoder_1", "encoder_2", "encoder_nomask",
                      "lstm_uni", "lstm_bi", "lstm_bi_t1", "lstm_nomask"] +
                     ["multipath_" + f for f in MASKED_FUSIONS])


def masked_case_inputs(name, seed=7):
    """(x, mask or None) of a case; x is (B, T, F), or (B, F) for "default"."""
    g = torch.Generator().manual_seed(seed)
    F = {"mha_d32_t1": 32, "mha_d128": 128}.get(name, 64)
    mask = torch.tensor(MASKED_MASK, dtype=torch.bool)
    if name.endswith("_t1"):
        mask = mask[:, :1]
    B, T = mask.shape
    x = torch.randn(B, F, generator=g) if name == "default" else torch.randn(B, T, F, generator=g)
    return x, (None if name.endswith("nomask") or name == "posenc" else mask)


def build_masked_case(name, ns, seed=1234):
    """The case's module tree built from ``ns``, a namespace with the masked_multistream classes, ``PositionalEncoding``
    and ``make_fusion_layer`` (this package's or the reference's), with seeded parameters; eval mode."""
    torch.manual_seed(seed)
    F = {"mha_d32_t1": 32, "mha_d128": 128}.get(name, 64)
    if name.startswith("pool_"):
        m = ns.MaskedTemporalPooling(name.split("_")[1])
    elif name == "default":
        m = ns.LearnMaskedDefault(F)
    elif name == "posenc":
        m = ns.PositionalEncoding(F, seq_len=16)
    elif name.startswith("mha"):
        m = ns.TransposeMultiheadAttention(F, {"mha_d32_t1": 1, "mha_d128": 1}.get(name, 2))
    elif name == "chain":       # the usage example of models/masked_multistream.py:17-32
        m = ns.MaskedSequential(ns.PositionalEncoding(F), torch.nn.Dropout(p=0.1), ns.TransposeMultiheadAttention(F, 2),
                                ns.MaskedTemporalPooling(method="avg"), torch.nn.LayerNorm(F), ns.LearnMaskedDefault(F))
    elif name.startswith("encoder"):
        m = ns.TransposeTransformerEncoder(F, 2, 2 if name == "encoder_2" else 1)
    elif name.startswith("lstm"):
        m = ns.LSTM(F, 48 if name == "lstm_uni" else 32, bidirectional=name != "lstm_uni")
    elif name.startswith("multipath_"):
        m = ns.MaskedMultiPathWay(multipathway_blocks=torch.nn.ModuleList([
            ns.MaskedSequential(ns.TransposeMultiheadAttention(F, 2), ns.MaskedTemporalPooling("avg"),
                                ns.LearnMaskedDefault(F)),
            ns.MaskedSequential(torch.nn.Linear(F, F), ns.LSTM(F, F // 2, bidirectional=True), torch.nn.LayerNorm(F))]),
            multipathway_fusion=ns.make_fusion_layer(name[len("multipath_"):], [F, F]))
    else:
        raise KeyError(name)
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn(p.shape) * (0.5 / max(1, p.shape[-1]) ** 0.5 if p.dim() > 1 else 0.2))
    return m.eval()


def masked_namespace():
    """This package's masked_multistream classes, ``PositionalEncoding`` and ``make_fusion_layer``: the namespace
    build_masked_case takes."""
    import types
    import pytorchvideo_b200.layers as ML
    import pytorchvideo_b200.models as MM
    names = ("MaskedTemporalPooling", "LearnMaskedDefault", "TransposeMultiheadAttention", "TransposeTransformerEncoder",
             "LSTM", "MaskedSequential", "MaskedMultiPathWay")
    return types.SimpleNamespace(make_fusion_layer=ML.make_fusion_layer, PositionalEncoding=ML.PositionalEncoding,
                                 **{n: getattr(MM, n) for n in names})


def masked_engine_args(name, x, mask):
    """(inputs, extra) of a case as the masked modules hand them to the engine (engine/lower.py ``lower_only``)."""
    if name == "posenc":
        return x, ()
    multi = name.startswith("multipath_")
    has = mask is not None
    ins = ([x, mask] if has else [x]) * (2 if multi else 1)
    return ins, (("masks", multi) + (has,) * (2 if multi else 1),)


def masked_call(m, x, mask):
    """The reference's calling convention of a case's root module.  Each stream gets a mask object of its own: the
    reference's attention modules write mask[:, 0] = True into the object they receive, which would leak into the
    other streams through a shared one."""
    if type(m).__name__ == "MaskedMultiPathWay":
        return m([(x, None if mask is None else mask.clone()), (x, None if mask is None else mask.clone())])
    if type(m).__name__ == "MaskedSequential":
        return m(input=x, mask=mask)
    if type(m).__name__ == "PositionalEncoding":
        return m(x)
    return m(x, mask)


# ---- Efficient X3D / mobile efficient-block cases (tests/golden/efficient_x3d.pt) -----------------------------------
# name: (class in the efficient-block namespace, kwargs, input shape, f16_grid)
_XS_CLIP = (1, 3, 4, 160, 160)
EFFICIENT_CASES = {
    "xs_b2": ("EfficientX3d", {"expansion": "XS"}, (2, 3, 4, 160, 160), False),
    "xs_b8_f16grid": ("EfficientX3d", {"expansion": "XS"}, (8, 3, 4, 160, 160), True),
    "s_b1": ("EfficientX3d", {"expansion": "S"}, (1, 3, 13, 160, 160), False),
    "m_b1": ("EfficientX3d", {"expansion": "M"}, (1, 3, 16, 224, 224), False),
    "xs_no_head": ("EfficientX3d", {"enable_head": False}, _XS_CLIP, False),
    "xs_head_relu": ("EfficientX3d", {"head_act": "relu"}, _XS_CLIP, False),
    "xs_head_swish": ("EfficientX3d", {"head_act": "swish"}, _XS_CLIP, False),
    "xs_head_hswish": ("EfficientX3d", {"head_act": "hswish"}, _XS_CLIP, False),
    "block_hswish_se": ("X3dBottleneckBlock", dict(in_channels=24, mid_channels=54, out_channels=48, spatial_stride=2,
                                                   se_ratio=0.0625, act_functions=("hswish",) * 3), (2, 24, 4, 14, 14),
                        False),
    "block_hswish": ("X3dBottleneckBlock", dict(in_channels=24, mid_channels=54, out_channels=48, spatial_stride=2,
                                                se_ratio=0, act_functions=("hswish",) * 3), (2, 24, 4, 14, 14), False),
    "block_no_residual": ("X3dBottleneckBlock", dict(in_channels=24, mid_channels=54, out_channels=48, use_residual=False,
                                                     act_functions=("relu", "swish", "relu")), (2, 24, 4, 10, 10), False),
    "block_bias_no_bn": ("X3dBottleneckBlock", dict(in_channels=24, mid_channels=54, out_channels=24, bias=(True,) * 3,
                                                    use_bn=(False,) * 3, act_functions=("relu", "hswish", "hswish")),
                         (2, 24, 4, 12, 12), False),
    "conv_pw_hswish": ("Conv3dPwBnAct", dict(in_channels=24, out_channels=40, activation="hswish"), (2, 24, 3, 8, 8),
                       False),
    "conv_dw_swish": ("Conv3d3x3x3DwBnAct", dict(in_channels=40, spatial_stride=2, activation="swish"),
                      (2, 40, 3, 11, 11), False),
    "conv_t1_relu": ("Conv3dTemporalKernel1BnAct", dict(in_channels=24, out_channels=32, spatial_kernel=3,
                                                        spatial_stride=2, spatial_padding=1, activation="relu"),
                     (2, 24, 3, 12, 12), False),
    "conv_3x1x1_hswish": ("Conv3d3x1x1BnAct", dict(in_channels=24, out_channels=32, activation="hswish"),
                          (2, 24, 5, 6, 6), False),
    "conv_5x1x1_dw_hswish": ("Conv3d5x1x1BnAct", dict(in_channels=24, out_channels=24, groups=24, activation="hswish"),
                             (2, 24, 6, 8, 8), False),
}


def tree_digests_text(text):
    import hashlib
    return hashlib.sha256(text.encode()).hexdigest()


def tree_digests(model):
    """(sha256 of ``repr(model)``, sha256 of its ``state_dict`` keys in order): the module tree of a golden case in 128
    bytes instead of the ~70 kB of text of a whole Efficient X3D."""
    return tree_digests_text(repr(model)), tree_digests_text("\n".join(model.state_dict().keys()))


def efficient_namespace(root="pytorchvideo_b200"):
    """The efficient-block classes of ``root`` (this package, or "pytorchvideo" for the reference): both keep them at
    the same module paths."""
    import importlib
    import types
    ns = types.SimpleNamespace()
    for mod in ("models.accelerator.mobile_cpu.efficient_x3d", "models.accelerator.mobile_cpu.residual_blocks",
                "layers.accelerator.mobile_cpu.convolutions"):
        m = importlib.import_module(root + "." + mod)
        for k in dir(m):
            if not k.startswith("_"):
                setattr(ns, k, getattr(m, k))
    return ns


def build_efficient_case(name, ns, seed=31):
    """(module, input) of an EFFICIENT_CASES entry built from ``ns`` (efficient_namespace), with randomize_model
    weights (the residual branch's last BatchNorm drawn small, as for models/x3d.py); model inputs are synthetic clips, block inputs standard normal (straddling the HardSwish knees)."""
    cls, kw, shape, grid = EFFICIENT_CASES[name]
    torch.manual_seed(seed)
    m = getattr(ns, cls)(**kw)
    for blk in m.modules():     # the residual branch's last BatchNorm, as models/resnet.py marks norm_c
        if type(blk).__name__ == "X3dBottleneckBlock" and "bn" in blk.layers.conv_2.kernel._modules:
            blk.layers.conv_2.kernel.bn.block_final_bn = True
    m = randomize_model(m, seed=seed, f16_weights=grid).eval()
    if cls == "EfficientX3d":
        B, _, T, H, W = shape
        return m, synthetic_clip(B, T, H, W, seed=seed + 1, f16_values=grid)
    g = torch.Generator(device="cpu")
    g.manual_seed(seed + 1)
    return m, torch.randn(shape, generator=g)


@torch.no_grad()
def map_x3d_to_efficient(x3d, eff):
    """Copy the weights of a ``models.x3d.create_x3d`` network (hub x3d_xs / x3d_s) into the EfficientX3d of the same
    widths: the same network in another module tree.  The one structural difference: a stride-only shortcut
    projection of create_x3d has no BatchNorm, the efficient block's always has one; it gets the identity statistics
    (weight 1, bias 0, mean 0, var 1 - eps), which fold to scale 1.0 and bias 0.0 exactly."""
    def conv_bn(dst, conv, bn):
        k = dst.kernel
        k.conv.weight.copy_(conv.weight)
        if bn is not None:
            k.bn.load_state_dict(bn.state_dict())
        elif "bn" in k._modules:
            k.bn.weight.fill_(1.0)
            k.bn.bias.zero_()
            k.bn.running_mean.zero_()
            k.bn.running_var.fill_(1.0 - k.bn.eps)
    blocks = list(x3d.blocks)
    stem = blocks[0]
    conv_bn(eff.s1.pathway0_stem_conv_xy, stem.conv.conv_t, None)
    conv_bn(eff.s1.pathway0_stem_conv, stem.conv.conv_xy, stem.norm)
    for s, stage in enumerate(blocks[1:5]):
        dst_stage = list(getattr(eff, "s%d" % (s + 2)).children())
        assert len(dst_stage) == len(stage.res_blocks)
        for src, dst in zip(stage.res_blocks, dst_stage):
            b = src.branch2
            conv_bn(dst.layers.conv_0, b.conv_a, b.norm_a)
            conv_bn(dst.layers.conv_1, b.conv_b, b.norm_b[0])
            if "se" in dst.layers._modules:
                dst.layers.se.se.block.load_state_dict(b.norm_b[1].block.state_dict())
            else:
                assert type(b.norm_b[1]).__name__ == "Identity"
            conv_bn(dst.layers.conv_2, b.conv_c, b.norm_c)
            assert (src.branch1_conv is None) == (dst._res_proj is None)
            if src.branch1_conv is not None:
                conv_bn(dst._res_proj, src.branch1_conv, src.branch1_norm)
    head = blocks[5]
    conv_bn(eff.head.conv_5, head.pool.pre_conv, head.pool.pre_norm)
    conv_bn(eff.head.lin_5, head.pool.post_conv, head.pool.post_norm)
    eff.projection.model.load_state_dict(head.proj.state_dict())
    return eff


# ---- MViT builder variants (tests/golden/mvit_variants.pt, oracle/gen_golden_mvit_variants.py) ----------------------
_MVIT_SMALL = dict(spatial_size=64, temporal_size=4, depth=4, embed_dim_mul=[[1, 2.0], [3, 2.0]],
                   atten_head_mul=[[1, 2.0], [3, 2.0]], pool_q_stride_size=[[1, 1, 2, 2], [3, 1, 2, 2]],
                   pool_kv_stride_adaptive=[1, 4, 4], pool_kvq_kernel=[3, 3, 3])
_MVIT_B_BN = dict(spatial_size=224, temporal_size=8, norm="batchnorm", embed_dim_mul=[[1, 2.0], [3, 2.0], [14, 2.0]],
                  atten_head_mul=[[1, 2.0], [3, 2.0], [14, 2.0]], pool_q_stride_size=[[1, 1, 2, 2], [3, 1, 2, 2], [14, 1, 2, 2]],
                  pool_kv_stride_adaptive=[1, 8, 8], pool_kvq_kernel=[3, 3, 3], cls_embed_on=False)
# name: (what, builder kwargs, input shape, call fuse_bn() after randomising).  what: "model" (a clip or, without a
# patch embedding, a (B, T*H*W, C) token tensor) or "block" (a stand-alone MultiScaleBlock on tokens, thw_shape given).
# The BatchNorm MViT-B cases keep the builder's own initialisation (seed 42) and randomise only the BatchNorms, as the
# reference's tests/test_fuse_bn.py does: with randomize_model's linear weights the residual stream of 16 BatchNorm
# blocks (no LayerNorm anywhere) grows to |logit| ~ 3e4 (2.7e5 after fuse_bn()), beyond the f16 range.
MVIT_VARIANT_INIT_CASES = ("bn_mvit_b", "bn_mvit_b_fused")
MVIT_VARIANT_CASES = {
    "bn_mvit_b": ("model", _MVIT_B_BN, (2, 3, 8, 224, 224), False),
    "bn_mvit_b_fused": ("model", _MVIT_B_BN, (2, 3, 8, 224, 224), True),
    "bn_small": ("model", dict(_MVIT_SMALL, norm="batchnorm", separate_qkv=False, residual_pool=True, dim_mul_in_att=True),
                 (2, 3, 4, 64, 64), False),
    "pool_first_ln": ("model", dict(_MVIT_SMALL, pool_first=True), (2, 3, 4, 64, 64), False),
    "pool_first_bn": ("model", dict(_MVIT_SMALL, pool_first=True, norm="batchnorm"), (2, 3, 4, 64, 64), False),
    "pool_first_bn_avg": ("model", dict(_MVIT_SMALL, pool_first=True, norm="batchnorm", pooling_mode="avg",
                                        pool_kvq_kernel=None), (2, 3, 4, 64, 64), False),
    "avg": ("model", dict(_MVIT_SMALL, pooling_mode="avg", pool_kvq_kernel=None), (2, 3, 4, 64, 64), False),
    "tokens": ("model", dict(spatial_size=28, temporal_size=4, depth=2, patch_embed_dim=96, enable_patch_embed=False,
                             pool_q_stride_size=[[1, 1, 2, 2]], pool_kv_stride_adaptive=[1, 4, 4],
                             pool_kvq_kernel=[3, 3, 3]), (2, 4 * 28 * 28, 96), False),
    "tokens_no_cls": ("model", dict(spatial_size=28, temporal_size=4, depth=2, patch_embed_dim=96,
                                    enable_patch_embed=False, cls_embed_on=False, pool_q_stride_size=[[1, 1, 2, 2]],
                                    pool_kv_stride_adaptive=[1, 4, 4], pool_kvq_kernel=[3, 3, 3]),
                      (2, 4 * 28 * 28, 96), False),
    "head_none": ("model", dict(_MVIT_SMALL, head=None), (2, 3, 4, 64, 64), False),
    "bn_block": ("block", dict(dim=96, dim_out=192, num_heads=2, qkv_bias=True, dim_mul_in_att=True, kernel_q=(3, 3, 3),
                               kernel_kv=(3, 3, 3), stride_q=(1, 2, 2), stride_kv=(1, 4, 4)), (2, 1 + 4 * 8 * 8, 96),
                 False),
}
MVIT_VARIANT_BLOCK_THW = (4, 8, 8)


def build_mvit_variant_case(case, create_mvit, block_cls, weight_seed=1234, input_seed=42, fuse=None):
    """(model, input, extra forward args) of a MVIT_VARIANT_CASES entry built with ``create_mvit`` /
    ``block_cls`` (this package's or the reference's).  Every weight is drawn by randomize_model, BatchNorms included
    (the ranges of the reference's tests/test_fuse_bn.py), except in MVIT_VARIANT_INIT_CASES (builder initialisation,
    random BatchNorms); fuse_bn() runs after that where the case asks for it (or as ``fuse`` overrides)."""
    what, kw, shape, case_fuse = MVIT_VARIANT_CASES[case]
    fuse = case_fuse if fuse is None else fuse
    torch.manual_seed(42 if case in MVIT_VARIANT_INIT_CASES else 0)
    if what == "block":
        model = block_cls(norm_layer=nn.BatchNorm1d, attn_norm_layer=nn.BatchNorm3d, **kw)
        extra = (list(MVIT_VARIANT_BLOCK_THW),)
    else:
        model = create_mvit(**kw)
        extra = ()
    if case in MVIT_VARIANT_INIT_CASES:
        g = torch.Generator(device="cpu")
        g.manual_seed(weight_seed)
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, nn.modules.batchnorm._BatchNorm):
                    for t, lo, hi in ((m.weight, 0.5, 1.5), (m.bias, -0.5, 0.5), (m.running_var, 0.5, 1.5),
                                      (m.running_mean, -0.5, 0.5)):
                        t.copy_(torch.rand(t.shape, generator=g) * (hi - lo) + lo)
        model.eval()
    else:
        model = randomize_model(model, seed=weight_seed).eval()
    if fuse:
        model.fuse_bn()
    g = torch.Generator(device="cpu")
    g.manual_seed(input_seed)
    x = torch.rand(shape, generator=g) if len(shape) == 5 else torch.randn(shape, generator=g)
    return model, x, extra


# ---- detection input transforms (tests/golden/boxes.pt, oracle/gen_golden_boxes.py) -------------------------------
def synthetic_xyxy(n_boxes, H, W, seed, dtype=torch.float32):
    """(n, 4) (x1, y1, x2, y2) boxes in source pixels, drawn in float64 and rounded once to ``dtype``: random boxes that
    may reach past every edge, plus (n >= 4) a degenerate box, one wholly outside the frame, the whole frame and one
    with fractional edges just past the far corner."""
    g = torch.Generator().manual_seed(seed)
    x1 = torch.rand(n_boxes, generator=g, dtype=torch.float64) * (1.4 * W) - 0.2 * W
    y1 = torch.rand(n_boxes, generator=g, dtype=torch.float64) * (1.4 * H) - 0.2 * H
    x2 = x1 + torch.rand(n_boxes, generator=g, dtype=torch.float64) * (0.6 * W)
    y2 = y1 + torch.rand(n_boxes, generator=g, dtype=torch.float64) * (0.6 * H)
    b = torch.stack([x1, y1, x2, y2], 1)
    if n_boxes >= 4:
        b[0] = torch.tensor([W * 0.37, H * 0.61, W * 0.37, H * 0.61], dtype=torch.float64)
        b[1] = torch.tensor([-30.25, -9.5, -3.125, -0.5], dtype=torch.float64)
        b[2] = torch.tensor([0.0, 0.0, float(W), float(H)], dtype=torch.float64)
        b[3] = torch.tensor([W - 1.3, H - 2.7, W + 0.49, H - 0.51], dtype=torch.float64)
    return b.to(dtype).contiguous()


# name: (function of transforms.functional, frame (H, W), number of boxes, keyword arguments).  Every case runs on
# float32 and float64 boxes; the torch and numpy global seeds are BOX_SEED + the case's position before the call.
BOX_SEED = 2024
BOX_FUNCTIONAL_CASES = {
    "clip_landscape": ("clip_boxes_to_image", (48, 64), 9, {}),
    "clip_portrait": ("clip_boxes_to_image", (64, 40), 9, {}),
    "clip_empty": ("clip_boxes_to_image", (48, 64), 0, {}),
    "crop": ("crop_boxes", (48, 64), 9, {"x_offset": 7, "y_offset": 3}),
    "crop_negative": ("crop_boxes", (48, 64), 6, {"x_offset": -4, "y_offset": 11}),
    "scale_landscape_up": ("short_side_scale_with_boxes", (48, 64), 9, {"size": 71}),
    "scale_portrait_down": ("short_side_scale_with_boxes", (64, 40), 9, {"size": 27}),
    "scale_square": ("short_side_scale_with_boxes", (48, 48), 7, {"size": 37}),
    "scale_empty": ("short_side_scale_with_boxes", (48, 64), 0, {"size": 33}),
    "random_scale_landscape": ("random_short_side_scale_with_boxes", (48, 64), 9, {"min_size": 30, "max_size": 90}),
    "random_scale_portrait": ("random_short_side_scale_with_boxes", (64, 40), 9, {"min_size": 20, "max_size": 50}),
    "random_crop_landscape": ("random_crop_with_boxes", (48, 64), 9, {"size": 32}),
    "random_crop_portrait": ("random_crop_with_boxes", (64, 40), 9, {"size": 32}),
    "random_crop_wide": ("random_crop_with_boxes", (32, 64), 8, {"size": 32}),
    "random_crop_equal": ("random_crop_with_boxes", (32, 32), 8, {"size": 32}),
    "random_crop_empty": ("random_crop_with_boxes", (48, 64), 0, {"size": 32}),
    "uniform_crop_landscape_0": ("uniform_crop_with_boxes", (48, 64), 9, {"size": 40, "spatial_idx": 0}),
    "uniform_crop_landscape_1": ("uniform_crop_with_boxes", (48, 64), 9, {"size": 40, "spatial_idx": 1}),
    "uniform_crop_landscape_2": ("uniform_crop_with_boxes", (48, 64), 9, {"size": 40, "spatial_idx": 2}),
    "uniform_crop_portrait_0": ("uniform_crop_with_boxes", (64, 40), 9, {"size": 35, "spatial_idx": 0}),
    "uniform_crop_portrait_1": ("uniform_crop_with_boxes", (64, 40), 9, {"size": 35, "spatial_idx": 1}),
    "uniform_crop_portrait_2": ("uniform_crop_with_boxes", (64, 40), 9, {"size": 35, "spatial_idx": 2}),
    "flip_p0": ("horizontal_flip_with_boxes", (48, 64), 9, {"prob": 0.0}),
    "flip_p1": ("horizontal_flip_with_boxes", (48, 64), 9, {"prob": 1.0}),
    "flip_p1_portrait": ("horizontal_flip_with_boxes", (64, 40), 9, {"prob": 1.0}),
    "flip_half": ("horizontal_flip_with_boxes", (48, 64), 9, {"prob": 0.5}),
    "flip_empty": ("horizontal_flip_with_boxes", (48, 64), 0, {"prob": 1.0}),
}


def box_case_inputs(name, dtype):
    """(seed, float32 (3, 2, H, W) clip, (K, 4) boxes of ``dtype``) of a BOX_FUNCTIONAL_CASES entry."""
    fn, (H, W), K, _ = BOX_FUNCTIONAL_CASES[name]
    i = list(BOX_FUNCTIONAL_CASES).index(name)
    return BOX_SEED + i, synthetic_clip(1, 2, H, W, seed=BOX_SEED + i)[0], synthetic_xyxy(K, H, W, seed=BOX_SEED + 100 + i,
                                                                                         dtype=dtype)


def call_box_case(F, name, images, boxes):
    """Call the case's function from the functional module ``F`` (the reference's or this package's)."""
    fn, _, _, kw = BOX_FUNCTIONAL_CASES[name]
    f = getattr(F, fn)
    if fn == "clip_boxes_to_image":
        return f(boxes, images.shape[2], images.shape[3])
    if fn == "crop_boxes":
        return f(boxes, kw["x_offset"], kw["y_offset"])
    if fn == "short_side_scale_with_boxes":
        return f(images, boxes, kw["size"])
    if fn == "random_short_side_scale_with_boxes":
        return f(images, boxes, kw["min_size"], kw["max_size"])
    if fn == "random_crop_with_boxes":
        return f(images, kw["size"], boxes)
    if fn == "uniform_crop_with_boxes":
        return f(images, kw["size"], kw["spatial_idx"], boxes)
    return f(kw["prob"], images, boxes)


# The train chain of the detection transforms: per clip clip_boxes_to_image, random_short_side_scale_with_boxes,
# random_crop_with_boxes, horizontal_flip_with_boxes, clip_boxes_to_image, on 4 clips with 0, 1, 3 and 7 boxes.
BOX_TRAIN_CHAIN = {"T": 12, "H": 60, "W": 80, "num_samples": 4, "box_counts": (0, 1, 3, 7), "random_short_side": (40, 56),
                   "crop": 36, "hflip_prob": 0.5, "seed": 85}
# The detection tutorial's ava_inference_transform on uint8 frames, then the reference detection models.
# name: (hub builder, clip frames, num_frames, slow_fast_alpha); 2 clips of 72 x 96 frames with 3 and 4 boxes.
BOX_TUTORIAL_CASES = {
    "slow_r50_detection": ("slow_r50_detection", 12, 4, None),
    "slowfast_r50_detection": ("slowfast_r50_detection", 40, 32, 4),
}
BOX_TUTORIAL = {"H": 72, "W": 96, "crop_size": 80, "box_counts": (3, 4), "mean": (0.45, 0.45, 0.45),
                "std": (0.225, 0.225, 0.225)}


def train_chain_inputs():
    """(uint8 (4, 3, T, H, W) clips, float32 box list) of BOX_TRAIN_CHAIN."""
    c = BOX_TRAIN_CHAIN
    clips = torch.stack([synthetic_u8_clip(c["T"], c["H"], c["W"], seed=c["seed"] + b) for b in range(4)])
    boxes = [synthetic_xyxy(k, c["H"], c["W"], seed=c["seed"] + 10 + b) for b, k in enumerate(c["box_counts"])]
    return clips, boxes


def tutorial_inputs(case):
    """(uint8 (2, 3, T, H, W) clips, float32 box list) of a BOX_TUTORIAL_CASES entry."""
    _, T, _, _ = BOX_TUTORIAL_CASES[case]
    c = BOX_TUTORIAL
    clips = torch.stack([synthetic_u8_clip(T, c["H"], c["W"], seed=300 + b) for b in range(2)])
    boxes = [synthetic_xyxy(k, c["H"], c["W"], seed=310 + b) for b, k in enumerate(c["box_counts"])]
    return clips, boxes


def build_tutorial_model(case, hub_module, weight_seed=1234):
    """The case's detection model with logits out and weights randomised as build_detection_case does."""
    hub = BOX_TUTORIAL_CASES[case][0]
    return randomize_model(getattr(hub_module, hub)(head_activation=None), seed=weight_seed, f16_weights=True).eval()


# ---- self-supervised models (models/simclr.py, byol.py, memory_bank.py; oracle/gen_golden_ssl.py) -----------------
SSL_VIDEO_CLIP = (2, 8, 224, 224)          # (batch, frames, height, width) of the video cases
SSL_CASES = ("simclr_unit_b1", "simclr_unit", "byol_unit", "byol_unit_mmt", "byol_syncbn", "memory_bank_unit",
             "simclr_video", "byol_video", "memory_bank_video")


def _slow_r50_trunk(ns):
    """Slow-R50 (the torch.hub slow_r50 configuration) with its head projection removed, as a self-supervised
    checkpoint is stored (``blocks[-1].proj = None``)."""
    net = ns.create_resnet(model_depth=50, model_num_class=400, stem_conv_kernel_size=(1, 7, 7),
                           head_pool_kernel_size=(8, 7, 7))
    net.blocks[-1].proj = None
    return net


def build_ssl_case(name, ns, seed=2718):
    """(module, forward args) of an SSL_CASES entry built from ``ns`` (a namespace with SimCLR, BYOL, MemoryBank,
    make_multilayer_perceptron and create_resnet: this package's or the reference's).  The constructors run under
    torch.manual_seed(seed) (MemoryBank draws its bank there), then randomize_model sets every weight; BYOL's momentum
    backbone starts as a copy of the online one, as the reference's deepcopy makes it.  Inputs come from their own
    generator."""
    g = torch.Generator().manual_seed(seed + 1)
    torch.manual_seed(seed)
    video = name.endswith("_video")
    if video:
        B, T, H, W = SSL_VIDEO_CLIP
        x1 = torch.rand((B, 3, T, H, W), generator=g)
        x2 = torch.rand((B, 3, T, H, W), generator=g)
        mlp = ns.make_multilayer_perceptron([2048, 2048, 128], norm=nn.BatchNorm1d)[0]
    if name.startswith("simclr"):
        if video:
            m = ns.SimCLR(mlp=mlp, backbone=_slow_r50_trunk(ns))
        else:
            B = 1 if name.endswith("b1") else 2
            m = ns.SimCLR(backbone=nn.Linear(8, 4), mlp=nn.Linear(4, 2), temperature=0.07)
            x1, x2 = torch.rand((B, 8), generator=g), torch.rand((B, 8), generator=g)
        args = (x1, x2)
    elif name.startswith("byol"):
        if video:
            m = ns.BYOL(backbone=_slow_r50_trunk(ns), projector=mlp, feature_dim=128, predictor_inner=512,
                        norm=nn.BatchNorm1d)
        elif name in ("byol_unit", "byol_unit_mmt"):
            m = ns.BYOL(backbone=nn.Linear(8, 4), projector=nn.Linear(4, 4), feature_dim=4, norm=nn.BatchNorm1d)
            x1, x2 = torch.rand((2, 8), generator=g), torch.rand((2, 8), generator=g)
        else:                                   # the default predictor norm, nn.SyncBatchNorm
            m = ns.BYOL(backbone=nn.Linear(16, 8), feature_dim=8, predictor_inner=32)
            x1, x2 = torch.rand((4, 16), generator=g), torch.rand((4, 16), generator=g)
        args = (x1, x2)
    else:
        if video:
            m = ns.MemoryBank(backbone=_slow_r50_trunk(ns), mlp=mlp, neg_size=4096, temperature=0.07, bank_size=4096,
                              dim=128)
        else:
            m = ns.MemoryBank(backbone=nn.Linear(8, 4), mlp=nn.Linear(4, 2), temperature=0.07, bank_size=8, dim=2)
            x1 = torch.rand((2, 8), generator=g)
        args = (x1, torch.randint(0, m.bank_size, (x1.shape[0],), generator=g))
    randomize_model(m, seed=seed + 2)
    if name.startswith("byol"):
        m.backbone_mmt.load_state_dict(m.backbone.state_dict())
    if name == "byol_unit_mmt":               # online and momentum weights apart, a momentum that moves them far
        randomize_model(m.backbone, seed=seed + 3)
        m.update_mmt(0.5)
    return m.eval(), args


SOFT_CE_CASES = {                          # name: (N, C, target kind, normalize_targets, reduction)
    "c2_dense": (5, 2, "dense", True, "mean"),
    "c4_index": (7, 4, "index", True, "mean"),
    "c128_dense_none": (33, 128, "dense", True, "none"),
    "c2048_dense_raw": (3, 2048, "dense", False, "mean"),
    "c400_index_none": (9, 400, "index", False, "none"),
}


def soft_ce_case(name, seed=404):
    """(logits, targets, kwargs) of a SOFT_CE_CASES entry: logits with a spread of 8, soft rows that do not sum to 1
    (the normalisation then matters), or int64 class indices."""
    N, C, kind, norm, red = SOFT_CE_CASES[name]
    g = torch.Generator().manual_seed(seed + C)
    x = torch.randn((N, C), generator=g) * 4
    if kind == "dense":
        t = torch.rand((N, C), generator=g) * (torch.rand((N, C), generator=g) < 0.3)
    else:
        t = torch.randint(0, C, (N,), generator=g)
    return x, t, {"normalize_targets": norm, "reduction": red}


# ---- MoCo v2 and the kNN memory (models/moco_v2.py, knn_memory.py; oracle/gen_golden_knn_moco.py) ---------------
MOCO_CASES = {"moco_linear_v2": 2, "moco_linear_v3": 3, "moco_slow_r50": 2}    # name: views
MOCO_STEPS = {"moco_linear_v2": 2, "moco_linear_v3": 2, "moco_slow_r50": 1}    # steps (the linear cases wrap the queue)
MOCO_QUEUE_SEED = 5
MOCO_STEP_SEED = 7


def build_moco_case(name, ns, seed=2718):
    """(MOCO model, views, queue size k, dim) of a MOCO_CASES entry from ``ns`` (a namespace with MOCO,
    create_moco_resnet_50, create_mlp_util and create_resnet: this package's or the reference's).  The constructors
    run under torch.manual_seed(seed); randomize_model then sets the online and the momentum weights apart."""
    g = torch.Generator().manual_seed(seed + 1)
    torch.manual_seed(seed)
    V = MOCO_CASES[name]
    if name == "moco_slow_r50":
        m = ns.create_moco_resnet_50(backbone_creator=ns.create_resnet)
        B, k, dim = 2, 65536, 128
        views = [torch.rand((B, 3, 8, 224, 224), generator=g) for _ in range(V)]
    else:
        def part():
            return nn.Linear(16, 12), ns.create_mlp_util(12, 8, 32, 3, norm=nn.BatchNorm1d)
        (b, p), (bm, pm) = part(), part()
        m = ns.MOCO(mmt=0.5, backbone=b, projector=p, backbone_mmt=bm, projector_mmt=pm)
        B, k, dim = 4, 16, 8
        views = [torch.rand((B, 16), generator=g) for _ in range(V)]
    randomize_model(m.backbone, seed=seed + 2)
    randomize_model(m.backbone_mmt, seed=seed + 3)
    return m.eval(), views, k, dim


KNN_CASES = {                  # name: (bank rows, dim, k, classes, T, queries)
    "m1000_d8_k1": (1000, 8, 1, 10, 0.1, 5),
    "m1000_d100_k20": (1000, 100, 20, 10, 0.1, 5),
    "m1000_d128_kM": (1000, 128, 1000, 10, 0.1, 5),
    "k400_n64": (239975, 128, 200, 400, 0.1, 64),
}
KNN_UPDATES = {                # name: (bank rows, dim, momentum, batch sizes of the update sequence)
    "mmt1": (100, 16, 1.0, (8, 8)),
    "mmt05": (100, 16, 0.5, (8, 8, 8)),
    "duplicates": (10, 16, 0.5, (5000,)),
    "n1": (100, 16, 0.5, (1, 1)),
}


def knn_case(name, knn_cls, seed=31):
    """(KnnMemory on the CPU with its labels, fp32 query rows) of a KNN_CASES entry; the bank is KnnMemory's own draw
    under torch.manual_seed(seed)."""
    import types
    M, dim, k, C, T, N = KNN_CASES[name]
    torch.manual_seed(seed)
    knn = knn_cls(M, dim, momentum=1.0, downstream_classes=C, temperature=T, knn_k=k)
    g = torch.Generator().manual_seed(seed + 1)
    labels = torch.randint(0, C, (M,), generator=g)
    loader = types.SimpleNamespace(dataset=types.SimpleNamespace(
        _labeled_videos=[(i, {"label": int(v)}) for i, v in enumerate(labels.tolist())]))
    knn.init_knn_labels(loader)
    q = torch.randn((N, dim), generator=g)
    return knn, q / q.norm(dim=1, keepdim=True)


def knn_overflow_case(knn_cls, seed=41):
    """The trainer's overflow: update(momentum 1.0) stores +-1 rows; a unit query whose L1 norm exceeds 8.87 finds its
    own sign row with exp(s / 0.1) = inf.  (KnnMemory after the update, queries, the update's rows and indices)."""
    import types
    M, dim, C = 1000, 128, 10
    torch.manual_seed(seed)
    knn = knn_cls(M, dim, momentum=1.0, downstream_classes=C, temperature=0.1, knn_k=20)
    g = torch.Generator().manual_seed(seed + 1)
    labels = torch.randint(0, C, (M,), generator=g)
    loader = types.SimpleNamespace(dataset=types.SimpleNamespace(
        _labeled_videos=[(i, {"label": int(v)}) for i, v in enumerate(labels.tolist())]))
    knn.init_knn_labels(loader)
    x = torch.randn((M, dim), generator=g)
    ind = torch.arange(M)
    q = x[:4] / x[:4].norm(dim=1, keepdim=True)
    return knn, q, x, ind


def knn_update_inputs(name, seed=51):
    """[(rows, indices)] of a KNN_UPDATES sequence (repeated indices included)."""
    M, dim, _, sizes = KNN_UPDATES[name]
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn((n, dim), generator=g) * 0.1, torch.randint(0, M, (n,), generator=g)) for n in sizes]
