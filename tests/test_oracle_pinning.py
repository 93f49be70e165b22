"""CPU: the oracle (oracle/) is pinned to the reference.

* golden vectors under tests/golden/ were produced by the REAL reference (oracle/gen_golden.py,
  run where /root/reference exists, asserting oracle == reference bit-for-bit);
* here the oracle is re-run on the regenerated seeded weights/inputs and must reproduce them;
* the reference's own known-answer tests for the transform path are restated verbatim.
"""
import os

import numpy as np
import pytest
import torch

from oracle import transforms_ref as O
from oracle.interp import oracle_forward
from pytorchvideo_b200 import testing as TS
import pytorchvideo_b200.models.hub as PH

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _gold(name):
    return torch.load(os.path.join(GOLD, name), weights_only=False)


# ---- reference known answers (reference tests/test_transforms.py) -------------------------------
def test_uniform_temporal_subsample_known_answer():
    # tests/test_transforms.py:85-102: 20 frames -> 10 samples
    assert O.linspace_indices(20, 10).tolist() == [0, 2, 4, 6, 8, 10, 12, 14, 16, 19]
    assert O.linspace_indices(20, 20).tolist() == list(range(20))       # identity
    assert O.linspace_indices(20, 1).tolist() == [0]                    # single sample = first frame
    # SlowFast slow pathway of a 32-frame clip (datamodule/transforms.py:129-136)
    assert O.linspace_indices(32, 8).tolist() == [0, 4, 8, 13, 17, 22, 26, 31]
    assert O.linspace_indices(64, 16).tolist() == [0, 4, 8, 12, 16, 21, 25, 29, 33, 37, 42, 46, 50, 54, 58, 63]


def test_indices_match_torch_linspace_everywhere():
    for t in range(1, 301, 1):
        for n in (1, 2, 3, 5, 8, 13, 16, 27, 29, 32, 64, 100, 128):
            ref = torch.clamp(torch.linspace(0, t - 1, n), 0, t - 1).long().numpy()
            assert np.array_equal(ref, O.linspace_indices(t, n)), (t, n)


def test_index_goldens_from_reference():
    g = _gold("transforms.pt")["indices"]
    for key, idx in g.items():
        t, n = (int(v) for v in key.split("_"))
        assert np.array_equal(O.linspace_indices(t, n), idx), key


def test_short_side_scale_shapes_known_answer():
    # tests/test_transforms.py:104-144: 20x10 -> short side 5 -> 10x5 ; 10x20 -> 5x10
    assert O.short_side_size(20, 10, 5) == (10, 5)
    assert O.short_side_size(10, 20, 5) == (5, 10)
    assert O.short_side_size(1080, 1920, 256) == (256, 455)


def test_center_crop_known_answer():
    # tests/test_transforms.py:334-346: 30x40 frame, crop 10 -> window [10:20, 15:25]
    assert O.center_crop_window(30, 40, 10) == (10, 15, 10, 10)


def test_uniform_crop_goldens():
    g = _gold("transforms.pt")["uniform_crop"]
    for key, (y, x) in g.items():
        h, w, size, idx = (int(v) for v in key.split("_"))
        assert O.uniform_crop_window(h, w, size, idx)[:2] == (y, x)


def test_bilinear_table_matches_aten():
    import torch.nn.functional as F
    for (i, o) in [(1080, 256), (1920, 455), (320, 224), (7, 13), (224, 224), (61, 30), (12, 1), (700, 1), (1, 5)]:
        eye = torch.eye(i).view(1, i, 1, i)
        w = F.interpolate(eye, size=(1, o), mode="bilinear", align_corners=False)[0, :, 0, :].numpy()
        i0, i1, l1 = O.bilinear_table(i, o)
        W = np.zeros((i, o), np.float32)
        for j in range(o):
            W[i0[j], j] += np.float32(1) - l1[j]
            W[i1[j], j] += l1[j]
        assert np.array_equal(W, w), (i, o)


def test_transform_chain_small_goldens():
    for c in _gold("transforms.pt")["chain_small"]:
        clip = TS.synthetic_u8_clip(c["T"], c["H"], c["W"], seed=c["seed"])
        out = O.val_chain(clip.numpy(), c["n"], c["mean"], c["std"], c["side"], c["crop"])
        np.testing.assert_allclose(out, c["out"].numpy(), rtol=0, atol=2e-6)


def test_train_chain_goldens_and_rng_draw_order():
    """tests/golden/transforms.pt["train_small"]: outputs of the REAL reference
    create_video_transform(mode="train") (RandomShortSideScale -> torchvision RandomCrop -> RandomHorizontalFlip)
    under a fixed global seed.  (a) the numpy restatement reproduces them from the recorded draws; (b) the
    product's host-side planner makes the SAME draws in the same order from the same seed; (c) the crop
    offsets equal torchvision.transforms.RandomCrop.get_params under that seed."""
    import torchvision.transforms as TV
    from pytorchvideo_b200.transforms import create_video_transform
    flips = 0
    for c in _gold("transforms.pt")["train_small"]:
        clip = TS.synthetic_u8_clip(c["T"], c["H"], c["W"], seed=c["seed"])
        side, i, j, flip = c["draws"]
        out = O.train_chain(clip.numpy(), c["n"], (0.45,) * 3, (0.225,) * 3, side, c["crop"], i, j, flip)
        np.testing.assert_allclose(out, c["out"].numpy(), rtol=0, atol=2e-6)
        tr = create_video_transform(mode="train", num_samples=c["n"], min_size=c["min_size"], max_size=c["max_size"],
                                    crop_size=c["crop"])
        torch.manual_seed(c["rng_seed"])
        idx, hw, win, pflip = tr.plan(tuple(clip.shape))
        assert hw == O.short_side_size(c["H"], c["W"], side)
        assert win == O.random_crop_window(hw[0], hw[1], c["crop"], i, j) and pflip == flip
        # torchvision's own parameter draw after the short-side draw
        torch.manual_seed(c["rng_seed"])
        torch.randint(c["min_size"], c["max_size"] + 1, (1,))
        ti, tj, th, tw = TV.RandomCrop.get_params(torch.empty(3, hw[0], hw[1]), (c["crop"], c["crop"]))
        assert (ti, tj, th, tw) == win
        flips += int(flip)
    assert 0 < flips < len(_gold("transforms.pt")["train_small"])


def test_slowfast_pack_pathway_indices():
    # pytorchvideo_trainer/datamodule/transforms.py:129-136: slow = index_select(frames, 1, linspace(0, T-1, T//alpha).long())
    for key, idx in _gold("transforms.pt")["pack_pathway"].items():
        t, a = (int(v) for v in key.split("_"))
        assert np.array_equal(O.linspace_indices(t, t // a), idx.numpy()), key


def test_normalize_zero_mean_unit_std_property():
    # tests/test_transforms.py:324-332 style property: normalising by the clip's own stats
    x = np.random.RandomState(0).rand(3, 4, 8, 8).astype(np.float32)
    m, s = x.mean(axis=(1, 2, 3)), x.std(axis=(1, 2, 3))
    y = O.normalize(x, m, s)
    np.testing.assert_allclose(y.mean(axis=(1, 2, 3)), 0, atol=1e-5)
    np.testing.assert_allclose(y.std(axis=(1, 2, 3)), 1, atol=1e-5)


# ---- models ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["x3d_xs", "x3d_m", "slowfast_r50", "slow_r50", "csn_r101", "r2plus1d_r50", "i3d_r50",
                                  "mvit_base_8x112", "mvit_base_16x4", "slowfast_r101", "c2d_r50", "x3d_s", "x3d_l",
                                  "mvit_base_32x3"])
def test_oracle_reproduces_reference_model_goldens(case):
    g = _gold("model_%s.pt" % case)
    model, inp, is_sf = TS.build_case(case, PH, g["weight_seed"], g["input_seed"])
    assert abs(TS.state_checksum(model) - g["state_checksum"]) <= 1e-6 * abs(g["state_checksum"])
    np.testing.assert_allclose(TS.tensor_checksum(inp[1] if is_sf else inp), g["input_checksum"], rtol=1e-12)
    out = oracle_forward(model, inp)
    ref = g["output"]
    # same ATen ops in the same order; allow for a different CPU's summation order
    assert out.shape == ref.shape
    assert float((out - ref).abs().max()) <= 1e-4 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("case", ["c1_x3d_xs", "slow_r50_f16w", "mvit_base_8x112_f16w"])
def test_oracle_reproduces_f16_grid_goldens(case):
    """Goldens whose weights and clip lie on the f16 grid (reference and engine multiply identical operands).
    The BASELINE-batch ones (c2/c3/c4) are pinned by the generator run and used by the GPU suite only - a
    CPU re-run costs minutes."""
    g = _gold("model_%s.pt" % case)
    assert g["f16_grid"]
    model, inp, _ = TS.build_case(case, PH, g["weight_seed"], g["input_seed"])
    assert abs(TS.state_checksum(model) - g["state_checksum"]) <= 1e-6 * abs(g["state_checksum"])
    for m in model.modules():
        if isinstance(m, (torch.nn.Conv3d, torch.nn.Linear)):
            assert torch.equal(m.weight, m.weight.half().float())
    out = oracle_forward(model, inp)
    ref = g["output"]
    assert float((out - ref).abs().max()) <= 1e-4 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("name", TS.LAYER_CASES)
def test_oracle_reproduces_reference_layer_goldens(name):
    """tests/golden/layers*.pt: outputs of the REAL reference layer classes (ConvReduce3D, Conv2plus1d in both
    orders, Mlp, MultiScaleAttention, MultiScaleBlock, positional encoding, PatchEmbed, ViT head)."""
    g = TS.load_layer_goldens(GOLD)[name]
    m, x, thw = TS.build_layer_case(name)
    assert abs(TS.state_checksum(m) - g["state_checksum"]) <= 1e-6 * abs(g["state_checksum"])
    np.testing.assert_allclose(TS.tensor_checksum(x), g["input_checksum"], rtol=1e-12)
    out = oracle_forward(m, x, thw) if thw is not None else oracle_forward(m, x)
    if thw is not None:
        out, thw_out = out
        assert list(thw_out) == g["thw_out"]
    ref = g["output"]
    assert out.shape == ref.shape
    assert float((out - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))


def test_f16_operand_floor_of_the_reference_arithmetic():
    """Why the f16 tensor-core path cannot sit inside rtol 1e-3 / atol 1e-4 on ARBITRARY fp32 weights: round
    only the conv / linear WEIGHTS to f16 (everything else, including every activation, stays in the
    reference's own fp32 CPU arithmetic) and a large share of the logits already leaves the band - the
    per-weight error is the same for every output position, so it does not average out in the pooled
    logits.  Activation rounding alone costs far less.  (X3D-XS, 1 clip.)"""
    import torch.nn.functional as RF
    import oracle.interp as OI

    class Shim:
        def __init__(self, rw, rx):
            self.rw, self.rx = rw, rx

        def __getattr__(self, k):
            return getattr(RF, k)

        def conv3d(self, x, w, b=None, *a, **k):
            return RF.conv3d(x.half().float() if self.rx else x, w.half().float() if self.rw else w, b, *a, **k)

        def linear(self, x, w, b=None):
            return RF.linear(x.half().float() if self.rx else x, w.half().float() if self.rw else w, b)

    hub, kw, B, T, H, W, _ = TS.MODEL_CASES["x3d_xs"]
    model = TS.randomize_model(getattr(PH, hub)(**kw), seed=1234).eval()
    clip = TS.synthetic_clip(1, T, H, W, seed=42)
    ref = oracle_forward(model, clip)
    scale = max(1.0, float(ref.abs().max()))

    def inside(rw, rx):
        OI.F = Shim(rw, rx)
        try:
            out = oracle_forward(model, clip)
        finally:
            OI.F = RF
        return float(((out - ref).abs() <= 1e-3 * ref.abs() + 1e-4 * scale).float().mean())

    w_only, x_only = inside(True, False), inside(False, True)
    assert w_only < 0.95, w_only           # f16 weights alone: well outside "all logits in band"
    assert x_only > w_only                 # activation rounding is the smaller term


def test_state_dict_keys_follow_the_reference_naming():
    m = PH.slowfast_r50()
    keys = set(m.state_dict())
    for k in ["blocks.0.multipathway_blocks.0.conv.weight", "blocks.0.multipathway_fusion.conv_fast_to_slow.weight",
              "blocks.1.multipathway_blocks.0.res_blocks.0.branch1_conv.weight",
              "blocks.1.multipathway_blocks.1.res_blocks.2.branch2.norm_c.running_var", "blocks.6.proj.bias"]:
        assert k in keys
    v = PH.mvit_base_16x4()
    for k in ["cls_positional_encoding.pos_embed_spatial", "blocks.1.attn.pool_q.weight",
              "blocks.1.attn._attention_pool_q.pool.weight", "blocks.0.proj.weight", "head.proj.bias"]:
        assert k in v.state_dict()
    assert len(v.state_dict()) == 482
    x = PH.x3d_xs()
    assert "blocks.1.res_blocks.0.branch2.norm_b.1.block.0.weight" in x.state_dict()
    assert "blocks.0.conv.conv_t.weight" in x.state_dict() and "blocks.5.pool.pre_conv.weight" in x.state_dict()


# ---- detection heads (SURVEY 8 row f3): tests/golden/detection.pt was produced by the REAL reference -----------------
def test_roi_align_restatement_reproduces_torchvision_golden():
    """oracle.interp.roi_align_ref (torchvision's roi_align, aligned=False, restated) vs the committed outputs of
    torchvision.ops.roi_align on the op-level case: bit-exact (same fp32 operation order)."""
    from oracle.interp import roi_align_ref
    g = _gold("detection.pt")["roi_align"]
    x, boxes, settings = TS.roi_align_case()
    np.testing.assert_allclose(TS.tensor_checksum(x), g["input_checksum"], rtol=1e-12)
    assert torch.equal(boxes, g["boxes"])
    for (osz, scale, sr), ref in zip(settings, g["outputs"]):
        out = roi_align_ref(x, boxes, osz, scale, sr)
        assert torch.equal(out, ref), (osz, scale, sr, float((out - ref).abs().max()))


@pytest.mark.parametrize("case", sorted(TS.DETECTION_CASES))
def test_oracle_reproduces_reference_detection_goldens(case):
    """Trunk + ResNetRoIHead (models/head.py:441-482, net.py:62-74) through the oracle vs the reference's own
    slow_r50_detection / slowfast_r50_detection outputs."""
    g = _gold("detection.pt")[case]
    model, inp, boxes, is_sf = TS.build_detection_case(case, PH)
    assert abs(TS.state_checksum(model) - g["state_checksum"]) <= 1e-6 * abs(g["state_checksum"])
    assert torch.equal(boxes, g["boxes"])
    out = oracle_forward(model, inp, boxes)
    ref = g["output"]
    assert out.shape == ref.shape
    assert float((out - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))


def test_fp32_trunk_emulation_predicts_the_mvit_parity_gain():
    """Why the f16 engine keeps MViT's residual stream in fp32 (DESIGN 3.4b): the reference arithmetic with every STORED
    activation rounded to f16 at the points where the engine stores f16 (Linear / LayerNorm / GELU / pooling-conv outputs,
    the softmax probabilities, the attention output) loses ~14 points of in-band logits when the residual trunk is
    rounded as well.  Emulated: 0.675 -> 0.819 for this case."""
    from oracle.interp import Oracle

    def h(t):
        return t.half().float()

    class Emu(Oracle):
        def __init__(self, trunk32):
            self.trunk32 = trunk32

        def run(self, m, x):
            y = super().run(m, x)
            if type(m).__name__ in ("Linear", "LayerNorm", "Conv3d", "GELU") and torch.is_tensor(y):
                y = h(y)
            return y

        def f_MultiScaleAttention(self, m, x, thw):     # layers/attention.py:501-544 with the engine's rounding points
            B, N, C = x.shape
            H = m.num_heads
            if m.separate_qkv:
                q, k, v = (self.run(l, x).reshape(B, N, H, -1).permute(0, 2, 1, 3) for l in (m.q, m.k, m.v))
            else:
                qkv = self.run(m.qkv, x).reshape(B, N, 3, H, -1).permute(2, 0, 3, 1, 4)
                q, k, v = qkv[0], qkv[1], qkv[2]
            q, q_thw = self._attention_pool(q, m.pool_q, thw, m.has_cls_embed, getattr(m, "norm_q", None))
            k, _ = self._attention_pool(k, m.pool_k, thw, m.has_cls_embed, getattr(m, "norm_k", None))
            v, _ = self._attention_pool(v, m.pool_v, thw, m.has_cls_embed, getattr(m, "norm_v", None))
            attn = h(((q * m.scale) @ k.transpose(-2, -1)).softmax(dim=-1))
            o = attn @ v + q if m.residual_pool else attn @ v
            return self.run(m.proj, h(o.transpose(1, 2).reshape(B, -1, m.dim_out))), q_thw

        def f_MultiScaleBlock(self, m, x, thw):         # layers/attention.py:729-757
            t = (lambda v: v) if self.trunk32 else h
            x_norm = self.run(m.norm1, x)
            x_block, thw_new = self.f_MultiScaleAttention(m.attn, x_norm, thw)
            if m.dim_mul_in_att and m.dim != m.dim_out:
                x = self.run(m.proj, x_norm)
            x_res, _ = self._attention_pool(x, m.pool_skip, thw, m.has_cls_embed, None)
            x = t(x_res + x_block)
            x_norm = self.run(m.norm2, x)
            x_mlp = self.f_Mlp(m.mlp, x_norm)
            if not m.dim_mul_in_att and m.dim != m.dim_out:
                x = self.run(m.proj, x_norm)
            return t(x + x_mlp), thw_new

        def f_SpatioTemporalClsPositionalEncoding(self, m, x):
            y = super().f_SpatioTemporalClsPositionalEncoding(m, x)
            return y if self.trunk32 else h(y)

    model, x, _ = TS.build_case("mvit_base_8x112_f16w", PH)
    with torch.no_grad():
        ref = oracle_forward(model, x)
        scale = max(1.0, float(ref.abs().max()))
        inside = {}
        for trunk32 in (False, True):
            out = Emu(trunk32).run(model, x)
            inside[trunk32] = float(((out - ref).abs() <= 1e-3 * ref.abs() + 1e-4 * scale).float().mean())
    assert inside[True] >= inside[False] + 0.08, inside
    assert inside[True] >= 0.78, inside
