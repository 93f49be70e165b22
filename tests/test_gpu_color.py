"""ColorJitterVideoSSl and the fused contrastive view chain: the oracle against Pillow and the host draws against the
reference on the CPU, the kernels on the GPU.

Exactness tiers:
  - the colour kernels (ColorJitterVideoSSl, and the uint8 views under the fused chain) are bit-exact: Pillow's
    arithmetic is integer, or float / double with one rounding per C operation, which the kernels reproduce step for
    step;
  - the fused chain's network input goes through pv_clip_transform_rrc, whose bilinear resize is held to the existing
    RandomResizedCrop tiers (f32 rtol 1e-5 / atol 2e-6, f16 rtol 1e-3 / atol 1e-4) against the reference's eager fp32
    resize.
"""
import ctypes
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import color_ref as R
from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200.transforms import (ApplyTransformToKeyOnList, ColorJitterVideoSSl, FusedContrastiveTransform,
                                          RepeatandConverttoList)
from pytorchvideo_b200.transforms import color as CJ

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "color.pt"), weights_only=False)
CHAIN = GOLD["chain_args"]
TIERS = {torch.float32: (1e-5, 2e-6), torch.float16: (1e-3, 1e-4)}
CJ_KERNELS = {"colorjitter_stats_kernel<uint8_t>", "colorjitter_apply_kernel<uint8_t>", "colorjitter_vblur_kernel"}


def _seed(s):
    torch.manual_seed(s)
    random.seed(s)


def _order(d):
    return [i for i in d["perm"] if d["factors"][i] is not None] if d["jitter"] else []


def oracle_view(u8, draw):
    """color_ref on one (3, T, H, W) uint8 clip with one view's draws (dict as recorded) -> uint8 (3, T, H, W)."""
    c, t, h, w = u8.shape
    img = np.ascontiguousarray(u8.cpu().numpy().reshape(c, t * h, w).transpose(1, 2, 0))
    out = R.color_jitter_view(img, _order(draw), draw["factors"][:3], draw["factors"][3], draw["gray"], draw["sigma"])
    return torch.from_numpy(np.ascontiguousarray(out.transpose(2, 0, 1).reshape(c, t, h, w)))


def _chain(out_dtype=torch.float32, num_views=2):
    return FusedContrastiveTransform(CHAIN["num_samples"], CHAIN["mean"], CHAIN["std"], CHAIN["bri_con_sat"],
                                     CHAIN["hue"], CHAIN["p_color_jitter"], CHAIN["p_convert_gray"],
                                     CHAIN["target_height"], CHAIN["target_width"], CHAIN["scale"],
                                     CHAIN["aspect_ratio"], hflip_prob=CHAIN["hflip_prob"], num_views=num_views,
                                     out_dtype=out_dtype)


# ---- CPU: the oracle against Pillow --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def all_rgb():
    v = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)


def test_oracle_luma_and_hsv_match_pillow_on_every_rgb_value(all_rgb):
    from PIL import Image
    for part in np.split(all_rgb, 8):                  # 2^21 values at a time keeps the float64 temporaries small
        im = Image.fromarray(part, "RGB")
        assert np.array_equal(np.asarray(im.convert("L")), R.rgb_to_l(part))
        assert np.array_equal(np.asarray(im.convert("HSV")), R.rgb_to_hsv(part))
        # every (h, s, v) byte triple through HSV -> RGB
        assert np.array_equal(np.asarray(Image.fromarray(part, "HSV").convert("RGB")), R.hsv_to_rgb(part))


@pytest.mark.parametrize("factor", [0.0, 0.1, 0.37, 0.5, 0.999, 1.0, 1.0001, 1.3, 1.6, 2.0])
def test_oracle_blends_match_pillow(factor):
    from PIL import Image, ImageEnhance
    img = np.random.default_rng(1).integers(0, 256, (48, 70, 3), dtype=np.uint8)
    img[:4, :4] = 255
    img[-4:, -4:] = 0
    pim = Image.fromarray(img)
    assert np.array_equal(np.asarray(ImageEnhance.Brightness(pim).enhance(factor)), R.brightness(img, factor))
    assert np.array_equal(np.asarray(ImageEnhance.Contrast(pim).enhance(factor)), R.contrast(img, factor))
    assert np.array_equal(np.asarray(ImageEnhance.Color(pim).enhance(factor)), R.saturation(img, factor))


@pytest.mark.parametrize("sigma", [0.1, 0.5, 1.0, 1.7, 2.0])
@pytest.mark.parametrize("shape", [(40, 57), (2, 9), (1, 5), (3, 1)])
def test_oracle_blur_matches_pillow(sigma, shape):
    """Including images shorter / narrower than the box radius, where the repeated edge pixel fills the window."""
    from PIL import Image, ImageFilter
    img = np.random.default_rng(int(sigma * 10) + shape[0]).integers(0, 256, shape + (3,), dtype=np.uint8)
    want = np.asarray(Image.fromarray(img).filter(ImageFilter.GaussianBlur(radius=sigma)))
    assert np.array_equal(R.gaussian_blur(img, sigma), want)


def test_oracle_hue_matches_torchvision():
    from PIL import Image
    import torchvision.transforms.functional as TF
    img = np.random.default_rng(2).integers(0, 256, (30, 41, 3), dtype=np.uint8)
    for h in (-0.5, -0.13, 0.0, 0.07, 0.4, 0.5):
        assert np.array_equal(np.asarray(TF.adjust_hue(Image.fromarray(img), h)), R.hue(img, h))


def test_box_blur_params_match_the_oracle():
    for sigma in (0.1, 0.5, 1.0, 1.7, 2.0, 0.73, 6.0, 8.0):
        radius = R.box_radius(sigma)
        assert CJ.box_blur_params(sigma) == R.box_weights(radius)
    assert CJ.box_blur_params(0.0) is None


# ---- CPU: goldens and draws ---------------------------------------------------------------------------------------
def test_oracle_reproduces_the_goldens():
    for c in GOLD["jitter"]:
        assert torch.equal(oracle_view(c["input"], c["draws"][0]), c["output"]), (c["name"], c["seed"])


def test_goldens_cover_every_branch():
    draws = [c["draws"][0] for c in GOLD["jitter"]]
    assert {op for d in draws for op in _order(d)} == {0, 1, 2, 3}
    for key in ("jitter", "gray"):
        assert {bool(d[key]) for d in draws} == {True, False}
    assert {d["sigma"] is None for d in draws} == {True, False}
    assert any(c["input"].shape[1] * c["input"].shape[2] < 5 and c["draws"][0]["sigma"] for c in GOLD["jitter"])
    assert {c["input"].shape[3] % 2 for c in GOLD["jitter"]} == {0, 1}


def test_jitter_host_draws_match_the_reference():
    for c in GOLD["jitter"]:
        _seed(c["seed"])
        got = ColorJitterVideoSSl(**c["args"]).sample().as_dict()
        assert got == c["draws"][0], (c["name"], c["seed"])


def test_chain_host_draws_match_the_reference():
    """B clips x 2 views, clip-major: the jitter's draws, the crop window, then the flip."""
    tr = _chain()
    for c in GOLD["chain"]:
        B, _, T, H, W = c["input"].shape
        _seed(c["seed"])
        got = [tr.sample(CHAIN["num_samples"], H, W) for _ in range(2 * B)]
        for (view, boxes, flip), want in zip(got, c["draws"]):
            assert view.as_dict() == {k: want[k] for k in ("jitter", "perm", "factors", "gray", "sigma")}
            assert boxes == want["boxes"] * CHAIN["num_samples"]
            assert flip == want["flip"]


def test_descriptor_layout_matches_the_header():
    probe = r'''
    #include <stddef.h>
    #include <stdio.h>
    #include "pv_b200.h"
    int main(){ printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n",
                       offsetof(pv_cj_view, ops), offsetof(pv_cj_view, factor), offsetof(pv_cj_view, hue_shift),
                       offsetof(pv_cj_view, gray), offsetof(pv_cj_view, blur_r), offsetof(pv_cj_view, blur_fw),
                       sizeof(pv_cj_view), offsetof(pv_colorjitter_desc, s_clip), offsetof(pv_colorjitter_desc, sw),
                       offsetof(pv_colorjitter_desc, src_dtype), offsetof(pv_colorjitter_desc, src_scale),
                       sizeof(pv_colorjitter_desc), (size_t)PV_CJ_BLUR_PASSES); return 0; }'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "p.c")
        open(c, "w").write(probe)
        exe = os.path.join(td, "p")
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True).stdout.split()]
    V, D = L.CjView, L.ColorJitterDesc
    assert got == [V.ops.offset, V.factor.offset, V.hue_shift.offset, V.gray.offset, V.blur_r.offset,
                   V.blur_fw.offset, ctypes.sizeof(V), D.s_clip.offset, D.sw.offset, D.src_dtype.offset,
                   D.src_scale.offset, ctypes.sizeof(D), 3]


def test_dict_plumbing_follows_the_reference():
    sample = {"video": "clip", "label": 3}
    out = RepeatandConverttoList(2)(sample)
    assert out is sample and out == {"video": ["clip", "clip"], "label": [3, 3]}
    out = ApplyTransformToKeyOnList("video", lambda v: v + "!")(out)
    assert out["video"] == ["clip!", "clip!"] and out["label"] == [3, 3]


def test_argument_checks_follow_torchvision():
    with pytest.raises(ValueError):
        ColorJitterVideoSSl([0.6, 0.6, 0.6], 0.7, 0.8, 0.2)           # hue range beyond 0.5
    with pytest.raises(ValueError):
        ColorJitterVideoSSl([-0.1, 0.6, 0.6], 0.1, 0.8, 0.2)
    cj = ColorJitterVideoSSl([0, 0, 0], 0, 1.0, 0.0)
    assert (cj.brightness, cj.contrast, cj.saturation, cj.hue) == (None, None, None, None)


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _deltas(before):
    after = L.kernel_counts()
    return {k: v - before.get(k, 0) for k, v in after.items() if v != before.get(k, 0)}


@pytest.mark.gpu
def test_gpu_color_jitter_matches_the_golden_bit_for_bit():
    dev = torch.device("cuda")
    for c in GOLD["jitter"]:
        x = (c["input"].float() / 255.0).to(dev)
        _seed(c["seed"])
        out = ColorJitterVideoSSl(**c["args"])(x)
        assert out.dtype == torch.float32 and out.shape == x.shape
        assert torch.equal(out.cpu(), c["output"].float() / 255.0), (c["name"], c["seed"])


@pytest.mark.gpu
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.float16])
def test_gpu_fused_chain_matches_the_golden(out_dtype):
    dev = torch.device("cuda")
    rtol, atol = TIERS[out_dtype]
    for c in GOLD["chain"]:
        _seed(c["seed"])
        views = _chain(out_dtype)(c["input"].to(dev))
        assert len(views) == 2
        for v, got in enumerate(views):
            assert got.dtype == out_dtype and got.is_contiguous()
            torch.testing.assert_close(got.float().cpu(), c["output"][:, v], rtol=rtol, atol=atol)


@pytest.mark.gpu
def test_gpu_views_equal_the_oracle_on_multi_strip_clips():
    """Every op, grayscale and the blur on clips wide and tall enough for several vertical-blur strips (a partial
    last strip included), read through a frame-index table."""
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(5)
    for (B, T, H, W) in [(2, 5, 40, 70), (1, 8, 256, 45)]:
        x = torch.randint(0, 256, (B, 3, T, H, W), dtype=torch.uint8, generator=g)
        x[:, :, :, : H // 4] = 128                                            # grey rows: HSV's s == 0 branch
        idx = [0, T - 1, T // 2] if T > 3 else [0, 1]
        draws = [dict(jitter=True, perm=[2, 1, 3, 0], factors=[1.4, 0.55, 1.7, -0.31], gray=False, sigma=1.9),
                 dict(jitter=True, perm=[3, 1, 0, 2], factors=[0.6, 1.9, 0.2, 0.45], gray=True, sigma=0.1),
                 dict(jitter=True, perm=[1, 0, 2, 3], factors=[1.0, 1.25, None, None], gray=False, sigma=None)]
        views = [CJ.ViewDraw(d["jitter"], d["perm"], d["factors"], d["gray"], d["sigma"]) for d in draws]
        clips = [k % B for k in range(len(views))]
        got = CJ.color_jitter_views(x.to(dev), views, clips, frame_idx=idx).cpu()
        for k, d in enumerate(draws):
            assert torch.equal(got[k], oracle_view(x[clips[k]][:, idx], d)), ((B, T, H, W), k)


@pytest.mark.gpu
def test_gpu_batch_equals_sequential_calls():
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(7)
    x = torch.randint(0, 256, (4, 3, 6, 18, 23), dtype=torch.uint8, generator=g).to(dev)
    cj = ColorJitterVideoSSl([0.6, 0.6, 0.6], 0.15, 0.8, 0.5, 0.7)
    xf = x.float() / 255.0
    _seed(11)
    batch = cj(xf)
    _seed(11)
    seq = torch.stack([cj(xf[b]) for b in range(4)])
    assert torch.equal(batch, seq)
    tr = _chain(torch.float16, num_views=3)
    _seed(12)
    views = tr(x)
    _seed(12)
    singles = [tr(x[b:b + 1]) for b in range(4)]
    for v in range(3):
        assert torch.equal(views[v], torch.cat([s[v] for s in singles]))


@pytest.mark.gpu
def test_gpu_uint8_float_and_thwc_inputs_agree():
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(8)
    thwc = torch.randint(0, 256, (3, 7, 20, 25, 3), dtype=torch.uint8, generator=g).to(dev)
    x_thwc = thwc.permute(0, 4, 1, 2, 3)                                       # the decoder's layout, a view
    x = x_thwc.contiguous()
    tr = _chain(torch.float32)
    runs = []
    for inp in (x, x.float(), x_thwc, x_thwc.float()):
        _seed(21)
        runs.append(tr(inp))
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert torch.equal(a, b)
    cj = ColorJitterVideoSSl([0.6, 0.6, 0.6], 0.15, 1.0, 0.3, 1.0)
    _seed(22)
    a = cj(x.float() / 255.0)
    _seed(22)
    b = cj((x_thwc.float() / 255.0))
    assert torch.equal(a, b)


@pytest.mark.gpu
def test_gpu_launch_set_is_fixed():
    """Three colour launches and one pv_clip_transform_rrc per batch, whatever the batch size and number of views."""
    dev = torch.device("cuda")
    x = torch.randint(0, 256, (8, 3, 6, 18, 23), dtype=torch.uint8).to(dev)
    seen = []
    for B, V in ((1, 1), (2, 2), (8, 2), (8, 4)):
        tr = _chain(torch.float16, num_views=V)
        _seed(3)
        before = L.kernel_counts()
        tr(x[:B])
        torch.cuda.synchronize()
        seen.append(_deltas(before))
    assert all(d == seen[0] for d in seen)
    assert seen[0] == dict({k: 1 for k in CJ_KERNELS}, **{"clip_transform_rrc_kernel<uint8_t,__half>": 1})
    before = L.kernel_counts()
    ColorJitterVideoSSl([0.6, 0.6, 0.6], 0.15, 0.8, 0.2)(x[:3].float() / 255.0)
    torch.cuda.synchronize()
    d = _deltas(before)
    assert {k: d[k] for k in d if k.startswith("colorjitter")} == {
        "colorjitter_stats_kernel<float>": 1, "colorjitter_apply_kernel<float>": 1, "colorjitter_vblur_kernel": 1}


@pytest.mark.gpu
def test_gpu_edge_cases():
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(9)
    u8 = torch.randint(0, 256, (2, 3, 3, 5, 9), dtype=torch.uint8, generator=g)
    x = (u8.float() / 255.0).to(dev)
    # hue = 0 and factors of 1 (nothing to draw), no grayscale, no blur: the clip comes back unchanged
    _seed(0)
    assert torch.equal(ColorJitterVideoSSl([0, 0, 0], 0, 1.0, 0.0, 0.0)(x), x)
    # p = 0 everywhere: unchanged; p = 1 everywhere: always grey and blurred
    _seed(0)
    assert torch.equal(ColorJitterVideoSSl([0.6, 0.6, 0.6], 0.15, 0.0, 0.0, 0.0)(x), x)
    cj = ColorJitterVideoSSl([0.6, 0.6, 0.6], 0.15, 1.0, 1.0, 1.0, (4.0, 6.0))
    _seed(1)
    draws = [cj.sample().as_dict() for _ in range(2)]
    _seed(1)
    out = cj(x)
    assert all(d["jitter"] and d["gray"] and d["sigma"] for d in draws)
    for b in range(2):                      # T*H = 15 rows, shorter than the box window; odd W = 9
        assert torch.equal((out[b].cpu() * 255).round().to(torch.uint8), oracle_view(u8[b], draws[b]))
    assert torch.equal(out[:, 0], out[:, 1]) and torch.equal(out[:, 1], out[:, 2])
    # a single row and a single column
    for shape in ((3, 1, 1, 6), (3, 2, 4, 1)):
        u = torch.randint(0, 256, shape, dtype=torch.uint8, generator=g)
        _seed(2)
        d = cj.sample().as_dict()
        _seed(2)
        got = cj((u.float() / 255.0).to(dev))
        assert torch.equal((got.cpu() * 255).round().to(torch.uint8), oracle_view(u, d))
