"""RandAugment, AugMix and RandomResizedCrop: host draws and the oracle on the CPU, the kernels on the GPU.

Goldens (tests/golden/augment.pt, oracle/gen_golden_augment.py) hold the reference's outputs and draws under fixed
seeds.  Tiers on the GPU: Invert, Posterize, Solarize, Equalize, AutoContrast, Brightness and Saturation are bit-exact;
AdjustContrast, AdjustSharpness and the warps sum in an order ATen does not fix, so float32 is held to 1e-5 absolute
and uint8 to at most 1, only at pixels whose float64 pre-cast value lies within 1e-3 of a rounding or truncation
boundary.
"""
import os
import re

import pytest
import torch

from oracle import augment_ref as O
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.transforms import AugMix, FusedClipTransform, Permute, RandAugment, RandomResizedCrop
from pytorchvideo_b200.transforms import augment as A
from pytorchvideo_b200.transforms import functional as Fv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorchvideo_b200", "csrc")
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "augment.pt"), weights_only=False)
EXACT_OPS = ("AdjustBrightness", "AdjustSaturation", "AutoContrast", "Equalize", "Invert", "Posterize", "Solarize")


def _dev():
    return torch.device("cuda:0")


def _op_id(c):
    return "%s-%s-%s" % (c["name"], c["arg"], str(c["dtype"]).split(".")[-1])


# ---- CPU: oracle and host draws ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", GOLD["ops"], ids=[_op_id(c) for c in GOLD["ops"]])
def test_oracle_reproduces_op_golden(case):
    got = O.apply_op(GOLD["op_inputs"][case["dtype"]], case["name"], case["arg"])
    assert got.dtype == case["out"].dtype and torch.equal(got, case["out"])


def test_oracle_reproduces_composite_goldens():
    for c in GOLD["randaug"]:
        assert torch.equal(O.apply_chain(c["input"], c["plan"]), c["out"]), c["seed"]
    for c in GOLD["augmix"]:
        assert torch.equal(O.augmix(c["input"], c["weights"], c["m"], c["chains"]), c["out"]), c["seed"]
    for c in GOLD["rrc"]:
        assert torch.equal(O.random_resized_crop(c["input"], c["boxes"], *c["target"]), c["out"]), c["seed"]


def test_host_draws_equal_recorded_draws():
    for c in GOLD["randaug"]:
        torch.manual_seed(c["seed"])
        assert RandAugment(**c["kwargs"]).sample() == c["plan"], c["seed"]
    for c in GOLD["augmix"]:
        torch.manual_seed(c["seed"])
        w, m, chains = AugMix(**c["kwargs"]).sample()
        assert torch.equal(w, c["weights"]) and m == c["m"] and chains == c["chains"], c["seed"]
    for c in GOLD["rrc"]:
        kw = c["kwargs"]
        torch.manual_seed(c["seed"])
        boxes = Fv.random_resized_crop_boxes(c["input"].shape[1], c["input"].shape[2], c["input"].shape[3], kw["scale"],
                                             kw["aspect_ratio"], kw.get("shift", False), kw.get("log_uniform_ratio", True))
        assert boxes == c["boxes"], c["seed"]
    for c in GOLD["fused_rrc"]:
        torch.manual_seed(c["seed"])
        H, W = c["input"].shape[2:]
        assert Fv.random_resized_crop_boxes(4, H, W, c["rrc"]["scale"], c["rrc"]["aspect_ratio"]) == c["boxes"]
        assert bool(torch.rand(1) < 0.5) == c["flip"]


def test_rrc_goldens_cover_fallback_and_shift():
    # scale > 1 fails every try: the central crop, whole frame (ratio in range) or cut to the nearest ratio
    assert GOLD["rrc"][1]["input"].shape[2:] == (29, 35)
    assert GOLD["rrc"][1]["boxes"] == [(0, 0, 29, 35)] * 3
    assert GOLD["rrc"][2]["boxes"] == [(5, 0, 18, 35)] * 3
    assert len(set(GOLD["rrc"][3]["boxes"])) > 1                       # shift=True: the window moves


def test_rotate_matrix_is_torchvisions():
    import torchvision.transforms.functional as TF
    for a in (-30.0, -7.3, 0.0, 12.5, 30.0):
        assert A.rotate_matrix(a) == TF._get_inverse_affine_matrix([0.0, 0.0], -a, [0.0, 0.0], 1.0, [0.0, 0.0])


def test_op_descriptors():
    u8, f32 = torch.uint8, torch.float32
    assert A.encode_op(("Posterize", 2), u8, 9, 9, O.FILL)[:2] == [8, 0xC0]
    assert A.encode_op(("Posterize", 0), f32, 9, 9, O.FILL)[:2] == [8, 0]
    assert A.encode_op(("Posterize", 8), u8, 9, 9, O.FILL)[0] == 0                  # 8 bits: unchanged
    assert A.encode_op(("Solarize", 0.37), u8, 9, 9, O.FILL)[:2] == [9, int(0.37 * 255.0)]
    assert A.encode_op(("Solarize", 0.37), f32, 9, 9, O.FILL)[2] == pytest.approx(0.37)
    assert A.encode_op(("AdjustSharpness", 1.5), f32, 2, 9, O.FILL)[0] == 0          # torchvision: frames <= 2 unchanged
    r = A.encode_op(("AdjustContrast", 1.3), u8, 9, 9, O.FILL)
    assert r[0] == 2 and r[2] == pytest.approx(1.3) and r[3] == pytest.approx(-0.3)
    assert A.encode_op(None, u8, 9, 9, O.FILL)[:4] == [0, 0, 0.0, 0.0]
    # the grid generator divides theta^T by (W/2, H/2) in the matrix dtype
    h, w, f = 17, 21, 0.13
    rec = A.encode_op(("ShearX", f), f32, h, w, O.FILL)
    theta = torch.tensor(O.warp_matrix("ShearX", f, h, w), dtype=torch.float32).reshape(1, 2, 3)
    want = (theta.transpose(1, 2) / torch.tensor([0.5 * w, 0.5 * h])).transpose(1, 2).reshape(-1)
    assert rec[0] == 10 and torch.equal(torch.tensor(rec[4:10], dtype=torch.float32), want)
    with pytest.raises(TypeError):
        A.encode_op(("Solarize", 1.2), f32, 9, 9, O.FILL)


def test_argument_validation():
    x = torch.zeros(2, 3, 8, 8, dtype=torch.uint8)
    with pytest.raises(RuntimeError):
        RandAugment()(x)                                              # CPU tensor
    with pytest.raises(RuntimeError):
        AugMix()(x)
    with pytest.raises(RuntimeError):
        RandomResizedCrop(4, 4, (0.5, 1.0), (0.75, 1.33))(x.float())
    with pytest.raises(NotImplementedError):
        RandomResizedCrop(4, 4, (0.5, 1.0), (0.75, 1.33), interpolation="bicubic")(x.float())
    with pytest.raises(ValueError):
        FusedClipTransform(4, random_resized_crop=dict(target_height=4, target_width=4, scale=(0.5, 1), aspect_ratio=(1, 1)),
                           crop=("center", 4))
    with pytest.raises(ValueError):
        FusedClipTransform(4, random_resized_crop=dict(target_height=4, target_width=4, scale=(0.5, 1), aspect_ratio=(1, 1),
                                                       size=3))
    with pytest.raises(NotImplementedError):
        FusedClipTransform(4, random_resized_crop=dict(target_height=4, target_width=4, scale=(0.5, 1), aspect_ratio=(1, 1),
                                                       interpolation="nearest"))
    with pytest.raises(ValueError):
        Permute((0, 0, 1))
    with pytest.raises(AssertionError):
        AugMix(magnitude=0)
    with pytest.raises(AssertionError):
        RandAugment(sampling_type="beta")
    assert Permute((1, 0, 2, 3))(x).shape == (3, 2, 8, 8)


# ---- CPU: instance ledger ---------------------------------------------------------------------------------------------
AUG_INSTANCES = {"augment_stats_kernel<uint8_t>", "augment_stats_kernel<float>", "augment_apply_kernel<uint8_t>",
                 "augment_apply_kernel<float>", "augment_mix_kernel<uint8_t>", "augment_mix_kernel<float>"}
RRC_INSTANCES = {"clip_transform_rrc_kernel<uint8_t,__half>", "clip_transform_rrc_kernel<uint8_t,float>",
                 "clip_transform_rrc_kernel<float,__half>", "clip_transform_rrc_kernel<float,float>"}
# which GPU test reaches each instance
LEDGER = {
    "augment_stats_kernel<uint8_t>": "test_gpu_op[AutoContrast-None-uint8]",
    "augment_stats_kernel<float>": "test_gpu_op[Equalize-None-float32]",
    "augment_apply_kernel<uint8_t>": "test_gpu_op[Invert-None-uint8]",
    "augment_apply_kernel<float>": "test_gpu_op[Invert-None-float32]",
    "augment_mix_kernel<uint8_t>": "test_gpu_augmix_golden",
    "augment_mix_kernel<float>": "test_gpu_augmix_golden",
    "clip_transform_rrc_kernel<uint8_t,__half>": "test_gpu_fused_rrc_golden",
    "clip_transform_rrc_kernel<uint8_t,float>": "test_gpu_fused_rrc_golden",
    "clip_transform_rrc_kernel<float,__half>": "test_gpu_rrc_f32_source_f16_out",
    "clip_transform_rrc_kernel<float,float>": "test_gpu_rrc_golden",
}


def test_instance_ledger():
    aug = open(os.path.join(CSRC, "pv_augment.cu")).read()
    assert set(re.findall(r'PV_LAUNCH_OK\("([^"]+)"\)', aug)) == AUG_INSTANCES
    tr = open(os.path.join(CSRC, "pv_transform.cu")).read()
    assert '"clip_transform_rrc_kernel<" #ST "," #OT ">"' in tr
    rrc = {"clip_transform_rrc_kernel<%s,%s>" % m for m in re.findall(r"PV_RRC\((\w+), (\w+), (?:true|false)\)", tr)}
    assert rrc == RRC_INSTANCES
    assert set(LEDGER) == AUG_INSTANCES | RRC_INSTANCES


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def _tier2(name, dtype, got, want, x):
    """Largest |difference| and the number of differing pixels, after checking the tier-2 rule."""
    d = (got.double() - want.double()).abs()
    if dtype == torch.float32:
        assert float(d.max()) <= 1e-5, (name, float(d.max()))
        return float(d.max()), int((d > 0).sum())
    assert float(d.max()) <= 1.0, (name, float(d.max()))
    return float(d.max()), int((d > 0).sum())


def _check_op(name, arg, x, got, want):
    if name in EXACT_OPS:
        assert torch.equal(got, want), (name, arg, float((got.double() - want.double()).abs().max()))
        return 0.0, 0
    worst, n = _tier2(name, x.dtype, got, want, x)
    if x.dtype == torch.uint8 and n:
        near = O.near_boundary(O.pre_cast64(x, name, arg))
        assert bool(near[got != want].all()), (name, arg, "a differing pixel is not at a rounding boundary")
    return worst, n


@pytest.mark.gpu
@pytest.mark.parametrize("case", GOLD["ops"], ids=[_op_id(c) for c in GOLD["ops"]])
def test_gpu_op(case):
    x = GOLD["op_inputs"][case["dtype"]]
    plan = [[(case["name"], case["arg"])]]
    got, launched = TS.launched_kernels(lambda: A.run_layers(x.to(_dev()).unsqueeze(0), plan)[0].cpu())
    tag = "uint8_t" if x.dtype == torch.uint8 else "float"
    assert launched.get("augment_apply_kernel<%s>" % tag) == 1, launched
    stats = case["name"] in ("AdjustContrast", "AutoContrast", "Equalize")
    assert launched.get("augment_stats_kernel<%s>" % tag, 0) == (1 if stats else 0), launched
    worst, n = _check_op(case["name"], case["arg"], x, got, case["out"])
    print("AUGOP %s max|d|=%g differing=%d" % (_op_id(case), worst, n))


def _check_composite(what, got, want):
    d = (got.double() - want.double()).abs()
    if want.dtype == torch.float32:
        assert float(d.max()) <= 1e-5, (what, float(d.max()))
    else:
        assert float(d.max()) <= 1.0, (what, float(d.max()))
    print("AUGCOMP %s max|d|=%g differing=%d of %d" % (what, float(d.max()), int((d > 0).sum()), d.numel()))


@pytest.mark.gpu
def test_gpu_randaug_golden():
    for c in GOLD["randaug"]:
        torch.manual_seed(c["seed"])
        got = RandAugment(**c["kwargs"])(c["input"].to(_dev())).cpu()
        _check_composite("randaug-%d-%s" % (c["seed"], c["input"].dtype), got, c["out"])


@pytest.mark.gpu
def test_gpu_augmix_golden():
    seen = set()
    for c in GOLD["augmix"]:
        torch.manual_seed(c["seed"])
        got, launched = TS.launched_kernels(lambda: AugMix(**c["kwargs"])(c["input"].to(_dev())).cpu())
        seen |= {k for k in launched if k.startswith("augment_mix_kernel")}
        _check_composite("augmix-%d-%s" % (c["seed"], c["input"].dtype), got, c["out"])
    assert seen == {"augment_mix_kernel<uint8_t>", "augment_mix_kernel<float>"}


@pytest.mark.gpu
def test_gpu_rrc_golden():
    for c in GOLD["rrc"]:
        torch.manual_seed(c["seed"])
        got, launched = TS.launched_kernels(lambda: RandomResizedCrop(*c["target"], **c["kwargs"])(c["input"].to(_dev())).cpu())
        assert launched == {"clip_transform_rrc_kernel<float,float>": 1}, launched
        _check_composite("rrc-%d" % c["seed"], got, c["out"])


@pytest.mark.gpu
def test_gpu_rrc_f32_source_f16_out():
    c = GOLD["rrc"][0]
    got, launched = TS.launched_kernels(lambda: Fv.clip_transform_rrc(c["input"].to(_dev()), c["boxes"], c["target"],
                                                                      out_dtype=torch.float16).cpu())
    assert launched == {"clip_transform_rrc_kernel<float,__half>": 1}, launched
    assert torch.equal(got, c["out"].half())


@pytest.mark.gpu
def test_gpu_fused_rrc_golden():
    seen = set()
    for c in GOLD["fused_rrc"]:
        for out_dtype in (torch.float32, torch.float16):
            tr = FusedClipTransform(c["num_samples"], c["mean"], c["std"], random_resized_crop=c["rrc"], hflip_prob=0.5,
                                    out_dtype=out_dtype)
            torch.manual_seed(c["seed"])
            got, launched = TS.launched_kernels(lambda: tr(c["input"].to(_dev())).cpu())
            assert len(launched) == 1 and sum(launched.values()) == 1, launched
            seen |= set(launched)
            if out_dtype == torch.float32:
                _check_composite("fused-rrc-%d" % c["seed"], got, c["out"])
            else:
                assert float((got.float() - c["out"].half().float()).abs().max()) <= 2.0 ** -10 * float(c["out"].abs().max())
    assert seen == {"clip_transform_rrc_kernel<uint8_t,float>", "clip_transform_rrc_kernel<uint8_t,__half>"}


def _batch(dtype, B=4, T=3, H=29, W=35):
    clips = [TS.synthetic_u8_clip(T, H, W, seed=s).permute(1, 0, 2, 3) for s in range(B)]     # (T, 3, H, W)
    x = torch.stack(clips)
    return x if dtype == torch.uint8 else x.float() / 255.0


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32], ids=["uint8", "float32"])
@pytest.mark.parametrize("which", ["randaug", "augmix"])
def test_gpu_batch_equals_clips_and_repeats(dtype, which):
    x = _batch(dtype).to(_dev())
    make = (lambda: RandAugment(magnitude=9, num_layers=3, prob=0.8)) if which == "randaug" else (lambda: AugMix(width=3))
    torch.manual_seed(5)
    batch = make()(x).cpu()
    torch.manual_seed(5)
    m = make()
    single = torch.stack([m(x[b]).cpu() for b in range(x.shape[0])])
    assert torch.equal(batch, single)
    torch.manual_seed(5)
    assert torch.equal(make()(x).cpu(), batch)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32], ids=["uint8", "float32"])
def test_gpu_strided_inputs(dtype):
    x = _batch(dtype)                                                  # (B, T, 3, H, W)
    thwc = x.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)   # decoder THWC frames viewed as T, C, H, W
    cthw = x.permute(0, 2, 1, 3, 4).contiguous()                       # CTHW clips
    view = Permute((0, 2, 1, 3, 4))(cthw.to(_dev()))                   # (B, T, C, H, W) view
    outs = []
    for inp in (x.to(_dev()), thwc.to(_dev()), view):
        torch.manual_seed(9)
        outs.append(RandAugment(magnitude=9, num_layers=4, prob=1.0)(inp).cpu())
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    # RandomResizedCrop on a (C, T, H, W) view of (T, C, H, W) frames
    f = x[0].float().to(_dev())
    torch.manual_seed(3)
    a = RandomResizedCrop(13, 17, (0.3, 1.0), (0.75, 1.33))(Permute((1, 0, 2, 3))(f)).cpu()
    torch.manual_seed(3)
    b = RandomResizedCrop(13, 17, (0.3, 1.0), (0.75, 1.33))(f.permute(1, 0, 2, 3).contiguous()).cpu()
    assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32], ids=["uint8", "float32"])
def test_gpu_randaug_launches(dtype):
    x = _batch(dtype, B=8).to(_dev())
    torch.manual_seed(1)
    _, launched = TS.launched_kernels(lambda: RandAugment(magnitude=7, num_layers=4)(x))
    tag = "uint8_t" if dtype == torch.uint8 else "float"
    assert set(launched) <= {"augment_stats_kernel<%s>" % tag, "augment_apply_kernel<%s>" % tag}, launched
    assert launched["augment_apply_kernel<%s>" % tag] == 4 and sum(launched.values()) <= 8, launched
