"""Golden vectors of the contrastive view augmentations (tests/golden/color.pt).

Runs the trainer's own ColorJitterVideoSSl, RepeatandConverttoList and ApplyTransformToKeyOnList
(pytorchvideo_trainer/datamodule/transforms.py, loaded by file path: the trainer package's __init__ needs Lightning,
and the module's ``import hydra`` gets a stub) with torchvision and Pillow on the CPU, under fixed torch and Python
seeds.  Hooks on the reference's calls record each view's draws: ColorJitter.get_params, the grayscale conversion, the
blur's sigma, the RandomResizedCrop window and the flip.  Asserts that oracle/color_ref.py applied to those draws gives
the reference's bytes, and writes the inputs, the draws and the outputs.  Runs only where the reference is importable.

    python oracle/gen_golden_color.py
"""
import importlib.util
import os
import random
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
sys.path.insert(1, "/root/reference")

GOLD = os.path.join(ROOT, "tests", "golden", "color.pt")
TRAINER_TRANSFORMS = "/root/reference/pytorchvideo_trainer/pytorchvideo_trainer/datamodule/transforms.py"

RECIPE = dict(bri_con_sat=[0.6, 0.6, 0.6], hue=0.15, p_color_jitter=0.8, p_convert_gray=0.2)
# (name, ColorJitterVideoSSl arguments, seeds, (T, H, W))
JITTER_CASES = [
    ("recipe", RECIPE, list(range(12)), (4, 12, 17)),
    ("moco_v2", dict(bri_con_sat=[0.4, 0.4, 0.4], hue=0.4, p_color_jitter=0.8, p_convert_gray=0.2), [3, 4, 5], (3, 10, 14)),
    ("all_on", dict(bri_con_sat=[0.9, 0.9, 0.9], hue=0.5, p_color_jitter=1.0, p_convert_gray=1.0, p_gaussian_blur=1.0),
     [0, 1], (3, 9, 13)),
    ("all_off", dict(bri_con_sat=[0.6, 0.6, 0.6], hue=0.15, p_color_jitter=0.0, p_convert_gray=0.0, p_gaussian_blur=0.0),
     [0], (2, 8, 11)),
    ("identity_factors", dict(bri_con_sat=[0, 0, 0], hue=0, p_color_jitter=1.0, p_convert_gray=0.0, p_gaussian_blur=0.0),
     [0], (2, 8, 11)),
    ("wide_blur_short_clip", dict(bri_con_sat=[0.6, 0.6, 0.6], hue=0.15, p_color_jitter=1.0, p_convert_gray=0.0,
                                  p_gaussian_blur=1.0, gaussian_blur_sigma=(6.0, 8.0)), [0, 1], (2, 2, 7)),
    ("fixed_sigma", dict(bri_con_sat=[0.6, 0.6, 0.6], hue=0.15, p_color_jitter=0.0, p_convert_gray=0.0,
                         p_gaussian_blur=1.0, gaussian_blur_sigma=(1.7,)), [0], (3, 6, 9)),
]
CHAIN = dict(num_samples=4, mean=(0.45, 0.45, 0.45), std=(0.225, 0.225, 0.225), target_height=12, target_width=14,
             scale=(0.2, 0.766), aspect_ratio=(0.75, 1.3333), hflip_prob=0.5)
CHAIN_SEEDS = [0, 1, 2]
CHAIN_SHAPE = (3, 10, 16, 21)          # B, T, H, W


def test_clip(t, h, w, seed):
    """uint8 (3, T, H, W): smooth colour gradients, noise, saturated corners and a grey patch (the HSV grey branch)."""
    g = torch.Generator().manual_seed(seed)
    yy = torch.linspace(0, 1, h).view(1, h, 1)
    xx = torch.linspace(0, 1, w).view(1, 1, w)
    tt = torch.linspace(0, 1, t).view(t, 1, 1)
    chans = []
    for c in range(3):
        a = torch.rand(3, generator=g)
        chans.append(a[0] * yy + a[1] * xx + a[2] * tt + 0.15 * torch.rand(t, h, w, generator=g))
    v = torch.stack(chans)
    v = (v - v.min()) / (v.max() - v.min())
    v[:, :, : max(1, h // 5), : max(1, w // 4)] = 0.0
    v[:, :, -max(1, h // 6):, -max(1, w // 5):] = 1.0
    v[:, :, h // 2, : max(1, w // 3)] = 0.5
    return (v * 255).round().to(torch.uint8)


def load_trainer_transforms():
    hydra = types.ModuleType("hydra")
    hydra.utils = types.SimpleNamespace(instantiate=None)
    sys.modules.setdefault("hydra", hydra)
    spec = importlib.util.spec_from_file_location("trainer_datamodule_transforms", TRAINER_TRANSFORMS)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class Recorder:
    """Hooks that record each view's draws from the reference's own calls."""

    def __init__(self):
        import pytorchvideo.transforms.functional as PF
        import torchvision.transforms as TT
        import torchvision.transforms.functional as TF
        from PIL import ImageFilter
        self.views = []
        rec = self
        orig_params = TT.ColorJitter.get_params
        orig_gray = TF.rgb_to_grayscale
        orig_crop = PF._get_param_spatial_crop
        orig_hflip = TF.hflip
        orig_blur = ImageFilter.GaussianBlur.__init__

        def get_params(*a):
            res = orig_params(*a)
            rec.cur.update(jitter=True, perm=[int(i) for i in res[0]], factors=list(res[1:]))
            return res

        def gray(img, num_output_channels=1):
            rec.cur["gray"] = True
            return orig_gray(img, num_output_channels)

        def crop(*a, **k):
            res = orig_crop(*a, **k)
            rec.cur.setdefault("boxes", []).append(tuple(int(v) for v in res))
            return res

        def hflip(img):
            rec.cur["flip"] = True
            return orig_hflip(img)

        def blur_init(self_, radius=2):
            rec.cur["sigma"] = radius
            orig_blur(self_, radius)

        TT.ColorJitter.get_params = staticmethod(get_params)
        TF.rgb_to_grayscale = gray
        PF._get_param_spatial_crop = crop
        TF.hflip = hflip
        ImageFilter.GaussianBlur.__init__ = blur_init

    def start(self):
        self.cur = dict(jitter=False, perm=[0, 1, 2, 3], factors=[None] * 4, gray=False, sigma=None, flip=False)
        self.views.append(self.cur)


def per_view(rec, fn):
    def run(x):
        rec.start()
        return fn(x)
    return run


def oracle_view(u8_clip, draw):
    """oracle/color_ref.py on a (3, T, H, W) uint8 clip with one view's recorded draws -> uint8 (3, T, H, W)."""
    from oracle import color_ref as R
    c, t, h, w = u8_clip.shape
    img = u8_clip.numpy().reshape(c, t * h, w).transpose(1, 2, 0)
    order = [i for i in draw["perm"] if draw["factors"][i] is not None] if draw["jitter"] else []
    out = img
    for op in order:
        f = draw["factors"][op]
        out = {0: R.brightness, 1: R.contrast, 2: R.saturation, 3: R.hue}[op](out, f)
    if draw["gray"]:
        out = R.gray3(out)
    if draw["sigma"] is not None:
        out = R.gaussian_blur(out, draw["sigma"])
    return torch.from_numpy(np.ascontiguousarray(out.transpose(2, 0, 1).reshape(c, t, h, w)))


def main():
    import torchvision
    from pytorchvideo.transforms.transforms import Div255, Normalize, RandomResizedCrop, UniformTemporalSubsample
    T = load_trainer_transforms()
    rec = Recorder()
    gold = {"jitter": [], "chain": []}
    seen = set()
    for name, args, seeds, (t, h, w) in JITTER_CASES:
        for seed in seeds:
            u8 = test_clip(t, h, w, seed + 100)
            x = u8.float() / 255.0
            torch.manual_seed(seed)
            random.seed(seed)
            cj = T.ColorJitterVideoSSl(**args)
            rec.start()
            out = cj(x)
            draw = dict(rec.cur)
            ub = (out * 255).round().to(torch.uint8)
            assert torch.equal(out, ub.float() / 255.0), "ToTensor output is not u / 255"
            assert torch.equal(oracle_view(u8, draw), ub), (name, seed, draw)
            if draw["jitter"]:
                seen.update("op%d" % i for i in draw["perm"] if draw["factors"][i] is not None)
            seen.update(k for k in ("gray", "sigma") if draw[k] not in (False, None))
            seen.update("no_" + k for k in ("jitter", "gray", "sigma") if draw[k] in (False, None))
            gold["jitter"].append({"name": name, "args": args, "seed": seed, "input": u8, "output": ub,
                                   "draws": [{k: draw[k] for k in ("jitter", "perm", "factors", "gray", "sigma")}]})
    need = {"op0", "op1", "op2", "op3", "gray", "sigma", "no_jitter", "no_gray", "no_sigma"}
    assert need <= seen, need - seen

    B, t, h, w = CHAIN_SHAPE
    for seed in CHAIN_SEEDS:
        clips = torch.stack([test_clip(t, h, w, 200 + 10 * seed + b) for b in range(B)])      # (B, 3, T, H, W)
        view_tf = torchvision.transforms.Compose([
            UniformTemporalSubsample(CHAIN["num_samples"]), Div255(), T.ColorJitterVideoSSl(**RECIPE),
            Normalize(CHAIN["mean"], CHAIN["std"]),
            RandomResizedCrop(CHAIN["target_height"], CHAIN["target_width"], CHAIN["scale"], CHAIN["aspect_ratio"]),
            torchvision.transforms.RandomHorizontalFlip(CHAIN["hflip_prob"])])
        pipeline = torchvision.transforms.Compose([
            T.RepeatandConverttoList(2), T.ApplyTransformToKeyOnList("video", per_view(rec, view_tf))])
        torch.manual_seed(seed)
        random.seed(seed)
        first = len(rec.views)
        outs = [torch.stack(pipeline({"video": clips[b]})["video"]) for b in range(B)]
        draws = [dict(v) for v in rec.views[first:]]
        assert len(draws) == 2 * B
        gold["chain"].append({"seed": seed, "input": clips, "output": torch.stack(outs), "draws": draws})
    gold["chain_args"] = dict(CHAIN, **RECIPE)
    torch.save(gold, GOLD)
    print("wrote", GOLD, "jitter cases:", len(gold["jitter"]), "chain seeds:", len(gold["chain"]))


if __name__ == "__main__":
    main()
