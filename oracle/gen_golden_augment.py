"""Golden vectors of the video augmentations (tests/golden/augment.pt).

Runs the reference's own modules (RandAugment, AugMix, RandomResizedCrop and its MViT recipe tail) on the CPU under
fixed seeds, re-draws the same seeds with this package's host sampler, and asserts that oracle/augment_ref.py applied
to those draws equals the reference bit for bit.  Writes the inputs, the draws and the reference outputs.  Runs only
where the reference is importable.

    python oracle/gen_golden_augment.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
sys.path.insert(1, "/root/reference")

GOLD = os.path.join(ROOT, "tests", "golden", "augment.pt")

# per-op arguments, extremes included (RandAugment and AugMix ranges)
OP_ARGS = {
    "AdjustBrightness": [0.1, 0.55, 1.0, 1.9],
    "AdjustContrast": [0.1, 0.7, 1.9],
    "AdjustSaturation": [0.1, 1.3, 1.9],
    "AdjustSharpness": [0.1, 0.82, 1.9],
    "AutoContrast": [None],
    "Equalize": [None],
    "Invert": [None],
    "Posterize": [0, 2, 4, 8],
    "Solarize": [0.0, 0.37, 1.0],
    "Rotate": [-30.0, -7.3, 21.1],
    "ShearX": [-0.3, 0.13],
    "ShearY": [0.3, -0.07],
    "TranslateX": [-0.45, 0.21],
    "TranslateY": [0.45, -1.0 / 3.0],
}


def test_clip(t, h, w, dtype, seed):
    """Smooth gradients with saturated 0 / 255 patches, and one constant frame (AutoContrast's min == max and
    Equalize's step == 0 branches)."""
    g = torch.Generator().manual_seed(seed)
    yy = torch.linspace(0, 1, h).view(h, 1)
    xx = torch.linspace(0, 1, w).view(1, w)
    frames = []
    for i in range(t):
        if i == t - 1:
            frames.append(torch.full((3, h, w), 0.3))
            continue
        a = torch.rand(3, generator=g)
        f = torch.stack([(a[c] * yy + (1 - a[c]) * xx + 0.1 * torch.sin(6 * xx * (c + 1) + 3 * yy * i)) for c in range(3)])
        f = (f - f.min()) / (f.max() - f.min())
        f[:, : h // 5, : w // 4] = 0.0
        f[:, -(h // 6):, -(w // 5):] = 1.0
        frames.append(f)
    v = torch.stack(frames)                                  # (T, 3, H, W)
    return (v * 255).round().to(torch.uint8) if dtype == torch.uint8 else v.float()


def main():
    import torchvision
    from pytorchvideo.transforms import augmentations as RA
    from pytorchvideo.transforms.augmix import AugMix as RefAugMix
    from pytorchvideo.transforms.rand_augment import RandAugment as RefRandAugment
    from pytorchvideo.transforms.transforms import Div255, Normalize, RandomResizedCrop, UniformTemporalSubsample
    from oracle import augment_ref as O
    from pytorchvideo_b200.transforms import augment as A
    from pytorchvideo_b200.transforms import functional as Fv

    gold = {"ops": [], "randaug": [], "augmix": [], "rrc": [], "fused_rrc": []}
    clips = {dt: test_clip(2, 17, 21, dt, 7) for dt in (torch.uint8, torch.float32)}
    gold["op_inputs"] = clips
    for name, args in OP_ARGS.items():
        for arg in args:
            for dt, x in clips.items():
                fn = RA._NAME_TO_TRANSFORM_FUNC[name]
                ref = fn(x, *(() if arg is None else (arg,)), fill=O.FILL)
                got = O.apply_op(x, name, arg)
                assert got.dtype == ref.dtype and torch.equal(got, ref), (name, arg, dt)
                gold["ops"].append({"name": name, "arg": arg, "dtype": dt, "out": ref.clone()})

    for seed, kw in [(11, dict(magnitude=7, num_layers=4)), (12, dict(magnitude=9, num_layers=2, prob=0.9)),
                     (13, dict(magnitude=7, num_layers=4, sampling_type="uniform")),
                     (14, dict(magnitude=10, num_layers=3, prob=1.0))]:
        for dt in (torch.uint8, torch.float32):
            x = test_clip(2, 21, 25, dt, seed)
            torch.manual_seed(seed)
            ref = RefRandAugment(**kw)(x)
            torch.manual_seed(seed)
            plan = A.RandAugment(**kw).sample()
            assert torch.equal(O.apply_chain(x, plan), ref), (seed, dt, plan)
            gold["randaug"].append({"seed": seed, "kwargs": kw, "input": x, "plan": plan, "out": ref.clone()})

    for seed, kw in [(21, dict()), (22, dict(magnitude=6, depth=2, width=2)), (23, dict(magnitude=10, alpha=0.5))]:
        for dt in (torch.uint8, torch.float32):
            x = test_clip(2, 19, 23, dt, seed)
            torch.manual_seed(seed)
            ref = RefAugMix(**kw)(x)
            torch.manual_seed(seed)
            w, m, chains = A.AugMix(**kw).sample()
            assert torch.equal(O.augmix(x, w, m, chains), ref), (seed, dt)
            gold["augmix"].append({"seed": seed, "kwargs": kw, "input": x, "weights": w, "m": m, "chains": chains,
                                   "out": ref.clone()})

    frames = test_clip(3, 29, 35, torch.float32, 31).permute(1, 0, 2, 3).contiguous()    # (C, T, H, W)
    for seed, kw in [(31, dict(scale=(0.08, 1.0), aspect_ratio=(0.75, 1.3333))),
                     (32, dict(scale=(2.0, 3.0), aspect_ratio=(0.75, 1.3333))),               # every try fails
                     (33, dict(scale=(2.0, 3.0), aspect_ratio=(2.0, 3.0), log_uniform_ratio=False)),
                     (34, dict(scale=(0.2, 0.9), aspect_ratio=(0.5, 2.0), shift=True))]:
        torch.manual_seed(seed)
        ref = RandomResizedCrop(19, 23, **kw)(frames)
        torch.manual_seed(seed)
        boxes = Fv.random_resized_crop_boxes(frames.shape[1], 29, 35, kw["scale"], kw["aspect_ratio"],
                                             kw.get("shift", False), kw.get("log_uniform_ratio", True))
        assert torch.equal(O.random_resized_crop(frames, boxes, 19, 23), ref), seed
        gold["rrc"].append({"seed": seed, "kwargs": kw, "target": (19, 23), "input": frames, "boxes": boxes,
                            "out": ref.clone()})

    # the MViT recipe's tail after RandAugment: subsample, /255, Normalize, RandomResizedCrop, RandomHorizontalFlip
    u8 = test_clip(6, 29, 35, torch.uint8, 41).permute(1, 0, 2, 3).contiguous()
    mean, std = (0.45, 0.45, 0.45), (0.225, 0.225, 0.225)
    rrc = dict(target_height=19, target_width=23, scale=(0.08, 1.0), aspect_ratio=(0.75, 1.3333))
    for seed in (41, 42, 43):
        chain = torchvision.transforms.Compose([UniformTemporalSubsample(4), Div255(), Normalize(mean, std),
                                                RandomResizedCrop(**rrc), torchvision.transforms.RandomHorizontalFlip()])
        torch.manual_seed(seed)
        ref = chain(u8)
        torch.manual_seed(seed)
        boxes = Fv.random_resized_crop_boxes(4, 29, 35, rrc["scale"], rrc["aspect_ratio"])
        flip = bool(torch.rand(1) < 0.5)
        idx = Fv.temporal_indices(6, 4)
        x = (u8[:, idx].float() / 255.0 - torch.tensor(mean).view(3, 1, 1, 1)) / torch.tensor(std).view(3, 1, 1, 1)
        want = O.random_resized_crop(x, boxes, 19, 23)
        want = want.flip(-1) if flip else want
        assert torch.equal(want, ref), seed
        gold["fused_rrc"].append({"seed": seed, "rrc": rrc, "mean": mean, "std": std, "num_samples": 4, "input": u8,
                                  "boxes": boxes, "flip": flip, "out": ref.clone()})
    torch.save(gold, GOLD)
    print("wrote", GOLD, os.path.getsize(GOLD), "bytes;", {k: len(v) for k, v in gold.items() if isinstance(v, list)})


if __name__ == "__main__":
    main()
