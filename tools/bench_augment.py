"""Time the MViT-B 16x4 recipe's augmentation on the GPU: RandAugment(magnitude=7, num_layers=4) on (T, C, H, W)
clips, then Normalize + RandomResizedCrop(224, scale (0.08, 1), ratio (0.75, 1.3333)) + horizontal flip as one
FusedClipTransform launch.  A batch of 8 clips of 16 frames, uint8 and float32, at 3x256x340 and 3x1080x1920.

Reports ms per batch, each kernel's time (torch.profiler, a separate run) and its achieved GB/s against the H100 SXM's
3.35 TB/s, the card name and power limit, and for context the oracle's eager torchvision ops on CUDA tensors of the same
batch, whose outputs are checked against the kernels' at the timed sizes.

    python tools/bench_augment.py [--iters 20] [--out results/bench_augment.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernel_times(fn, iters):
    """{kernel name: (mean us per launch, launches per call)} from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and ("augment_" in e.key or "clip_transform_rrc" in e.key):
            out[e.key.split("(")[0]] = (e.device_time_total / max(e.count, 1), e.count / iters)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from oracle import augment_ref as O
    from pytorchvideo_b200.transforms import FusedClipTransform, RandAugment
    from pytorchvideo_b200.transforms import augment as A
    dev = torch.device("cuda:0")
    mean, std = (0.45, 0.45, 0.45), (0.225, 0.225, 0.225)
    rrc = dict(target_height=224, target_width=224, scale=(0.08, 1.0), aspect_ratio=(0.75, 1.3333))
    results = {"card": card(), "rows": []}
    print("card:", results["card"])
    for (H, W) in ((256, 340), (1080, 1920)):
        for dtype in (torch.uint8, torch.float32):
            B, T = 8, 16
            g = torch.Generator().manual_seed(0)
            x = torch.randint(0, 256, (B, T, 3, H, W), generator=g, dtype=torch.uint8)
            x = (x if dtype == torch.uint8 else x.float() / 255.0).to(dev)
            ra = RandAugment(magnitude=7, num_layers=4)
            tail = FusedClipTransform(None, mean, std, div255=dtype == torch.uint8, out_dtype=torch.float32,
                                      random_resized_crop=rrc, hflip_prob=0.5)

            def recipe():
                y = ra(x)                                   # (B, T, C, H, W)
                return tail(y.permute(0, 2, 1, 3, 4))       # (B, C, T, H, W) view, no copy

            torch.manual_seed(0)
            ms = timed(recipe, args.iters)
            ktimes = kernel_times(recipe, max(2, args.iters // 4))
            frame_bytes = T * 3 * H * W * x.element_size()
            kern = {}
            for name, (us, per_call) in ktimes.items():
                if "rrc" in name:
                    nbytes = B * T * 3 * 224 * 224 * 4           # output written; the window taps are read once
                elif "stats" in name:
                    nbytes = B * frame_bytes
                else:
                    nbytes = 2 * B * frame_bytes
                kern[name] = {"us": round(us, 1), "per_call": per_call, "GBps": round(nbytes / (us * 1e-6) / 1e9, 1),
                              "share_of_hbm": round(nbytes / (us * 1e-6) / (HBM_TBS * 1e12), 3)}
            # eager torchvision ops of the oracle on the same CUDA batch, and agreement at this size
            torch.manual_seed(1)
            plans = [ra.sample() for _ in range(B)]

            def eager():
                return [O.apply_chain(x[b], plans[b]) for b in range(B)]

            eager_ms = timed(eager, max(2, args.iters // 4))
            worst, differing = 0.0, 0
            for b in range(B):                              # clip by clip: the 1080p float batch is 3.2 GB
                d = (A.run_layers(x[b:b + 1], plans[b:b + 1])[0].float() - O.apply_chain(x[b], plans[b]).float()).abs()
                worst, differing = max(worst, float(d.max())), differing + int((d > 0).sum())
                del d
            row = {"H": H, "W": W, "dtype": str(dtype).split(".")[-1], "ms_per_batch": round(ms, 3),
                   "eager_torchvision_randaug_ms": round(eager_ms, 3), "kernels": kern,
                   "randaug_vs_eager_max_abs": worst, "randaug_vs_eager_differing": differing}
            results["rows"].append(row)
            print(json.dumps(row))
            del x
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(results, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
