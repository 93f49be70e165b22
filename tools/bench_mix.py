"""Time the in-place MixUp and CutMix kernels on batches of B clips of 3x16x224x224, float32 and float16.

Reports each kernel's time (CUDA events over many launches after warm-up) and its achieved GB/s against the bytes the
algorithm must move: one read and one write of the batch for MixUp, two reads and two writes of the box region per
pair of clips for CutMix (the box of lambda = 0.5, 158 x 158).  Also the whole module call (host draws, the labels
launch and its one host sync), and, for context only, the reference's eager ATen sequence on the same GPU, whose
result is checked against the kernel's.  Prints the card name and power limit of the same run.

    python tools/bench_mix.py [--iters 50] [--out results/bench_mix.json]

Writes the results as JSON to the --out path when it is given.
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
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def eager_mixup_(x, lam):
    flipped = x.flip(0).mul_(1.0 - lam)
    x.mul_(lam).add_(flipped)
    return x


def eager_cutmix_(x, box):
    yl, yh, xl, xh = box
    x[..., yl:yh, xl:xh] = x.flip(0)[..., yl:yh, xl:xh]
    return x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from pytorchvideo_b200 import _lib
    from pytorchvideo_b200.transforms import CutMix, MixUp
    from pytorchvideo_b200.transforms import mix as M
    _lib.require_device()
    dev = torch.device("cuda:0")
    T, H, W, K = 16, 224, 224, 400
    lam = torch.tensor(0.7, dtype=torch.float32)                  # a float32 draw, as Beta.sample() returns
    side = int(H * float((1 - torch.tensor(0.5)) ** 0.5)) // 2
    box = (H // 2 - side, H // 2 + side, W // 2 - side, W // 2 + side)
    rows = []
    print("card:", card())
    for dtype in (torch.float32, torch.float16):
        es = torch.finfo(dtype).bits // 8
        for B in (8, 16, 64):
            g = torch.Generator(device=dev).manual_seed(B)
            x = torch.randn((B, 3, T, H, W), generator=g, device=dev).to(dtype)
            labels = torch.randint(0, K, (B,), device=dev)
            # correctness at the timed size: kernel against the eager sequence, from the same input
            want = eager_mixup_(x.clone(), lam)
            got = M.mixup_(x.clone(), lam, 1.0 - lam)
            mix_ok = bool(torch.equal(got, want))
            want = eager_cutmix_(x.clone(), box)
            got = M.cutmix_(x.clone(), box)
            cut_ok = bool(torch.equal(got, want))
            del want, got
            mix_bytes = 2 * x.numel() * es
            cut_bytes = 4 * (B // 2) * 3 * T * (box[1] - box[0]) * (box[3] - box[2]) * es
            t_mix = timed(lambda: M.mixup_(x, lam, 1.0 - lam), args.iters)
            t_cut = timed(lambda: M.cutmix_(x, box), args.iters)
            mixup, cutmix = MixUp(alpha=0.8, label_smoothing=0.1), CutMix(label_smoothing=0.1)
            t_mix_call = timed(lambda: mixup(x, labels), args.iters)
            t_cut_call = timed(lambda: cutmix(x, labels), args.iters)
            t_mix_eager = timed(lambda: eager_mixup_(x, lam), args.iters)
            t_cut_eager = timed(lambda: eager_cutmix_(x, box), args.iters)
            x.copy_(torch.randn((B, 3, T, H, W), generator=g, device=dev))   # keep the values finite and varied
            row = {"dtype": str(dtype).split(".")[-1], "B": B, "batch_MB": x.numel() * es / 1e6,
                   "mixup_kernel_us": t_mix * 1e3, "mixup_GBps": mix_bytes / t_mix / 1e6,
                   "mixup_share_of_hbm": mix_bytes / t_mix / 1e9 / HBM_TBS,
                   "cutmix_kernel_us": t_cut * 1e3, "cutmix_GBps": cut_bytes / t_cut / 1e6,
                   "mixup_call_us": t_mix_call * 1e3, "cutmix_call_us": t_cut_call * 1e3,
                   "eager_mixup_us": t_mix_eager * 1e3, "eager_cutmix_us": t_cut_eager * 1e3,
                   "mixup_equals_eager": mix_ok, "cutmix_equals_eager": cut_ok}
            rows.append(row)
            print(("%(dtype)s B=%(B)d (%(batch_MB).0f MB): MixUp %(mixup_kernel_us).1f us %(mixup_GBps).0f GB/s "
                   "(%(mixup_share_of_hbm).2f of 3.35 TB/s), call %(mixup_call_us).1f us, eager %(eager_mixup_us).1f us; "
                   "CutMix %(cutmix_kernel_us).1f us %(cutmix_GBps).0f GB/s, call %(cutmix_call_us).1f us, "
                   "eager %(eager_cutmix_us).1f us; equal to eager: %(mixup_equals_eager)s %(cutmix_equals_eager)s")
                  % row)
            del x
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": card(), "box": box, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
