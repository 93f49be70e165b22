"""Time the contrastive view chain of the SimCLR / BYOL recipes (kinetics_contrastive.yaml) on the GPU.

A batch of 32 uint8 clips of 3x64x256x340, 8 frames kept, 2 views, 224x224 f16 output:
FusedContrastiveTransform = three colour launches (pv_colorjitter_stats / _apply / _vblur) and one
pv_clip_transform_rrc.  Reports from CUDA events the time per batch and per launch (each launch timed on its own,
over the same views), the launches per batch, each launch's HBM bytes computed from the shapes and the draws, and its
achieved GB/s against the H100 SXM's 3.35 TB/s; for comparison, the unfused composition of this package's ops (per
view: frame selection and /255, ColorJitterVideoSSl, then FusedClipTransform's RandomResizedCrop mode).  Prints the card
name and power limit.

    python tools/bench_color.py [--iters 20] [--out results/bench_color.json]
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
B, T, H, W, N_T, V, OUT = 32, 64, 256, 340, 8, 2, 224
RECIPE = dict(bri_con_sat=[0.6, 0.6, 0.6], hue=0.15, p_color_jitter=0.8, p_convert_gray=0.2)
MEAN, STD = (0.45, 0.45, 0.45), (0.225, 0.225, 0.225)
RRC = dict(target_height=OUT, target_width=OUT, scale=(0.2, 0.766), aspect_ratio=(0.75, 1.3333))


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from pytorchvideo_b200 import _lib as L
    from pytorchvideo_b200.transforms import ColorJitterVideoSSl, FusedClipTransform, FusedContrastiveTransform
    from pytorchvideo_b200.transforms import color as CJ
    from pytorchvideo_b200.transforms import functional as Fv
    dev = torch.device("cuda:0")
    results = {"card": card(), "shape": [B, 3, T, H, W], "kept_frames": N_T, "views": V, "out": [OUT, OUT]}
    print("card:", results["card"])
    g = torch.Generator().manual_seed(0)
    x = torch.randint(0, 256, (B, 3, T, H, W), generator=g, dtype=torch.uint8).to(dev)
    tr = FusedContrastiveTransform(N_T, MEAN, STD, **RECIPE, **RRC, hflip_prob=0.5, num_views=V,
                                   out_dtype=torch.float16)
    torch.manual_seed(0)
    before = L.kernel_counts()
    tr(x)
    torch.cuda.synchronize()
    after = L.kernel_counts()
    launches = {k: v - before.get(k, 0) for k, v in after.items() if v != before.get(k, 0)}
    results["launches_per_batch"] = launches
    results["ms_per_batch"] = round(timed(lambda: tr(x), args.iters), 3)

    # each launch on its own, over one batch's draws
    torch.manual_seed(1)
    idx = Fv.temporal_indices(T, N_T)
    draws = [[tr.sample(N_T, H, W) for _ in range(V)] for _ in range(B)]
    order = [(b, v) for v in range(V) for b in range(B)]
    views = [draws[b][v][0] for b, v in order]
    plan = CJ.plan_views(x, views, [b for b, _ in order], frame_idx=idx, src_scale=1)
    frame = N_T * H * W * 3
    n_contrast = sum(1 for vw in views if 1 in vw.order)
    n_blur = sum(1 for vw in views if vw.sigma is not None and CJ.box_blur_params(vw.sigma) is not None)
    nbytes = {"stats": n_contrast * frame, "apply": len(views) * 2 * frame, "vblur": n_blur * 2 * frame}
    kern = {}
    for stage in CJ.STAGES:
        us = timed(lambda: CJ.launch_stage(plan, stage), args.iters) * 1e3
        kern["colorjitter_" + stage] = {"us": round(us, 1), "bytes": nbytes[stage],
                                        "GBps": round(nbytes[stage] / (us * 1e-6) / 1e9, 1),
                                        "share_of_hbm": round(nbytes[stage] / (us * 1e-6) / (HBM_TBS * 1e12), 3)}
    u8 = plan["out"]
    boxes = [draws[b][v][1] for b, v in order]
    flips = [draws[b][v][2] for b, v in order]
    rrc_read = sum(3 * h * w for bx in boxes for (_, _, h, w) in bx)      # each window's source pixels, at least once
    rrc_bytes = rrc_read + len(views) * 3 * N_T * OUT * OUT * 2
    us = timed(lambda: Fv.clip_transform_rrc(u8, boxes, (OUT, OUT), flips=flips, mean=MEAN, std=STD, div255=True,
                                             out_dtype=torch.float16), args.iters) * 1e3
    kern["clip_transform_rrc"] = {"us": round(us, 1), "bytes": rrc_bytes, "GBps": round(rrc_bytes / (us * 1e-6) / 1e9, 1),
                                  "share_of_hbm": round(rrc_bytes / (us * 1e-6) / (HBM_TBS * 1e12), 3)}
    results["kernels"] = kern
    results["views_with_contrast"], results["views_blurred"] = n_contrast, n_blur

    # unfused: per view, frame selection + /255, ColorJitterVideoSSl, then FusedClipTransform's RandomResizedCrop mode
    cj = ColorJitterVideoSSl(**RECIPE)
    tail = FusedClipTransform(None, MEAN, STD, div255=False, out_dtype=torch.float16, random_resized_crop=RRC,
                              hflip_prob=0.5)

    def unfused():
        sub = Fv.clip_transform_batch(x, frame_idx=idx, div255=True, out_dtype=torch.float32)
        return [tail(cj(sub)) for _ in range(V)]

    torch.manual_seed(0)
    results["unfused_ms_per_batch"] = round(timed(unfused, max(2, args.iters // 4)), 3)
    print(json.dumps(results))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(results, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
