"""DetectionBatchLoader throughput on a seeded AVA-like frame set: 8 SlowFast detection clips x 32 frames with their
boxes -> [slow, fast] f16 224² and the fp32 RoI rows.

Writes 32 videos of 150 JPEG frames at 30 fps (340x256, 320x240 and a portrait 256x340, q90), an AVA frame list and a
labels csv with keyframes at seconds 902, 903 and 904 of every video, 1 to 6 boxes each, to a temporary directory.
Then times, in ms per batch and frames/s, with random short side (256..320), random 224 crop and flip:
  * loader_w0 / loader_w8 : DetectionBatchLoader with 0 and 8 DataLoader workers (one decode, one clip launch and one
                            box launch a batch)
  * per_sample            : Ava's normal mode, boxes to pixels in torch and FusedDetectionTransform per sample,
                            stacked and concatenated per batch
``--profile`` instead records a few loader batches with torch.profiler and prints the CUDA time per kernel.
The card's name and power limit are read in the same run.  The result is printed as JSON, and also written to the
file ``--out`` names.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from fractions import Fraction

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from pytorchvideo_b200 import data as D  # noqa: E402
from pytorchvideo_b200.transforms import FusedDetectionTransform  # noqa: E402

SIZES = [(256, 340), (240, 320), (340, 256)]
N_VIDEOS, N_FRAMES, CLIP_T, BATCH = 32, 150, 32, 8
KEYFRAMES = (902, 903, 904)
MEAN, STD = (0.45, 0.45, 0.45), (0.225, 0.225, 0.225)


def write_frames(root):
    rows, labels = ["original_vido_id video_id frame_id path labels"], []
    rng = np.random.default_rng(0)
    for v in range(N_VIDEOS):
        h, w = SIZES[v % 3]
        y, x = np.mgrid[0:h, 0:w].astype(np.float32)
        os.makedirs(os.path.join(root, "v%02d" % v))
        for t in range(N_FRAMES):
            img = np.stack([(x + 4 * t) % 256, y * 255 / h, 128 + 80 * np.sin((x + y + t) / 9.0)], -1)
            img = np.clip(img + rng.normal(0, 6, img.shape), 0, 255).astype(np.uint8)
            rel = "v%02d/%05d.jpg" % (v, t + 1)
            ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])
            assert ok
            with open(os.path.join(root, rel), "wb") as f:
                f.write(buf.tobytes())
            rows.append('v%02d %d %d %s ""' % (v, v, t, rel))
        for sec in KEYFRAMES:
            for _ in range(int(rng.integers(1, 7))):
                x1, y1 = rng.uniform(0, 0.7, 2)
                x2, y2 = x1 + rng.uniform(0.1, 0.3), y1 + rng.uniform(0.1, 0.3)
                labels.append("v%02d,%04d,%.3f,%.3f,%.3f,%.3f,%d,%d" % (v, sec, x1, y1, x2, y2, rng.integers(1, 81), 0))
    with open(os.path.join(root, "frames.csv"), "w") as f:
        f.write("\n".join(rows) + "\n")
    with open(os.path.join(root, "labels.csv"), "w") as f:
        f.write("\n".join(labels) + "\n")


def dataset(root):
    return D.Ava(os.path.join(root, "frames.csv"), os.path.join(root, "labels.csv"), root,
                 clip_sampler=D.UniformClipSampler(Fraction(CLIP_T, 30)),
                 video_sampler=torch.utils.data.SequentialSampler)


def transform():
    return FusedDetectionTransform(CLIP_T, MEAN, STD, random_short_side=(256, 320), crop=("random", 224),
                                   hflip_prob=0.5, slowfast_alpha=4, out_dtype=torch.float16)


def per_sample(root, tr):
    cur = []
    for s in dataset(root):
        H, W = s["video"].shape[-2:]
        b = torch.tensor(s["boxes"], dtype=torch.float32) * torch.tensor([W, H, W, H], dtype=torch.float32)
        cur.append(tr(s["video"], b))
        if len(cur) == BATCH:
            rois = []
            for pos, (_, r) in enumerate(cur):
                r[:, 0] = pos
                rois.append(r)
            yield [torch.stack([v[0] for v, _ in cur]), torch.stack([v[1] for v, _ in cur])], torch.cat(rois)
            cur = []


def timed(batches, warmup=2):
    """ms per batch over the batches after the first ``warmup`` (host clock, each batch ending in a synchronise)."""
    n, t0 = 0, None
    for i, b in enumerate(batches):
        torch.cuda.synchronize()
        if i == warmup - 1:
            t0 = time.perf_counter()
        elif i >= warmup:
            n += 1
        del b
    dt = time.perf_counter() - t0
    return {"batches": n, "ms_per_batch": 1e3 * dt / n, "frames_per_s": n * BATCH * CLIP_T / dt}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown: " + q.stderr.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ava_loader measures on the GPU; no CUDA device is visible")
    torch.manual_seed(0)
    np.random.seed(0)
    with tempfile.TemporaryDirectory() as root:
        write_frames(root)
        tr = transform()
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            it = iter(D.DetectionBatchLoader(dataset(root), BATCH, tr))
            next(it)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(4):
                    next(it)
                torch.cuda.synchronize()
            kern = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA":
                    kern[e.key] = {"calls": e.count, "ms_total": e.device_time_total / 1e3}
            res = {"card": card(), "batches": 4, "kernels": kern}
        else:
            res = {"card": card(), "batch": "%d clips x %d frames + boxes -> SlowFast [slow, fast] f16 224^2 and RoI "
                                             "rows" % (BATCH, CLIP_T),
                   "frames": "%d videos x %d frames, 340x256 / 320x240 / 256x340 q90, %d keyframes each, 1-6 boxes"
                             % (N_VIDEOS, N_FRAMES, len(KEYFRAMES))}
            res["loader_w0"] = timed(D.DetectionBatchLoader(dataset(root), BATCH, tr, drop_last=True))
            res["loader_w8"] = timed(D.DetectionBatchLoader(dataset(root), BATCH, tr, num_workers=8, drop_last=True))
            res["per_sample"] = timed(per_sample(root, tr))
            res["cpu_threads"] = os.cpu_count()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
