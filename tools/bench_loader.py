"""ClipBatchLoader throughput on a seeded Charades-like frame set: 8 clips x 32 frames -> SlowFast [slow, fast] f16 224².

Writes 48 videos of 64 JPEG frames (340x256, 320x240 and 480x270 at q90; half of them with a restart marker per MCU row)
to a temporary directory with a Charades frame csv, then times, in ms per batch and frames/s:
  * loader_w0 / loader_w8 : ClipBatchLoader with 0 and 8 DataLoader workers (one decode, one transform launch a batch)
  * per_sample            : the dataset's normal mode, FusedClipTransform per sample, torch.stack per batch
  * cv2_cpu_w8            : a CPU restatement in 8 workers (cv2.imdecode, torch bilinear resize, crop, normalise),
                            collated and copied to the GPU
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
import torch.nn.functional as F  # noqa: E402

from pytorchvideo_b200 import data as D  # noqa: E402
from pytorchvideo_b200.transforms import FusedClipTransform  # noqa: E402

SIZES = [(256, 340), (240, 320), (270, 480)]
N_VIDEOS, N_FRAMES, CLIP_T, BATCH = 48, 64, 32, 8
MEAN, STD = (0.45, 0.45, 0.45), (0.225, 0.225, 0.225)


def write_frames(root):
    rows = ["original_vido_id video_id frame_id path labels"]
    for v in range(N_VIDEOS):
        h, w = SIZES[v % 3]
        rng = np.random.default_rng(v)
        y, x = np.mgrid[0:h, 0:w].astype(np.float32)
        params = [cv2.IMWRITE_JPEG_QUALITY, 90]
        if v % 2:
            params += [cv2.IMWRITE_JPEG_RST_INTERVAL, (w + 15) // 16]
        os.makedirs(os.path.join(root, "v%02d" % v))
        for t in range(N_FRAMES):
            img = np.stack([(x + 4 * t) % 256, y * 255 / h, 128 + 80 * np.sin((x + y + t) / 9.0)], -1)
            img = np.clip(img + rng.normal(0, 6, img.shape), 0, 255).astype(np.uint8)
            rel = "v%02d/%05d.jpg" % (v, t)
            ok, buf = cv2.imencode(".jpg", img, params)
            assert ok
            with open(os.path.join(root, rel), "wb") as f:
                f.write(buf.tobytes())
            rows.append('v%02d %d %d %s "%d"' % (v, v, t, rel, v % 157))
    with open(os.path.join(root, "frames.csv"), "w") as f:
        f.write("\n".join(rows) + "\n")


def dataset(root):
    return D.Charades(os.path.join(root, "frames.csv"), D.UniformClipSampler(Fraction(CLIP_T, 30)),
                      torch.utils.data.SequentialSampler, video_path_prefix=root)


def transform():
    return FusedClipTransform(CLIP_T, MEAN, STD, random_short_side=(256, 320), crop=("random", 224), hflip_prob=0.5,
                              slowfast_alpha=4, out_dtype=torch.float16)


class CpuClips(torch.utils.data.Dataset):
    """The CPU restatement: per clip, cv2 decodes, torch resizes (bilinear), crops at the centre and normalises."""

    def __init__(self, root):
        self.clips = []
        for v in range(N_VIDEOS):
            for c in range(N_FRAMES // CLIP_T):
                self.clips.append([os.path.join(root, "v%02d/%05d.jpg" % (v, c * CLIP_T + t)) for t in range(CLIP_T)])

    def __len__(self):
        return len(self.clips)

    def __getitem__(self, i):
        frames = [cv2.cvtColor(cv2.imdecode(np.fromfile(p, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)
                  for p in self.clips[i]]
        x = torch.from_numpy(np.stack(frames)).permute(0, 3, 1, 2).float() / 255.0     # (T, 3, H, W)
        h, w = x.shape[-2:]
        nh, nw = (256, int(w * 256 / h)) if h < w else (int(h * 256 / w), 256)
        x = F.interpolate(x, size=(nh, nw), mode="bilinear", align_corners=False)
        top, left = (nh - 224) // 2, (nw - 224) // 2
        x = x[..., top:top + 224, left:left + 224]
        x = (x - torch.tensor(MEAN).view(1, 3, 1, 1)) / torch.tensor(STD).view(1, 3, 1, 1)
        fast = x.permute(1, 0, 2, 3).contiguous()
        return fast[:, torch.linspace(0, CLIP_T - 1, CLIP_T // 4).long()], fast


def per_sample(root, tr):
    cur = []
    for s in dataset(root):
        cur.append(tr(s["video"]))
        if len(cur) == BATCH:
            yield [torch.stack([c[0] for c in cur]), torch.stack([c[1] for c in cur])]
            cur = []


def cpu_batches(root):
    for slow, fast in torch.utils.data.DataLoader(CpuClips(root), batch_size=BATCH, num_workers=8, drop_last=True):
        yield [slow.cuda(non_blocking=True).half(), fast.cuda(non_blocking=True).half()]


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
        raise SystemExit("bench_loader measures on the GPU; no CUDA device is visible")
    torch.manual_seed(0)
    with tempfile.TemporaryDirectory() as root:
        write_frames(root)
        tr = transform()
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            it = iter(D.ClipBatchLoader(dataset(root), BATCH, tr))
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
            res = {"card": card(), "batch": "%d clips x %d frames -> SlowFast [slow, fast] f16 224^2" % (BATCH, CLIP_T),
                   "frames": "48 videos x 64 frames, 340x256 / 320x240 / 480x270 q90, half with RST per MCU row"}
            res["loader_w0"] = timed(D.ClipBatchLoader(dataset(root), BATCH, tr, drop_last=True))
            res["loader_w8"] = timed(D.ClipBatchLoader(dataset(root), BATCH, tr, num_workers=8, drop_last=True))
            res["per_sample"] = timed(per_sample(root, tr))
            res["cv2_cpu_w8"] = timed(cpu_batches(root))
            res["cpu_threads"] = os.cpu_count()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
